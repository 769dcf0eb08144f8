"""Boundary-MPS contraction of 2D tensor networks on the device: the
array-level mirror of quimb's ``TensorNetwork2D.contract_boundary``
(``mode='mps'``) for BASELINE config 5 (PEPS norm, two-layer boundary).

What is mirrored, with the reference line it follows
(quimb/tensor/tn2d/core.py unless noted):

  contract_boundary / interleaved sequence      :2322-2500, :2502-2647
  one inward step (absorb a row, layer by layer,
      canonize the boundary row, compress it)   :1355-1484 (_contract_boundary_core)
  sweep orders of canonize_plane/compress_plane :842-935 (gen_pairs), :937-971, :1085-1129
  compress_between: fuse multibonds, QR-only
      shortcut when cutoff == 0                 tensor_core.py:6667-6762
  canonize_between / tensor_canonize_bond       tensor_core.py:671-824
  tensor_compress_bond(reduced='left')          tensor_core.py:1023-1037
  multibond fusion                              tensor_core.py:1119-1238

The network is given as labelled arrays ``(array, inds, (i, j), layer)``;
nothing of quimb's tag / index machinery is needed beyond "which tensors sit at
a site" and "which indices two tensors share".  Every contraction is a launch
of the pairwise kernel (tree executor for the multi-tensor merges), every
canonize / compress goes through the device QR / Jacobi SVD; the only host
reads are the kept ranks of the truncated SVDs.

Truncation makes the result an approximation of the exact contraction, but a
deterministic one: with the same sequence of gauge moves the value agrees with
the reference's to rounding (truncated SVDs are gauge independent), which is
how the parity tests pin it (tests/golden/boundary.*).
"""

import itertools

import numpy as np

from . import ops
from .array import Array
from .split import tensor_canonize_bond, tensor_compress_bond
from .tree import tensor_contract


class LTensor:
    """A device array with index names, the site(s) it sits on and its layer."""

    __slots__ = ("data", "inds", "layer", "left_inds")

    def __init__(self, data, inds, layer=None):
        self.data = ops.asarray(data)
        self.inds = tuple(inds)
        self.layer = layer
        self.left_inds = None
        if len(self.inds) != self.data.ndim:
            raise ValueError(f"indices {self.inds} do not match shape {self.data.shape}")

    def ind_size(self, ix):
        return self.data.shape[self.inds.index(ix)]

    def size_of(self, inds):
        n = 1
        for ix in inds:
            n *= self.ind_size(ix)
        return n


def _group_inds(ta, tb):
    """(left, shared, right) index tuples (tensor_core.py: group_inds)."""
    sb = set(tb.inds)
    sa = set(ta.inds)
    left = tuple(ix for ix in ta.inds if ix not in sb)
    shared = tuple(ix for ix in ta.inds if ix in sb)
    right = tuple(ix for ix in tb.inds if ix not in sa)
    return left, shared, right


def _contract(tensors, output_inds=None, optimize="auto"):
    data, inds = tensor_contract([t.data for t in tensors], [t.inds for t in tensors],
                                 output_inds=output_inds, optimize=optimize)
    return LTensor(data, inds)


def _fuse(t, shared, bond):
    """Fuse the indices ``shared`` of ``t`` into one index named ``bond`` placed
    where the first of them was (Tensor.fuse; one permute-copy kernel)."""
    pos = min(t.inds.index(ix) for ix in shared)
    rest = [ix for ix in t.inds if ix not in shared]
    order = rest[:pos] + list(shared) + rest[pos:]
    x = t.data.transpose(*[t.inds.index(ix) for ix in order])
    shape = ([t.ind_size(ix) for ix in rest[:pos]] + [t.size_of(shared)]
             + [t.ind_size(ix) for ix in rest[pos:]])
    t.data = x.reshape(*shape)
    t.inds = tuple(rest[:pos] + [bond] + rest[pos:])
    t.left_inds = None


def make_single_bond(ta, tb):
    """tensor_make_single_bond (tensor_core.py:1171-1238): fuse multibonds in
    place; returns (left, bond or None, right)."""
    left, shared, right = _group_inds(ta, tb)
    if not shared:
        return left, None, right
    bond = shared[0]
    if len(shared) > 1:
        _fuse(ta, shared, bond)
        _fuse(tb, shared, bond)
    return left, bond, right


def canonize_between(ta, tb, absorb="right"):
    """QR ``ta`` over its (fused) bond with ``tb`` and absorb R into ``tb``
    (tensor_canonize_bond, tensor_core.py:671-824), in place."""
    if absorb == "left":
        return canonize_between(tb, ta, "right")
    lix, bond, _ = make_single_bond(ta, tb)
    if bond is None:
        return
    if ta.left_inds is not None and set(ta.left_inds) == set(lix):
        return                       # already isometric w.r.t. the bond (:780-786)
    ta.data, tb.data = tensor_canonize_bond(ta.data, ta.inds, tb.data, tb.inds, "right")
    ta.left_inds = lix
    tb.left_inds = None


def compress_between(ta, tb, max_bond=None, cutoff=1e-10, absorb="both",
                     reduced=True, cutoff_mode="rel", method="svd", info=None):
    """_compress_between_tids (tensor_core.py:6667-6762, mode='basic'), in
    place on the two labelled tensors."""
    lix, bond, rix = make_single_bond(ta, tb)
    if bond is None:
        return
    if max_bond is not None and cutoff == 0.0:
        lsize, rsize = ta.size_of(lix), tb.size_of(rix)
        if lsize <= max_bond or rsize <= max_bond:
            # a QR already bounds the bond: no SVD needed (:6692-6721)
            c_abs = "right" if lsize <= rsize else "left"
            canonize_between(ta, tb, c_abs)
            if absorb != c_abs:
                canonize_between(ta, tb, absorb)
            return
    ta.data, tb.data = tensor_compress_bond(
        ta.data, ta.inds, tb.data, tb.inds, max_bond=max_bond, cutoff=cutoff,
        cutoff_mode=cutoff_mode, absorb=absorb, reduced=reduced, method=method,
        info=info)
    ta.left_inds = lix if absorb == "right" else None
    tb.left_inds = rix if absorb == "left" else None


def _gen_pairs(irange, jrange, plane, reverse):
    """Bonds of one boundary line in sweep order (gen_pairs, :842-935, for a
    line of width one): coordinates are (i, j) in network orientation."""
    (i,) = set(irange)
    js = range(min(jrange), max(jrange) + 1)
    js = list(reversed(js)) if reverse else list(js)
    step = -1 if reverse else +1
    for j in js:
        jn = j + step
        if min(jrange) <= jn <= max(jrange):
            if plane == "x":
                yield (i, j), (i, jn)
            else:
                yield (j, i), (jn, i)


class BoundaryContractor2D:
    """The state of a 2D network while its boundaries are contracted inwards.

    Parameters
    ----------
    tensors : iterable of (array, inds, (i, j), layer)
        ``layer`` is a tag such as 'KET' / 'BRA' or None for flat networks.
    Lx, Ly : int
    widen : bool
        float32 / complex64 networks are held in double precision internally
        (one conversion per input tensor).
    """

    def __init__(self, tensors, Lx, Ly, widen=True):
        self.Lx, self.Ly = int(Lx), int(Ly)
        self.sites = {(i, j): [] for i in range(self.Lx) for j in range(self.Ly)}
        for data, inds, coo, layer in tensors:
            data = ops.asarray(data)
            if widen and data.dtype in (np.float32, np.complex64):
                # single precision: widen ONCE here instead of around every
                # contraction / factorisation (the fp64 engines would convert
                # each operand and result on the fly: three extra HBM passes per
                # step); the value is then at least as accurate as the
                # reference's single-precision arithmetic
                from .contract import _WIDE, convert
                src = ops.materialize(data).t
                data = Array(convert(src, _WIDE[src.dtype]))
            self.sites[tuple(coo)].append(LTensor(data, inds, layer))
        self.n_compress = 0
        self.max_bond_seen = 1

    # ---- site helpers -----------------------------------------------------
    def _merge_site(self, coo):
        ts = self.sites[coo]
        if len(ts) > 1:
            self.sites[coo] = [_contract(ts)]
        return self.sites[coo][0] if self.sites[coo] else None

    def _line(self, plane, i, jrange, reverse):
        return _gen_pairs((i,), jrange, plane, reverse)

    def canonize_plane(self, plane, i, jrange, reverse, absorb="right"):
        for ca, cb in self._line(plane, i, jrange, reverse):
            if not self.sites[ca] or not self.sites[cb]:
                continue
            ta, tb = self._merge_site(ca), self._merge_site(cb)
            canonize_between(ta, tb, absorb)

    def compress_plane(self, plane, i, jrange, reverse, max_bond, cutoff,
                       absorb="right", reduced="left", **opts):
        for ca, cb in self._line(plane, i, jrange, reverse):
            if not self.sites[ca] or not self.sites[cb]:
                continue
            ta, tb = self._merge_site(ca), self._merge_site(cb)
            compress_between(ta, tb, max_bond=max_bond, cutoff=cutoff,
                             absorb=absorb, reduced=reduced, **opts)
            self.n_compress += 1
            _, shared, _ = _group_inds(ta, tb)
            for ix in shared:
                self.max_bond_seen = max(self.max_bond_seen, ta.ind_size(ix))

    # ---- one inward step (tn2d/core.py:1355-1484) ----------------------------
    def contract_boundary_from(self, xrange, yrange, from_which, max_bond,
                               cutoff=1e-10, canonize=True, layer_tags=None,
                               sweep_reverse=False, compress_opts=None,
                               canonize_opts=None):
        plane = from_which[0]
        irange, jrange = (xrange, yrange) if plane == "x" else (yrange, xrange)
        imin, imax = sorted(irange)
        if "min" in from_which:
            sweep, istep = range(imin, imax + 1), +1
        else:
            sweep, istep = range(imax, imin - 1, -1), -1
        site = (lambda i, j: (i, j)) if plane == "x" else (lambda i, j: (j, i))
        copts = dict(compress_opts or {})
        copts.setdefault("absorb", "right")
        copts.setdefault("reduced", "left")
        qopts = dict(canonize_opts or {})
        qopts.setdefault("absorb", "right")
        layers = list(layer_tags) if layer_tags is not None else [None]
        for i in list(sweep)[:-1]:
            for layer in layers:
                for j in range(min(jrange), max(jrange) + 1):
                    c1, c2 = site(i, j), site(i + istep, j)
                    if not self.sites[c1] or not self.sites[c2]:
                        continue
                    if layer is None or len(self.sites[c2]) == 1:
                        # contract *any* tensors with the pair of coordinates
                        merged = _contract(self.sites[c1] + self.sites[c2])
                        self.sites[c1], self.sites[c2] = [merged], []
                        absorbed_all = True
                    else:
                        t1 = self._merge_site(c1)
                        inner = [t for t in self.sites[c2] if t.layer == layer]
                        if len(inner) != 1:
                            raise ValueError(f"site {c2}: expected one tensor of "
                                             f"layer {layer!r}, found {len(inner)}")
                        merged = _contract([t1, inner[0]])
                        self.sites[c1] = [merged]
                        self.sites[c2] = [t for t in self.sites[c2] if t is not inner[0]]
                        absorbed_all = not self.sites[c2]
                    del absorbed_all
                # compress_late (the default): gauge, then compress, the line
                if canonize:
                    self.canonize_plane(plane, i, jrange, not sweep_reverse, **qopts)
                self.compress_plane(plane, i, jrange, sweep_reverse, max_bond, cutoff,
                                    **copts)
            # the boundary now lives on line i + istep
            for j in range(min(jrange), max(jrange) + 1):
                c1, c2 = site(i, j), site(i + istep, j)
                self.sites[c2] = self.sites[c1] + self.sites[c2]
                self.sites[c1] = []

    # ---- full contraction (tn2d/core.py:2322-2500) ---------------------------
    def contract_boundary(self, max_bond=None, cutoff=1e-10, canonize=True,
                          layer_tags=None, compress_opts=None, sequence=None,
                          max_separation=1, max_unfinished=1, final_contract=True,
                          optimize="auto", strip_exponent=False, **step_opts):
        b = {"xmin": 0, "xmax": self.Lx - 1, "ymin": 0, "ymax": self.Ly - 1}
        sep = {"x": b["xmax"] - b["xmin"], "y": b["ymax"] - b["ymin"]}
        if sequence is None:
            sequence = ("xmin", "xmax") if self.Lx >= self.Ly else ("ymin", "ymax")
        elif isinstance(sequence, str):
            sequence = (sequence,)
        for d in sequence:
            if d not in b:
                raise ValueError(f"invalid boundary direction {d!r}")

        def finished(d):
            return sep[d[0]] <= max_separation

        sequence = [d for d in sequence if not finished(d)]
        while sequence:
            d = sequence.pop(0)
            if finished(d):
                continue
            sequence.append(d)
            if d[0] == "x":
                xr = (b["xmin"], b["xmin"] + 1) if d == "xmin" else (b["xmax"] - 1, b["xmax"])
                yr = (b["ymin"], b["ymax"])
            else:
                yr = (b["ymin"], b["ymin"] + 1) if d == "ymin" else (b["ymax"] - 1, b["ymax"])
                xr = (b["xmin"], b["xmax"])
            self.contract_boundary_from(xr, yr, d, max_bond, cutoff=cutoff,
                                        canonize=canonize, layer_tags=layer_tags,
                                        compress_opts=compress_opts, **step_opts)
            sep[d[0]] -= 1
            b[d] += 1 if d.endswith("min") else -1
            if sum(sep[w] > max_separation for w in "xy") <= max_unfinished:
                break
        if not final_contract:
            return self
        rest = list(itertools.chain.from_iterable(
            self.sites[c] for c in sorted(self.sites)))
        data, inds = tensor_contract([t.data for t in rest], [t.inds for t in rest],
                                     optimize=optimize, strip_exponent=strip_exponent)
        if strip_exponent:
            return data
        return data if inds else (data.item() if isinstance(data, Array) else data)


    # ---- environments (tn2d/core.py:2716-2835, :3075-3431) ------------------
    # An environment is a snapshot ``{(i, j): [LTensor, ...]}`` of the tensors
    # the reference selects by tag: the boundary line (or the raw first line,
    # or one dense tensor) on the coordinates it was contracted onto.  The
    # snapshot holds its own LTensor wrappers: canonize / compress replace
    # ``.data`` of the wrappers they touch with new arrays and never write into
    # an array, so a snapshot shares device memory but no mutable state.
    def _copy(self):
        bc = BoundaryContractor2D.__new__(BoundaryContractor2D)
        bc.Lx, bc.Ly = self.Lx, self.Ly
        bc.sites = {c: [_clone(t) for t in ts] for c, ts in self.sites.items()}
        bc.n_compress, bc.max_bond_seen = 0, 1
        return bc

    def _snapshot(self, coos):
        return {c: [_clone(t) for t in self.sites[c]] for c in coos if self.sites[c]}

    def compute_environments(self, from_which, xrange=None, yrange=None, max_bond=None, *,
                             cutoff=1e-10, canonize=True, layer_tags=None, dense=False):
        """``envs[from_which, i]`` for every line ``i`` of the sweep
        (compute_environments, tn2d/core.py:2716-2835): empty for the first
        line, the raw first line for the second, then the boundary after each
        inward step, or with ``dense`` the exact contraction of every line so
        far into one tensor.  The contractor itself is left unchanged."""
        if from_which not in ("xmin", "xmax", "ymin", "ymax"):
            raise ValueError(f"invalid boundary direction {from_which!r}")
        xrange = (0, self.Lx - 1) if xrange is None else tuple(xrange)
        yrange = (0, self.Ly - 1) if yrange is None else tuple(yrange)
        tn = self._copy()
        plane = from_which[0]
        irange, jrange = (xrange, yrange) if plane == "x" else (yrange, xrange)
        imin, imax = sorted(irange)
        step = +1 if "min" in from_which else -1
        sweep = list(range(imin, imax + 1)) if step > 0 else list(range(imax, imin - 1, -1))
        n_other = self.Ly if plane == "x" else self.Lx
        jmin = min(jrange)

        def site(i, j):
            return (i, j) if plane == "x" else (j, i)

        def line(i):
            # a line tag selects the whole row / column, not just jrange
            return [site(i, j) for j in range(n_other)]

        def merge_lines(*lines):
            ts = [t for i in lines for c in line(i) for t in tn.sites[c]]
            for i in lines:
                for c in line(i):
                    tn.sites[c] = []
            tn.sites[site(lines[-1], jmin)] = [_contract(ts)]

        envs = {(from_which, sweep[0]): {}}
        if len(sweep) < 2:
            return envs
        if dense:
            merge_lines(sweep[0])
        envs[from_which, sweep[1]] = tn._snapshot(line(sweep[0]))
        for i in sweep[2:]:
            iprevprev, iprev = i - 2 * step, i - step
            if dense:
                merge_lines(iprevprev, iprev)
            else:
                xr = (iprevprev, iprev) if plane == "x" else xrange
                yr = (iprevprev, iprev) if plane == "y" else yrange
                tn.contract_boundary_from(xr, yr, from_which, max_bond, cutoff=cutoff,
                                          canonize=canonize, layer_tags=layer_tags)
            envs[from_which, i] = tn._snapshot(line(iprev))
        return envs

    def compute_x_environments(self, max_bond=None, *, cutoff=1e-10, canonize=True,
                               layer_tags=None, dense=False, yrange=None):
        """The 'xmin' and 'xmax' environments of every row."""
        envs = {}
        for side in ("xmin", "xmax"):
            envs.update(self.compute_environments(side, None, yrange, max_bond, cutoff=cutoff,
                                                  canonize=canonize, layer_tags=layer_tags,
                                                  dense=dense))
        return envs

    def compute_y_environments(self, max_bond=None, *, cutoff=1e-10, canonize=True,
                               layer_tags=None, dense=False, xrange=None):
        """The 'ymin' and 'ymax' environments of every column."""
        envs = {}
        for side in ("ymin", "ymax"):
            envs.update(self.compute_environments(side, xrange, None, max_bond, cutoff=cutoff,
                                                  canonize=canonize, layer_tags=layer_tags,
                                                  dense=dense))
        return envs

    def compute_plaquette_environments(self, x_bsz=2, y_bsz=2, max_bond=None, *,
                                       cutoff=1e-10, canonize=True, layer_tags=None,
                                       first_contract=None, second_dense=None):
        """``{((i0, j0), (x_bsz, y_bsz)): [LTensor, ...]}``: the environment of
        every plaquette of the given size (compute_plaquette_environments,
        tn2d/core.py:3324-3431).  Rows (``first_contract='x'``) or columns
        are contracted from both sides first; then each strip of ``x_bsz``
        rows (``y_bsz`` columns) between its two environments is contracted
        from both ends in the rotated direction, exactly (``second_dense``,
        the default for a block size of 1) or by boundary sweeps."""
        if first_contract is None:
            if x_bsz != y_bsz:
                first_contract = "y" if x_bsz > y_bsz else "x"
            else:
                first_contract = "x" if self.Lx >= self.Ly else "y"
        if first_contract not in ("x", "y"):
            raise ValueError(f"first_contract must be 'x' or 'y', got {first_contract!r}")
        opts = dict(max_bond=max_bond, cutoff=cutoff, canonize=canonize, layer_tags=layer_tags)
        x_first = first_contract == "x"
        # the first direction's block size, lattice length and coordinate order
        bsz, osz = (x_bsz, y_bsz) if x_first else (y_bsz, x_bsz)
        L = self.Lx if x_first else self.Ly
        if second_dense is None:
            second_dense = bsz < 2
        first = (self.compute_x_environments if x_first else self.compute_y_environments)(**opts)
        a, b = ("xmin", "xmax") if x_first else ("ymin", "ymax")
        c, d = ("ymin", "ymax") if x_first else ("xmin", "xmax")

        def coo(i, j):   # (first-direction index, other index) -> site
            return (i, j) if x_first else (j, i)

        strips = {}
        for i in range(L - bsz + 1):
            strip = BoundaryContractor2D.__new__(BoundaryContractor2D)
            strip.Lx, strip.Ly = self.Lx, self.Ly
            strip.sites = {cc: [] for cc in self.sites}
            strip.n_compress, strip.max_bond_seen = 0, 1
            for env in (first[a, i], first[b, i + bsz - 1]):
                for cc, ts in env.items():
                    strip.sites[cc] += [_clone(t) for t in ts]
            for cc, ts in self.sites.items():
                if i <= cc[0 if x_first else 1] < i + bsz:
                    strip.sites[cc] += [_clone(t) for t in ts]
            rng = (max(i - 1, 0), min(i + bsz, L - 1))
            second = strip.compute_y_environments if x_first else strip.compute_x_environments
            strips[i] = second(dense=second_dense, **opts,
                               **({"xrange": rng} if x_first else {"yrange": rng}))

        def select(env, coos):
            return [t for cc in coos if cc in env for t in env[cc]]

        out = {}
        for i0, j0 in itertools.product(range(L - bsz + 1),
                                        range((self.Ly if x_first else self.Lx) - osz + 1)):
            # the rotated strip's ends span the first-direction neighbours too
            side_lo = [coo(i0 + x, j0 - 1) for x in range(-1, bsz + 1)]
            side_hi = [coo(i0 + x, j0 + osz) for x in range(-1, bsz + 1)]
            below = [coo(i0 - 1, j0 + y) for y in range(osz)]
            above = [coo(i0 + bsz, j0 + y) for y in range(osz)]
            env = (select(strips[i0][c, j0], side_lo) + select(strips[i0][d, j0 + osz - 1], side_hi)
                   + select(first[a, i0], below) + select(first[b, i0 + bsz - 1], above))
            (p0, p1), size = coo(i0, j0), (x_bsz, y_bsz)
            out[(p0, p1), size] = env
        return out


def _clone(t):
    c = LTensor.__new__(LTensor)
    c.data, c.inds, c.layer, c.left_inds = t.data, t.inds, t.layer, t.left_inds
    return c


def contract_boundary(tensors, Lx, Ly, max_bond=None, **opts):
    """``TensorNetwork2D.contract_boundary`` for labelled device arrays; see
    :class:`BoundaryContractor2D`.  Returns a Python scalar for a closed
    network."""
    widen = opts.pop("widen", True)
    return BoundaryContractor2D(tensors, Lx, Ly, widen=widen).contract_boundary(max_bond, **opts)


def peps_norm_tensors(arrays, site_inds=None):
    """Labelled two-layer norm network <psi|psi> of a PEPS given as a grid
    ``arrays[i][j]`` of site arrays with index order (up, right, down, left,
    phys) restricted to the bonds that exist at the site (quimb's PEPS
    convention, tn2d/core.py:4661-4753): the bra layer is the lazily
    conjugated ket (no data is copied), sharing only the physical indices."""
    Lx, Ly = len(arrays), len(arrays[0])
    out = []
    for i in range(Lx):
        for j in range(Ly):
            x = ops.asarray(arrays[i][j])
            names = []
            if i < Lx - 1:
                names.append(("v", i, j))
            if j < Ly - 1:
                names.append(("h", i, j))
            if i > 0:
                names.append(("v", i - 1, j))
            if j > 0:
                names.append(("h", i, j - 1))
            if len(names) + 1 != x.ndim:
                raise ValueError(f"site ({i},{j}): rank {x.ndim} does not match "
                                 f"{len(names)} bonds + 1 physical index")
            phys = f"k{i},{j}"
            kin = tuple(f"K{d}{a},{b}" for d, a, b in names) + (phys,)
            bin_ = tuple(f"B{d}{a},{b}" for d, a, b in names) + (phys,)
            out.append((x, kin, (i, j), "KET"))
            out.append((x.conj(), bin_, (i, j), "BRA"))
    return out, Lx, Ly


# ------------------------------------------------------------ two-sided ------
def _bcast_line(line, src, group, stage):
    """Broadcast the labelled tensors of one boundary line from rank ``src``
    (``line`` is ignored on the other ranks): one object broadcast of the
    metadata, one tensor broadcast per boundary tensor (NVLink under NCCL;
    staged through the host for gloo).  Complex data travels as real pairs."""
    import torch
    import torch.distributed as dist
    from .ops import default_device
    me = dist.get_rank(group)
    meta = [None]
    if me == src:
        meta[0] = [(coo, t.inds, t.layer, tuple(t.data.shape), str(t.data.dtype))
                   for coo, ts in line for t in ts]
    dist.broadcast_object_list(meta, src=src, group=group)
    out = {}
    flat = [t for _, ts in line for t in ts] if me == src else None
    for k, (coo, inds, layer, shape, dtype) in enumerate(meta[0]):
        if me == src:
            buf = ops.materialize(flat[k].data, force=True).t
        else:
            from .array import torch_dtype
            buf = torch.empty(shape, dtype=torch_dtype(dtype), device=default_device())
        wire = torch.view_as_real(buf) if buf.dtype.is_complex else buf
        if stage and wire.device.type != "cpu":
            host = wire.cpu()
            dist.broadcast(host, src=src, group=group)
            wire.copy_(host)
        else:
            dist.broadcast(wire, src=src, group=group)
        out.setdefault(tuple(coo), []).append(LTensor(Array(buf), inds, layer))
    return out


def contract_boundary_two_sided(tensors, Lx, Ly, max_bond=None, cutoff=1e-10,
                                canonize=True, layer_tags=None, compress_opts=None,
                                optimize="auto", group=None, **step_opts):
    """The default interleaved sequence ('xmin', 'xmax') -- or ('ymin', 'ymax')
    for Lx < Ly -- of ``contract_boundary`` with the two opposing half-sweeps
    on different GPUs (SURVEY.md 8e: they are independent,
    tn2d/core.py:2528-2543): rank 0 contracts inwards from the min side, rank 1
    from the max side, the two boundary lines are exchanged (one broadcast
    each, the only communication) and every rank performs the final exact
    contraction of the two lines.  Bit-for-bit the same sequence of operations
    as the single-process run, so the value is identical; ranks >= 2 only
    receive.  Without a process group it runs both halves locally."""
    import torch.distributed as dist
    active = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
    rank = dist.get_rank(group) if active else 0
    plane = "x" if Lx >= Ly else "y"
    L = Lx if plane == "x" else Ly
    n_steps = max(L - 2, 0)
    n_min, n_max = (n_steps + 1) // 2, n_steps // 2
    tensors = list(tensors)
    bc = BoundaryContractor2D(tensors, Lx, Ly, widen=step_opts.pop("widen", True))
    other = (0, (Ly if plane == "x" else Lx) - 1)

    def run(side, count):
        for s in range(count):
            lo = s if side == "min" else L - 2 - s
            rng_i = (lo, lo + 1)
            xr, yr = (rng_i, other) if plane == "x" else (other, rng_i)
            bc.contract_boundary_from(xr, yr, plane + side, max_bond, cutoff=cutoff,
                                      canonize=canonize, layer_tags=layer_tags,
                                      compress_opts=compress_opts, **step_opts)

    def line(i):
        js = range(other[0], other[1] + 1)
        coos = [(i, j) if plane == "x" else (j, i) for j in js]
        return [(c, bc.sites[c]) for c in coos]

    i_min, i_max = n_min, L - 1 - n_max
    if not active:
        run("min", n_min)
        run("max", n_max)
    else:
        if rank == 0:
            run("min", n_min)
        elif rank == 1:
            run("max", n_max)
        stage = dist.get_backend(group) != "nccl"
        got_min = _bcast_line(line(i_min) if rank == 0 else None, 0, group, stage)
        got_max = _bcast_line(line(i_max) if rank == 1 else None, 1, group, stage)
        if rank != 0:
            for c, ts in got_min.items():
                bc.sites[c] = ts
        if rank != 1:
            for c, ts in got_max.items():
                bc.sites[c] = ts
    keep = {c for c, _ in line(i_min)} | {c for c, _ in line(i_max)}
    rest = list(itertools.chain.from_iterable(bc.sites[c] for c in sorted(keep)))
    data, inds = tensor_contract([t.data for t in rest], [t.inds for t in rest],
                                 optimize=optimize)
    return data if inds else (data.item() if isinstance(data, Array) else data)
