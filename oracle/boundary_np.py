"""ORACLE (test infrastructure, never imported by the product package).

numpy restatement of the boundary-MPS contraction of a 2D network,
``TensorNetwork2D.contract_boundary`` with ``mode='mps'``, for labelled
arrays ``(array, inds, (i, j), layer)`` -- the input convention of
quimb_b200/boundary.py.  Written from the reference (quimb/tensor/tn2d/core.py
unless noted); the splits are those of oracle/decomp_np.py and the exact
contractions those of oracle/contract_np.py.

Besides the value, every run keeps a trace: one record per factorisation with
the bond, the kind ('qr' or 'svd'), the shape of the matrix factorised, the
kept rank and the relative gap at the cut.  The gap is
(s[k-1] - s[k]) / s[0] for a cut at rank k, or, when a cutoff decides the rank,
the smaller of that and the distance of the nearest singular value (or tail
sum) from the cutoff's threshold, relative to the largest; ``inf`` when
nothing could be cut (QR).  A kernel that rounds differently can only keep a
different rank where this gap is at rounding level, which is how tests derive
their tolerance from it.
"""

import itertools

import numpy as np

from oracle import contract_np as cnp
from oracle import decomp_np as dnp


class T:
    """An array with index names, its layer tag and the indices it is known
    to be isometric from (``Tensor.left_inds``)."""

    __slots__ = ("data", "inds", "layer", "left_inds")

    def __init__(self, data, inds, layer=None):
        self.data = np.asarray(data)
        self.inds = tuple(inds)
        self.layer = layer
        self.left_inds = None
        assert len(self.inds) == self.data.ndim, (self.inds, self.data.shape)

    def size(self, ix):
        return self.data.shape[self.inds.index(ix)]

    def size_of(self, inds):
        return int(np.prod([self.size(ix) for ix in inds], dtype=np.int64))

    def modify(self, data):
        # Tensor.modify(data=...) forgets left_inds (tensor_core.py:2157-2159)
        self.data = data
        self.left_inds = None


def contract(tensors, output_inds=None, optimize="auto"):
    """tensor_contract of several labelled tensors into one."""
    data, inds = cnp.tensor_contract([t.data for t in tensors], [t.inds for t in tensors],
                                     output_inds=output_inds, optimize=optimize)
    return T(data, inds)


def cut_gap(s, k, cutoff=0.0, cutoff_mode="rel"):
    """Relative gap at a cut at rank ``k`` of the descending values ``s``."""
    s = np.asarray(s, dtype=float)
    if s.size == 0 or s[0] == 0.0:
        return 0.0
    g = (s[k - 1] - s[k]) / s[0] if k < s.size else np.inf
    if cutoff and cutoff > 0.0:
        if cutoff_mode in ("rel", "abs"):
            thr = cutoff * s[0] if cutoff_mode == "rel" else cutoff
            g = min(g, float(np.min(np.abs(s - thr))) / s[0])
        else:
            pw = 2 if "2" in cutoff_mode else 1
            tails = np.cumsum((s ** pw)[::-1])[::-1]
            target = cutoff * (tails[0] if cutoff_mode.startswith("r") else 1.0)
            g = min(g, float(np.min(np.abs(tails - target))) / tails[0])
    return float(g)


# ---- bond operations (tensor_core.py) ---------------------------------------
def group_inds(ta, tb):
    shared = [ix for ix in ta.inds if ix in tb.inds]
    left = tuple(ix for ix in ta.inds if ix not in shared)
    right = tuple(ix for ix in tb.inds if ix not in shared)
    return left, tuple(shared), right


def _fuse(t, group, name):
    """Tensor.fuse: the group becomes one index, at the place of its first
    member, in the group's order (modify(inds=...) forgets left_inds)."""
    first = min(t.inds.index(ix) for ix in group)
    before = [ix for ix in t.inds[:first] if ix not in group]
    after = [ix for ix in t.inds[first:] if ix not in group]
    order = before + list(group) + after
    x = np.transpose(t.data, [t.inds.index(ix) for ix in order])
    shape = [t.size(ix) for ix in before] + [t.size_of(group)] + [t.size(ix) for ix in after]
    t.data = x.reshape(shape)
    t.inds = tuple(before + [name] + after)
    t.left_inds = None


def make_single_bond(ta, tb):
    """tensor_make_single_bond (:1171-1238): multibonds fused into the first
    shared index, in ``ta``'s order on both tensors."""
    left, shared, right = group_inds(ta, tb)
    if not shared:
        return left, None, right
    if len(shared) > 1:
        _fuse(ta, shared, shared[0])
        _fuse(tb, shared, shared[0])
    return left, shared[0], right


def _reorder(x, have, want):
    return np.transpose(x, [tuple(have).index(ix) for ix in want])


def canonize_between(ta, tb, absorb="right", trace=None, label=None):
    """tensor_canonize_bond (:671-824): QR of ``ta`` over the bond, R into
    ``tb``; absorb='left' is the mirror image.  Skipped when ``ta`` is already
    isometric from its other indices (:780-787)."""
    if absorb == "left":
        return canonize_between(tb, ta, "right", trace, label)
    lix, bond, _ = make_single_bond(ta, tb)
    if bond is None:
        return
    if ta.left_inds is not None and set(ta.left_inds) == set(lix):
        return
    q, _, r = dnp.tensor_split(ta.data, ta.inds, lix, (bond,), method="qr")
    if trace is not None:
        m, n = ta.size_of(lix), ta.size(bond)
        trace.append(dict(bond=label, kind="qr", shape=(m, n), rank=min(m, n),
                          gap=np.inf))
    new_b = np.tensordot(r, tb.data, axes=(1, tb.inds.index(bond)))
    rest = tuple(ix for ix in tb.inds if ix != bond)
    ta.modify(_reorder(q, lix + (bond,), ta.inds))
    ta.left_inds = lix
    tb.modify(_reorder(new_b, (bond,) + rest, tb.inds))


def compress_between(ta, tb, max_bond=None, cutoff=1e-10, absorb="both", reduced=True,
                     cutoff_mode="rel", trace=None, label=None):
    """_compress_between_tids (:6667-6772, mode='basic', no gauges):
    multibond fusion, the QR-only shortcut for ``cutoff == 0`` when one side's
    outer size is within ``max_bond``, else tensor_compress_bond (:864-1094)
    with ``reduced`` True or 'left'."""
    lix, bond, rix = make_single_bond(ta, tb)
    if bond is None:
        return
    if max_bond is not None and cutoff == 0.0:
        lsize, rsize = ta.size_of(lix), tb.size_of(rix)
        if lsize <= max_bond or rsize <= max_bond:
            c_absorb = "right" if lsize <= rsize else "left"
            canonize_between(ta, tb, c_absorb, trace, label)
            if absorb != c_absorb:
                canonize_between(ta, tb, absorb, trace, label)
            return
    info = {}
    if reduced is True:
        na, nb = dnp.tensor_compress_bond(ta.data, ta.inds, tb.data, tb.inds,
                                          max_bond=max_bond, cutoff=cutoff,
                                          cutoff_mode=cutoff_mode, absorb=absorb, info=info)
        m = min(ta.size_of(lix), ta.size(bond))
        n = min(tb.size(bond), tb.size_of(rix))
        mark = absorb
    elif reduced == "left":
        # (:1031-1045) SVD of the left tensor alone, the rest into the right one
        left, _, right = dnp.tensor_split(ta.data, ta.inds, lix, (bond,), method="svd",
                                          absorb=absorb, max_bond=max_bond, cutoff=cutoff,
                                          cutoff_mode=cutoff_mode, info=info)
        m, n = ta.size_of(lix), ta.size(bond)
        nb = np.tensordot(right, tb.data, axes=(1, tb.inds.index(bond)))
        rest = tuple(ix for ix in tb.inds if ix != bond)
        na = _reorder(left, lix + (bond,), ta.inds)
        nb = _reorder(nb, (bond,) + rest, tb.inds)
        mark = "both" if absorb == "left" else absorb
    else:
        raise ValueError(f"oracle: reduced={reduced!r} is not restated")
    ta.modify(na)
    tb.modify(nb)
    if mark == "right":
        ta.left_inds = lix
    elif mark == "left":
        tb.left_inds = rix
    if trace is not None:
        k = int(info["n_keep"])
        trace.append(dict(bond=label, kind="svd", shape=(m, n), rank=k,
                          gap=cut_gap(info["svals"], k, cutoff, cutoff_mode)))


# ---- the boundary sweep (tn2d/core.py) --------------------------------------
def _pairs(i, jrange, plane, reverse):
    """gen_pairs (:842-935) for a line of width one: neighbouring sites of
    line ``i`` stepping in the sweep direction."""
    lo, hi = min(jrange), max(jrange)
    js = range(hi, lo - 1, -1) if reverse else range(lo, hi + 1)
    step = -1 if reverse else 1
    for j in js:
        if lo <= j + step <= hi:
            if plane == "x":
                yield (i, j), (i, j + step)
            else:
                yield (j, i), (j + step, i)


class Boundary2D:
    """A 2D network as ``sites[(i, j)] -> [T, ...]`` while it is contracted
    inwards; ``trace`` collects every factorisation."""

    def __init__(self, tensors, Lx, Ly, widen=True):
        self.Lx, self.Ly = int(Lx), int(Ly)
        self.sites = {(i, j): [] for i in range(self.Lx) for j in range(self.Ly)}
        for data, inds, coo, layer in tensors:
            x = np.asarray(data)
            if widen and x.dtype in (np.float32, np.complex64):
                x = x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)
            self.sites[tuple(coo)].append(T(x, inds, layer))
        self.trace = []
        self.n_compress = 0
        self.max_bond_seen = 1

    def _single(self, coo):
        # ``self ^= site_tag``: merge the site into one tensor
        if len(self.sites[coo]) > 1:
            self.sites[coo] = [contract(self.sites[coo])]
        return self.sites[coo][0] if self.sites[coo] else None

    def canonize_plane(self, plane, i, jrange, reverse, absorb="right"):
        """canonize_plane (:937-971)."""
        for ca, cb in _pairs(i, jrange, plane, reverse):
            if not self.sites[ca] or not self.sites[cb]:
                continue
            ta, tb = self._single(ca), self._single(cb)
            canonize_between(ta, tb, absorb, self.trace, (ca, cb))

    def compress_plane(self, plane, i, jrange, reverse, max_bond, cutoff,
                       absorb="right", reduced="left", **opts):
        """compress_plane (:1085-1129)."""
        for ca, cb in _pairs(i, jrange, plane, reverse):
            if not self.sites[ca] or not self.sites[cb]:
                continue
            ta, tb = self._single(ca), self._single(cb)
            compress_between(ta, tb, max_bond=max_bond, cutoff=cutoff, absorb=absorb,
                             reduced=reduced, trace=self.trace, label=(ca, cb), **opts)
            self.n_compress += 1
            for ix in group_inds(ta, tb)[1]:
                self.max_bond_seen = max(self.max_bond_seen, ta.size(ix))

    def contract_boundary_from(self, xrange, yrange, from_which, max_bond, cutoff=1e-10,
                               canonize=True, layer_tags=None, sweep_reverse=False,
                               compress_opts=None, canonize_opts=None):
        """_contract_boundary_core (:1355-1484) with compress_late=True: absorb
        the next line layer by layer, then canonize the boundary line against
        the sweep and compress it along the sweep."""
        plane = from_which[0]
        irange, jrange = (xrange, yrange) if plane == "x" else (yrange, xrange)
        lo, hi = min(irange), max(irange)
        if from_which.endswith("min"):
            sweep, istep = list(range(lo, hi + 1)), 1
        else:
            sweep, istep = list(range(hi, lo - 1, -1)), -1

        def coo(i, j):
            return (i, j) if plane == "x" else (j, i)

        copts = dict(compress_opts or {})
        copts.setdefault("absorb", "right")
        copts.setdefault("reduced", "left")
        qopts = dict(canonize_opts or {})
        qopts.setdefault("absorb", "right")
        for i in sweep[:-1]:
            for layer in (layer_tags if layer_tags is not None else [None]):
                for j in range(min(jrange), max(jrange) + 1):
                    outer, inner = coo(i, j), coo(i + istep, j)
                    if not self.sites[outer] or not self.sites[inner]:
                        continue
                    if layer is None or len(self.sites[inner]) == 1:
                        self.sites[outer] = [contract(self.sites[outer] + self.sites[inner])]
                        self.sites[inner] = []
                    else:
                        t1 = self._single(outer)
                        (t2,) = [t for t in self.sites[inner] if t.layer == layer]
                        self.sites[outer] = [contract([t1, t2])]
                        self.sites[inner] = [t for t in self.sites[inner] if t is not t2]
                if canonize:
                    self.canonize_plane(plane, i, jrange, not sweep_reverse, **qopts)
                self.compress_plane(plane, i, jrange, sweep_reverse, max_bond, cutoff,
                                    **copts)
            # the boundary tensors now carry the next line's site tags
            for j in range(min(jrange), max(jrange) + 1):
                outer, inner = coo(i, j), coo(i + istep, j)
                self.sites[inner] = self.sites[outer] + self.sites[inner]
                self.sites[outer] = []

    def tensors(self):
        return list(itertools.chain.from_iterable(self.sites[c] for c in sorted(self.sites)))

    def close(self, optimize="auto"):
        """The exact contraction of what is left."""
        rest = self.tensors()
        data, _ = cnp.tensor_contract([t.data for t in rest], [t.inds for t in rest],
                                      optimize=optimize)
        return data

    def contract_boundary(self, max_bond=None, cutoff=1e-10, canonize=True, layer_tags=None,
                          compress_opts=None, sequence=None, max_separation=1,
                          max_unfinished=1, final_contract=True, optimize="auto", **step_opts):
        """contract_boundary (:2322-2500): the interleaved sequence of inward
        steps, then the exact contraction of the rest."""
        bounds = {"xmin": 0, "xmax": self.Lx - 1, "ymin": 0, "ymax": self.Ly - 1}
        sep = {"x": self.Lx - 1, "y": self.Ly - 1}
        if sequence is None:
            sequence = ("xmin", "xmax") if self.Lx >= self.Ly else ("ymin", "ymax")
        elif isinstance(sequence, str):
            sequence = (sequence,)

        def done(d):
            return sep[d[0]] <= max_separation

        todo = [d for d in sequence if not done(d)]
        while todo:
            d = todo.pop(0)
            if done(d):
                continue
            todo.append(d)
            if d[0] == "x":
                xr = (bounds[d], bounds[d] + 1) if d == "xmin" else (bounds[d] - 1, bounds[d])
                yr = (bounds["ymin"], bounds["ymax"])
            else:
                yr = (bounds[d], bounds[d] + 1) if d == "ymin" else (bounds[d] - 1, bounds[d])
                xr = (bounds["xmin"], bounds["xmax"])
            self.contract_boundary_from(xr, yr, d, max_bond, cutoff=cutoff, canonize=canonize,
                                        layer_tags=layer_tags, compress_opts=compress_opts,
                                        **step_opts)
            sep[d[0]] -= 1
            bounds[d] += 1 if d.endswith("min") else -1
            if sum(sep[w] > max_separation for w in "xy") <= max_unfinished:
                break
        if not final_contract:
            return self
        return self.close(optimize)


def contract_boundary(tensors, Lx, Ly, max_bond=None, widen=True, **opts):
    """(value, Boundary2D) of the boundary contraction; the value is the
    remaining network (the Boundary2D itself) with ``final_contract=False``."""
    bc = Boundary2D(tensors, Lx, Ly, widen=widen)
    return bc.contract_boundary(max_bond, **opts), bc


def peps_norm_tensors(arrays):
    """<psi|psi> of a PEPS grid ``arrays[i][j]`` (index order up, right, down,
    left, phys over the bonds present; tn2d/core.py:4661-4753) as labelled
    arrays: a 'KET' layer and a conjugated 'BRA' layer sharing the physical
    indices, site by site."""
    Lx, Ly = len(arrays), len(arrays[0])
    out = []
    for i, j in itertools.product(range(Lx), range(Ly)):
        bonds = [("v", i, j)] * (i < Lx - 1) + [("h", i, j)] * (j < Ly - 1)
        bonds += [("v", i - 1, j)] * (i > 0) + [("h", i, j - 1)] * (j > 0)
        x = np.asarray(arrays[i][j])
        assert x.ndim == len(bonds) + 1, (i, j, x.shape)
        phys = f"k{i},{j}"
        out.append((x, tuple(f"K{a}{b},{c}" for a, b, c in bonds) + (phys,), (i, j), "KET"))
        out.append((x.conj(), tuple(f"B{a}{b},{c}" for a, b, c in bonds) + (phys,), (i, j),
                    "BRA"))
    return out, Lx, Ly
