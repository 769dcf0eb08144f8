"""Local expectations and normalisation of a PEPS on the device, from
boundary-contracted plaquette environments: the array-level mirror of

  calc_plaquette_sizes, plaquette_to_sites,
  calc_plaquette_map                     quimb/tensor/tn2d/core.py:5447-5600
  compute_plaquette_environments         :3075-3431 (boundary.py)
  PEPS.compute_local_expectation         :4223-4356
  PEPS.normalize                         :4358-4415

Site arrays follow ``boundary.peps_norm_tensors`` (up, right, down, left,
phys over the bonds present).  The environments are the reference's
operations in the reference's order.  The per-term contraction is not: the
reference contracts ``ket.gate(G) | bra | env`` once per term; here each
plaquette's reduced density matrix is formed once,

  K[e, n]  = the plaquette's ket sites contracted (e: external ket bonds)
  T[e', m] = env . K                 (e': the same bonds on the bra layer)
  rho[m, n] = sum_e T[e, m] conj(K[e, n])        one qb_rdm_reduce, K read
                                                 in place: the bra half of
                                                 the plaquette is never formed

and every term of the call is then evaluated by one ``qb_plaquette_expec``
launch (csrc/plaquette.cu): Tr[G rho] with the other plaquette sites traced,
equal to the reference's gated contraction in exact arithmetic.  The only
host reads are the kept ranks of the truncated SVDs and the 2 n_terms values.
"""

import ctypes
import functools
import itertools
import numbers

import numpy as np
import torch

from . import _lib, ops
from .array import Array
from .boundary import BoundaryContractor2D, contract_boundary, peps_norm_tensors
from .contract import _WIDE, convert
from .observables import RDM_MAX_DIM, rdm_reduce
from .tree import find_tree, tensor_contract

LAYER_TAGS = ("KET", "BRA")
MAX_SITES = 6


# ---------------------------------------------------- plaquette bookkeeping ---
def _is_lone_coo(where):
    return len(where) == 2 and isinstance(where[0], numbers.Integral)


def calc_plaquette_sizes(coo_groups, autogroup=True):
    """The block sizes ``((x_bsz, y_bsz), ...)`` whose plaquettes cover every
    term: the bounding box of each term, minus those another contains, or with
    ``autogroup=False`` the one block covering them all."""
    bszs = set()
    for coos in coo_groups:
        if _is_lone_coo(coos):
            bszs.add((1, 1))
            continue
        xs, ys = zip(*coos)
        bszs.add((max(xs) - min(xs) + 1, max(ys) - min(ys) + 1))
    bszs = tuple(sorted(b for b in bszs
                        if not any(b[0] <= b2[0] and b[1] <= b2[1] for b2 in bszs - {b})))
    if autogroup:
        return bszs
    return (tuple(map(max, zip(*bszs))),)


def plaquette_to_sites(p):
    """The sites of plaquette ``((i0, j0), (di, dj))`` in row-major order."""
    (i0, j0), (di, dj) = p
    return tuple((i, j) for i in range(i0, i0 + di) for j in range(j0, j0 + dj))


def calc_plaquette_map(plaquettes):
    """Every site and every pair ``(a, b)`` with ``a`` before ``b`` in
    row-major order mapped to the smallest plaquette holding it."""
    mapping = {}
    for p in sorted(plaquettes, key=lambda p: (-p[1][0] * p[1][1], p)):
        sites = plaquette_to_sites(p)
        for site in sites:
            mapping[site] = p
        for ij_a, ij_b in itertools.combinations(sites, 2):
            mapping[ij_a, ij_b] = p
    return mapping


def _plaquettes(Lx, Ly, sizes):
    return [((i0, j0), (xb, yb)) for xb, yb in sizes
            for i0 in range(Lx - xb + 1) for j0 in range(Ly - yb + 1)]


# ---------------------------------------------------------------- inputs ---
def _widen(a):
    a = ops.asarray(a)
    if a.dtype in (np.float32, np.complex64):
        return Array(convert(ops.materialize(a).t, _WIDE[a.t.dtype]))
    return a


def _host(G):
    if isinstance(G, Array):
        return G.to_numpy()
    if isinstance(G, torch.Tensor):
        return G.detach().cpu().numpy()
    return np.asarray(G)


def _group_terms(terms, plaquette_map, dims):
    """``{plaquette: [(where, G (dg, dg) numpy, positions), ...]}`` in the
    reference's order; every argument error is raised here, before any
    launch."""
    groups = {}
    for where, G in terms.items():
        p = plaquette_map[where]               # KeyError, as the reference's lookup
        sites = plaquette_to_sites(p)
        tsites = (tuple(where),) if _is_lone_coo(where) else tuple(map(tuple, where))
        if any(s not in dims for s in sites):
            raise ValueError(f"plaquette {p} is not a plaquette of this lattice")
        if any(s not in sites for s in tsites):
            raise ValueError(f"term {where} does not lie in its plaquette {p}")
        pos = tuple(sites.index(s) for s in tsites)
        if list(pos) != sorted(set(pos)):
            raise KeyError(where)
        D = int(np.prod([dims[s] for s in sites]))
        if D > RDM_MAX_DIM or len(sites) > MAX_SITES:
            raise NotImplementedError(
                f"plaquette {p} has a physical dimension of {D}: the reduced density "
                f"matrix is limited to {RDM_MAX_DIM}")
        tdims = tuple(dims[s] for s in tsites)
        dg = int(np.prod(tdims))
        G = _host(G)
        if G.shape not in ((dg, dg), tdims + tdims):
            raise ValueError(f"term {where}: operator of shape {G.shape}, expected "
                             f"({dg}, {dg})")
        groups.setdefault(p, []).append((where, G.reshape(dg, dg), pos))
    return groups


# -------------------------------------------------------------- the parts ---
def plaquette_environments(arrays, sizes, max_bond=None, *, cutoff=1e-10, canonize=True,
                           first_contract=None, second_dense=None):
    """The environments of every plaquette of each block size in ``sizes``
    on the norm network of ``arrays`` (compute_local_expectation's
    ``plaquette_envs``, tn2d/core.py:4297-4311)."""
    tensors, Lx, Ly = peps_norm_tensors(arrays)
    bc = BoundaryContractor2D(tensors, Lx, Ly)
    envs = {}
    for x_bsz, y_bsz in sizes:
        envs.update(bc.compute_plaquette_environments(
            x_bsz, y_bsz, max_bond, cutoff=cutoff, canonize=canonize, layer_tags=LAYER_TAGS,
            first_contract=first_contract, second_dense=second_dense))
    return envs


_TREES = {}


def _env_tree(inputs, output, arrays):
    """The contraction tree of one plaquette's env . ket network, found with
    the 'auto-hq' search (random greedy picks trees up to 64x wider here)
    once per network structure: plaquettes of one shape and position class
    share it."""
    table = {}
    key = (tuple(tuple(table.setdefault(ix, len(table)) for ix in t) for t in inputs),
           tuple(table[ix] for ix in output),
           tuple(int(d) for a in arrays for d in a.shape))
    tree = _TREES.get(key)
    if tree is None:
        size = {ix: int(d) for t, a in zip(inputs, arrays) for ix, d in zip(t, a.shape)}
        tree = find_tree(list(inputs), output, size, "auto-hq")
        if len(_TREES) >= 1024:
            _TREES.clear()
        _TREES[key] = tree
    return tree


def plaquette_rhos(arrays, envs, plaquettes):
    """One packed device buffer with the reduced density matrix of every
    plaquette in ``plaquettes`` (rows: ket, columns: bra; each index the
    C-ordered multi-index of ``plaquette_to_sites``), and each one's element
    offset."""
    tensors, _, _ = peps_norm_tensors(arrays)
    kets = {coo: (x, inds) for x, inds, coo, layer in tensors if layer == "KET"}
    dtype = arrays[0][0].t.dtype
    sizes = []
    for p in plaquettes:
        D = int(np.prod([kets[s][0].shape[-1] for s in plaquette_to_sites(p)]))
        sizes.append(D * D)
    offsets = [0] + list(itertools.accumulate(sizes))[:-1]
    buf = torch.empty(max(sum(sizes), 1), dtype=dtype, device=arrays[0][0].t.device)
    for p, off, n in zip(plaquettes, offsets, sizes):
        sites = plaquette_to_sites(p)
        ks = [kets[s] for s in sites]
        count = {}
        for _, inds in ks:
            for ix in inds[:-1]:
                count[ix] = count.get(ix, 0) + 1
        ext = [ix for _, inds in ks for ix in inds[:-1] if count[ix] == 1]
        phys = [inds[-1] for _, inds in ks]
        K, _ = tensor_contract([x for x, _ in ks], [inds for _, inds in ks],
                               output_inds=ext + phys)
        env = envs[p]
        if env:
            # T from the environment and the separate ket sites, not from K:
            # with K as one hub every tree holds D^|ext| chi^2 d^n elements
            # (69 GB for a 2 x 2 plaquette at D = 4, chi = 64, complex128);
            # cutting through the plaquette site by site keeps the widest
            # intermediate near D^6 chi^2 d^2 (1 GB there)
            arrs = [t.data for t in env] + [x for x, _ in ks]
            inputs = [tuple(t.inds) for t in env] + [tuple(inds) for _, inds in ks]
            out = tuple(["B" + ix[1:] for ix in ext] + phys)
            T, _ = tensor_contract(arrs, inputs, output_inds=out,
                                   optimize=_env_tree(inputs, out, arrs))
        else:
            T = K
        D = int(np.prod(K.shape[len(ext):]))
        n1 = int(np.prod(K.shape[:len(ext)]))
        Kt = ops.materialize(K).t.reshape(n1, D, 1)
        Tt = Kt if T is K else ops.materialize(T).t.reshape(n1, D, 1)
        rdm_reduce(Tt, Kt, out=buf[off:off + n].view(D, D))
    return buf, offsets


def plaquette_expec(rho, offsets, items):
    """Run ``qb_plaquette_expec`` over ``items``: one ``(plaquette index,
    plaquette site dims, G (dg, dg), positions)`` per term.  Returns the
    (Tr[G rho], Tr[rho]) pairs as numpy (one H2D copy of the descriptors, one
    launch, one D2H copy).  A complex G on a real rho is evaluated as two
    descriptors, its real and imaginary parts."""
    cplx = rho.dtype.is_complex
    desc, gs, goff, split = [], [], 0, []
    np_dt = np.complex128 if cplx else np.float64
    for k, pdims, G, pos in items:
        parts = [G]
        if not cplx and np.iscomplexobj(G):
            parts = [G.real, G.imag]
        split.append(len(parts))
        for part in parts:
            row = [offsets[k], goff, len(pdims), len(pos), pos[0], pos[-1]]
            row += list(pdims) + [1] * (MAX_SITES - len(pdims))
            desc.append(row)
            g = np.ascontiguousarray(part, dtype=np_dt).ravel()
            gs.append(g)
            goff += g.size
    n = len(desc)
    table = np.ascontiguousarray(desc, dtype=np.int64).reshape(n, _lib.QB_PLAQ_DESC_WORDS)
    dev = rho.device
    G_dev = torch.from_numpy(np.concatenate(gs)).to(dev)
    desc_dev = torch.empty(n * _lib.QB_PLAQ_DESC_WORDS, dtype=torch.int64, device=dev)
    out = torch.empty(2 * n, dtype=rho.dtype, device=dev)
    lib = _lib.load()
    rc = lib.qb_plaquette_expec(
        _lib.qb_dtype(rho.dtype), n, table.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
        desc_dev.data_ptr(), rho.data_ptr(), rho.numel(), G_dev.data_ptr(), G_dev.numel(),
        out.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "qb_plaquette_expec")
    vals = out.cpu().numpy().reshape(n, 2)
    res, r = [], 0
    for s in split:
        e = vals[r, 0] if s == 1 else complex(vals[r, 0], vals[r + 1, 0])
        res.append((e, vals[r, 1]))
        r += s
    return res


def _scalar(x, cplx):
    return complex(x) if cplx else float(np.real(x))


# ------------------------------------------------------------ public API ---
def peps_compute_local_expectation(arrays, terms, max_bond=None, *, cutoff=1e-10,
                                   canonize=True, mode="mps", normalized=False,
                                   autogroup=True, return_all=False, plaquette_envs=None,
                                   plaquette_map=None, first_contract=None, second_dense=None,
                                   equalize_norms=False):
    """``PEPS.compute_local_expectation`` (tn2d/core.py:4223-4356) of the PEPS
    ``arrays[i][j]``: the sum over ``terms`` (``{(i, j) or ((i_a, j_a),
    (i_b, j_b)): G}``) of <G>, each divided by its plaquette's norm with
    ``normalized``; with ``return_all`` the dict ``where -> (expec, norm or
    None)``.  ``plaquette_envs`` may be precomputed with
    :func:`plaquette_environments`.  float32 / complex64 sites are widened
    once on entry; the values are Python scalars."""
    if mode != "mps":
        raise NotImplementedError(f"mode={mode!r}: only the 'mps' boundary is implemented")
    if equalize_norms:
        raise NotImplementedError("equalize_norms is not implemented")
    Lx, Ly = len(arrays), len(arrays[0])
    if any(len(row) != Ly for row in arrays):
        raise ValueError("arrays must be a rectangular grid")
    dims = {(i, j): int(arrays[i][j].shape[-1]) for i in range(Lx) for j in range(Ly)}
    sizes = None
    if plaquette_envs is None:
        sizes = calc_plaquette_sizes(terms.keys(), autogroup)
        plaqs = _plaquettes(Lx, Ly, sizes)
    else:
        plaqs = list(plaquette_envs)
    if plaquette_map is None:
        plaquette_map = calc_plaquette_map(plaqs)
    groups = _group_terms(terms, plaquette_map, dims)
    arrays = [[_widen(a) for a in row] for row in arrays]
    if plaquette_envs is None:
        plaquette_envs = plaquette_environments(
            arrays, sizes, max_bond, cutoff=cutoff, canonize=canonize,
            first_contract=first_contract, second_dense=second_dense)
    used = list(groups)
    rho, offsets = plaquette_rhos(arrays, plaquette_envs, used)
    items, keys = [], []
    for k, p in enumerate(used):
        pdims = [dims[s] for s in plaquette_to_sites(p)]
        for where, G, pos in groups[p]:
            items.append((k, pdims, G, pos))
            keys.append(where)
    vals = plaquette_expec(rho, offsets, items) if items else []
    cplx = rho.dtype.is_complex or any(np.iscomplexobj(G) for _, _, G, _ in items)
    expecs = {where: (_scalar(e, cplx), _scalar(n, cplx) if normalized else None)
              for where, (e, n) in zip(keys, vals)}
    if return_all:
        return expecs
    if normalized:
        return functools.reduce(lambda a, b: a + b, (e / n for e, n in expecs.values()))
    return functools.reduce(lambda a, b: a + b, (e for e, _ in expecs.values()))


def peps_normalize(arrays, max_bond=None, *, cutoff=1e-10, canonize=True):
    """``PEPS.normalize`` (tn2d/core.py:4358-4415): new site arrays, each
    the input times ``nfact ** (-1 / (2 N))`` with ``nfact`` the boundary
    norm <psi|psi> and N the number of sites; dtypes are kept.  A real PEPS
    whose (truncated) boundary norm is not positive raises ``ValueError``:
    no real factor normalises it."""
    tensors, Lx, Ly = peps_norm_tensors(arrays)
    nfact = contract_boundary(tensors, Lx, Ly, max_bond, cutoff=cutoff, canonize=canonize,
                              layer_tags=LAYER_TAGS)
    real = not any(np.dtype(ops.asarray(a).dtype).kind == "c" for row in arrays for a in row)
    if real and not complex(nfact).real > 0:
        # the reference would scale a real PEPS by a complex (or NaN) factor
        raise ValueError(f"the boundary norm of a real PEPS is {nfact}, not positive: "
                         "increase max_bond")
    f = nfact ** (-1 / (2 * Lx * Ly))
    out = []
    for row in arrays:
        new = []
        for a in row:
            y = ops.materialize(ops.asarray(a), force=True)
            ops.scale_(y, f if y.t.dtype.is_complex else float(np.real(f)))
            new.append(y)
        out.append(new)
    return out
