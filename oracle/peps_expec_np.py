"""ORACLE (test infrastructure, never imported by the product package).

numpy restatement of PEPS local expectations from plaquette environments,
``PEPS.compute_local_expectation`` with ``mode='mps'`` and
``PEPS.normalize`` (quimb/tensor/tn2d/core.py:4223-4415), on top of
oracle/boundary_np.py:

  compute_environments                  :2716-2835
  _compute_plaquette_environments_x/y_first,
  compute_plaquette_environments        :3075-3431
  calc_plaquette_sizes, plaquette_to_sites,
  calc_plaquette_map                    :5447-5600

Each term is evaluated as the reference does it: the gate is inserted on the
ket layer and the whole plaquette network ``ket.gate(G) | bra | env`` is
contracted, once per term (and once more, ungated, for the local norm).
Every factorisation of every sweep is recorded in the trace of
oracle/boundary_np.py, with the relative singular-value gap at each cut.
"""

import functools
import itertools
import numbers

import numpy as np

from oracle import boundary_np as bnp
from oracle import contract_np as cnp

LAYERS = ("KET", "BRA")


# ------------------------------------------------------------ bookkeeping ---
def is_lone_coo(where):
    return len(where) == 2 and isinstance(where[0], numbers.Integral)


def calc_plaquette_sizes(coo_groups, autogroup=True):
    bszs = set()
    for coos in coo_groups:
        if is_lone_coo(coos):
            bszs.add((1, 1))
            continue
        xs, ys = zip(*coos)
        bszs.add((max(xs) - min(xs) + 1, max(ys) - min(ys) + 1))
    bszs = tuple(sorted(b for b in bszs
                        if not any(b[0] <= c[0] and b[1] <= c[1] for c in bszs - {b})))
    return bszs if autogroup else (tuple(map(max, zip(*bszs))),)


def plaquette_to_sites(p):
    (i0, j0), (di, dj) = p
    return tuple((i, j) for i in range(i0, i0 + di) for j in range(j0, j0 + dj))


def calc_plaquette_map(plaquettes):
    mapping = {}
    for p in sorted(plaquettes, key=lambda p: (-p[1][0] * p[1][1], p)):
        sites = plaquette_to_sites(p)
        for s in sites:
            mapping[s] = p
        for a, b in itertools.combinations(sites, 2):
            mapping[a, b] = p
    return mapping


# ----------------------------------------------------------- environments ---
def _clone(t):
    c = bnp.T(t.data, t.inds, t.layer)
    c.left_inds = t.left_inds
    return c


def _copy(bc, sites=None):
    new = bnp.Boundary2D([], bc.Lx, bc.Ly)
    new.trace = bc.trace
    src = bc.sites if sites is None else sites
    for c, ts in src.items():
        new.sites[c] = [_clone(t) for t in ts]
    return new


def compute_environments(bc, from_which, xrange=None, yrange=None, max_bond=None,
                         cutoff=1e-10, canonize=True, layer_tags=None, dense=False):
    """envs[from_which, i] as ``{site: [T, ...]}`` (the tensors carrying the
    first line's tag, on the coordinates they were contracted onto)."""
    xrange = (0, bc.Lx - 1) if xrange is None else tuple(xrange)
    yrange = (0, bc.Ly - 1) if yrange is None else tuple(yrange)
    tn = _copy(bc)
    plane = from_which[0]
    irange, jrange = (xrange, yrange) if plane == "x" else (yrange, xrange)
    lo, hi = sorted(irange)
    step = 1 if from_which.endswith("min") else -1
    sweep = list(range(lo, hi + 1)) if step > 0 else list(range(hi, lo - 1, -1))
    n_other = bc.Ly if plane == "x" else bc.Lx

    def coo(i, j):
        return (i, j) if plane == "x" else (j, i)

    def line(i):
        return [coo(i, j) for j in range(n_other)]

    def dense_merge(*lines):
        ts = [t for i in lines for c in line(i) for t in tn.sites[c]]
        for i in lines:
            for c in line(i):
                tn.sites[c] = []
        tn.sites[coo(lines[-1], min(jrange))] = [bnp.contract(ts)]

    def snap(i):
        return {c: [_clone(t) for t in tn.sites[c]] for c in line(i) if tn.sites[c]}

    envs = {(from_which, sweep[0]): {}}
    if len(sweep) < 2:
        return envs
    if dense:
        dense_merge(sweep[0])
    envs[from_which, sweep[1]] = snap(sweep[0])
    for i in sweep[2:]:
        i2, i1 = i - 2 * step, i - step
        if dense:
            dense_merge(i2, i1)
        else:
            xr = (i2, i1) if plane == "x" else xrange
            yr = (i2, i1) if plane == "y" else yrange
            tn.contract_boundary_from(xr, yr, from_which, max_bond, cutoff=cutoff,
                                      canonize=canonize, layer_tags=layer_tags)
        envs[from_which, i] = snap(i1)
    return envs


def compute_plaquette_environments(bc, x_bsz, y_bsz, max_bond=None, cutoff=1e-10,
                                   canonize=True, layer_tags=LAYERS, first_contract=None,
                                   second_dense=None):
    if first_contract is None:
        if x_bsz > y_bsz:
            first_contract = "y"
        elif y_bsz > x_bsz:
            first_contract = "x"
        else:
            first_contract = "x" if bc.Lx >= bc.Ly else "y"
    opts = dict(max_bond=max_bond, cutoff=cutoff, canonize=canonize, layer_tags=layer_tags)
    Lx, Ly = bc.Lx, bc.Ly
    valid = set(bc.sites)

    def sel(env, coos):
        return [t for c in coos if c in valid and c in env for t in env[c]]

    out = {}
    if first_contract == "x":
        if second_dense is None:
            second_dense = x_bsz < 2
        xe = {}
        for side in ("xmin", "xmax"):
            xe.update(compute_environments(bc, side, **opts))
        ye = {}
        for i in range(Lx - x_bsz + 1):
            sites = {c: [] for c in bc.sites}
            for env in (xe["xmin", i], xe["xmax", i + x_bsz - 1]):
                for c, ts in env.items():
                    sites[c] += ts
            for c, ts in bc.sites.items():
                if i <= c[0] < i + x_bsz:
                    sites[c] += ts
            row = _copy(bc, sites)
            xr = (max(i - 1, 0), min(i + x_bsz, Lx - 1))
            ye[i] = {}
            for side in ("ymin", "ymax"):
                ye[i].update(compute_environments(row, side, xrange=xr, dense=second_dense,
                                                  **opts))
        for i0, j0 in itertools.product(range(Lx - x_bsz + 1), range(Ly - y_bsz + 1)):
            env = (sel(ye[i0]["ymin", j0], [(i0 + x, j0 - 1) for x in range(-1, x_bsz + 1)])
                   + sel(ye[i0]["ymax", j0 + y_bsz - 1],
                         [(i0 + x, j0 + y_bsz) for x in range(-1, x_bsz + 1)])
                   + sel(xe["xmin", i0], [(i0 - 1, j0 + y) for y in range(y_bsz)])
                   + sel(xe["xmax", i0 + x_bsz - 1], [(i0 + x_bsz, j0 + y) for y in range(y_bsz)]))
            out[(i0, j0), (x_bsz, y_bsz)] = env
    else:
        if second_dense is None:
            second_dense = y_bsz < 2
        ye = {}
        for side in ("ymin", "ymax"):
            ye.update(compute_environments(bc, side, **opts))
        xe = {}
        for j in range(Ly - y_bsz + 1):
            sites = {c: [] for c in bc.sites}
            for env in (ye["ymin", j], ye["ymax", j + y_bsz - 1]):
                for c, ts in env.items():
                    sites[c] += ts
            for c, ts in bc.sites.items():
                if j <= c[1] < j + y_bsz:
                    sites[c] += ts
            col = _copy(bc, sites)
            yr = (max(j - 1, 0), min(j + y_bsz, Ly - 1))
            xe[j] = {}
            for side in ("xmin", "xmax"):
                xe[j].update(compute_environments(col, side, yrange=yr, dense=second_dense,
                                                  **opts))
        for i0, j0 in itertools.product(range(Lx - x_bsz + 1), range(Ly - y_bsz + 1)):
            env = (sel(ye["ymin", j0], [(i0 + x, j0 - 1) for x in range(x_bsz)])
                   + sel(ye["ymax", j0 + y_bsz - 1], [(i0 + x, j0 + y_bsz) for x in range(x_bsz)])
                   + sel(xe[j0]["xmin", i0], [(i0 - 1, j0 + y) for y in range(-1, y_bsz + 1)])
                   + sel(xe[j0]["xmax", i0 + x_bsz - 1],
                         [(i0 + x_bsz, j0 + y) for y in range(-1, y_bsz + 1)]))
            out[(i0, j0), (x_bsz, y_bsz)] = env
    return out


# ------------------------------------------------------------ expectations ---
def _widen(x):
    x = np.asarray(x)
    if x.dtype == np.float32:
        return x.astype(np.float64)
    if x.dtype == np.complex64:
        return x.astype(np.complex128)
    return x


def compute_local_expectation(arrays, terms, max_bond=None, cutoff=1e-10, canonize=True,
                              normalized=False, autogroup=True, return_all=False,
                              first_contract=None, second_dense=None, widen=True,
                              per_term=True):
    """(value, trace): the value as the reference returns it (a scalar, or
    ``where -> (expec, norm or None)``) and the factorisation trace.  With
    ``per_term=False`` each plaquette's two-layer network is contracted once
    with open physical indices and every term is read from that density
    matrix (the same value in exact arithmetic, for large lattices)."""
    arrays = [[_widen(a) if widen else np.asarray(a) for a in row] for row in arrays]
    tensors, Lx, Ly = bnp.peps_norm_tensors(arrays)
    bc = bnp.Boundary2D(tensors, Lx, Ly)
    envs = {}
    for x_bsz, y_bsz in calc_plaquette_sizes(terms.keys(), autogroup):
        envs.update(compute_plaquette_environments(
            bc, x_bsz, y_bsz, max_bond, cutoff, canonize, LAYERS, first_contract, second_dense))
    pmap = calc_plaquette_map(envs)
    groups = {}
    for where, G in terms.items():
        groups.setdefault(pmap[where], []).append((where, np.asarray(G)))
    ket = {coo: (x, inds) for x, inds, coo, layer in tensors if layer == "KET"}
    bra = {coo: (x, inds) for x, inds, coo, layer in tensors if layer == "BRA"}
    expecs = {}
    for p, items in groups.items():
        sites = plaquette_to_sites(p)
        base = [(t.data, t.inds) for t in envs[p]] + [bra[s] for s in sites]

        def close(extra):
            data, _ = cnp.tensor_contract([a for a, _ in extra], [ix for _, ix in extra])
            return complex(np.asarray(data))

        if not per_term:
            kin = [(x, inds[:-1] + ("o" + inds[-1],)) for x, inds in (ket[s] for s in sites)]
            outs = ["o" + ket[s][1][-1] for s in sites] + [ket[s][1][-1] for s in sites]
            # ket block, then the environment around the ring, then the
            # explicit bra block
            K, kix = cnp.tensor_contract([a for a, _ in kin], [ix for _, ix in kin])
            B, bix = cnp.tensor_contract(*zip(*[bra[s] for s in sites]))
            envs_p = [(t.data, t.inds) for t in envs[p]]
            X, xix = K, tuple(kix)
            while envs_p:
                # the tensor sharing the most bonds with what is held, ties by
                # the smaller result
                def cost(k):
                    a, ix = envs_p[k]
                    shared = set(ix) & set(xix)
                    rest = np.prod([n for i, n in zip(ix, a.shape) if i not in shared])
                    return (-len(shared), rest)
                k = min(range(len(envs_p)), key=cost)
                a, ix = envs_p.pop(k)
                X, xix = cnp.tensor_contract([X, a], [xix, ix])
                xix = tuple(xix)
            data, _ = cnp.tensor_contract([X, B], [xix, bix], output_inds=outs)
            dims = [ket[s][0].shape[-1] for s in sites]
            rho = np.asarray(data).reshape(int(np.prod(dims)), -1)
            norm = complex(np.trace(rho)) if normalized else None
            for where, G in items:
                tsites = (tuple(where),) if is_lone_coo(where) else tuple(map(tuple, where))
                pos = [sites.index(s) for s in tsites]
                n = len(sites)
                bra_l = [n + k if k in pos else k for k in range(n)]
                tdims = [dims[k] for k in pos]
                e = np.einsum(G.reshape(tdims + tdims), [n + k for k in pos] + pos,
                              rho.reshape(dims + dims), list(range(n)) + bra_l, [])
                expecs[where] = (complex(e), norm)
            continue
        norm = close([ket[s] for s in sites] + base) if normalized else None
        for where, G in items:
            tsites = (tuple(where),) if is_lone_coo(where) else tuple(map(tuple, where))
            dims = [ket[s][0].shape[-1] for s in tsites]
            g = G.reshape(dims + dims)
            gated, outs, ins = [], [], []
            for s in sites:
                x, inds = ket[s]
                if s in tsites:
                    new = f"gate_in{s[0]},{s[1]}"
                    ins.append(new)
                    outs.append(inds[-1])
                    inds = inds[:-1] + (new,)
                gated.append((x, inds))
            order = [tsites.index(s) for s in sites if s in tsites]
            # G's legs in term order: (out_a, out_b, in_a, in_b)
            outs = [outs[order.index(k)] for k in range(len(tsites))]
            ins = [ins[order.index(k)] for k in range(len(tsites))]
            e = close(gated + [(g, tuple(outs + ins))] + base)
            expecs[where] = (e, norm)
    if return_all:
        return expecs, bc.trace
    if normalized:
        return functools.reduce(lambda a, b: a + b, (e / n for e, n in expecs.values())), bc.trace
    return functools.reduce(lambda a, b: a + b, (e for e, _ in expecs.values())), bc.trace


def normalize(arrays, max_bond=None, cutoff=1e-10, canonize=True):
    """PEPS.normalize: (new site arrays, nfact)."""
    tensors, Lx, Ly = bnp.peps_norm_tensors([[_widen(a) for a in row] for row in arrays])
    nfact, _ = bnp.contract_boundary(tensors, Lx, Ly, max_bond, cutoff=cutoff,
                                     canonize=canonize, layer_tags=LAYERS)
    nfact = complex(np.asarray(nfact)) if np.iscomplexobj(nfact) else float(np.asarray(nfact))
    f = nfact ** (-1 / (2 * Lx * Ly))
    out = [[(np.asarray(a) * (f if np.iscomplexobj(a) else np.real(f))).astype(np.asarray(a).dtype)
            for a in row] for row in arrays]
    return out, nfact


def min_gap(trace):
    return min((r["gap"] for r in trace), default=np.inf)


# -------------------------------------------------------------- the models ---
def spin(name):
    return {"X": np.array([[0, 1], [1, 0]], dtype=complex) / 2,
            "Y": np.array([[0, -1j], [1j, 0]]) / 2,
            "Z": np.array([[1, 0], [0, -1]], dtype=complex) / 2}[name]


def heis2(d=2):
    """The two-site Heisenberg term S.S for spin (d - 1) / 2."""
    if d == 2:
        ops = [spin(c) for c in "XYZ"]
    else:
        s = (d - 1) / 2
        m = np.arange(s, -s - 1, -1)
        sp = np.diag(np.sqrt(s * (s + 1) - m[1:] * (m[1:] + 1)), 1)
        ops = [(sp + sp.T) / 2, (sp - sp.T) / 2j, np.diag(m)]
    h = sum(np.kron(o, o) for o in ops)
    return np.real_if_close(h)


def heis_terms(Lx, Ly, d=2, field=0.0, nnn=0.0, long=0.0, seed=None):
    """Heisenberg bonds, a Z field on every site, both diagonals of each
    plaquette (``nnn``) and 1 x 3 / 3 x 1 terms (``long``); a seeded
    perturbation makes every term distinct."""
    rng = np.random.default_rng(seed)
    h = heis2(d)

    def jitter(x):
        if seed is None:
            return x
        return x * (1 + 0.1 * rng.standard_normal())

    terms = {}
    for i, j in itertools.product(range(Lx), range(Ly)):
        if j + 1 < Ly:
            terms[(i, j), (i, j + 1)] = jitter(h)
        if i + 1 < Lx:
            terms[(i, j), (i + 1, j)] = jitter(h)
        if nnn and i + 1 < Lx and j + 1 < Ly:
            terms[(i, j), (i + 1, j + 1)] = jitter(nnn * h)
            terms[(i, j + 1), (i + 1, j)] = jitter(nnn * h)
        if long and j + 2 < Ly:
            terms[(i, j), (i, j + 2)] = jitter(long * h)
        if long and i + 2 < Lx:
            terms[(i, j), (i + 2, j)] = jitter(long * h)
    if field:
        z = np.diag(np.linspace((d - 1) / 2, -(d - 1) / 2, d))
        for i, j in itertools.product(range(Lx), range(Ly)):
            terms[i, j] = jitter(field * z)
    return terms


def rand_peps(Lx, Ly, D, d, seed, dtype):
    """A PEPS grid in the (up, right, down, left, phys) site convention."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(Lx):
        row = []
        for j in range(Ly):
            nb = (i < Lx - 1) + (j < Ly - 1) + (i > 0) + (j > 0)
            x = rng.standard_normal((D,) * nb + (d,))
            if np.dtype(dtype).kind == "c":
                x = x + 1j * rng.standard_normal(x.shape)
            row.append(x.astype(dtype))
        out.append(row)
    return out


def to_dense(arrays):
    """The state vector of a small PEPS (phys indices in row-major order)."""
    tensors, Lx, Ly = bnp.peps_norm_tensors(arrays)
    kets = [(x, inds) for x, inds, _, layer in tensors if layer == "KET"]
    phys = [inds[-1] for _, inds in kets]
    data, _ = cnp.tensor_contract([x for x, _ in kets], [ix for _, ix in kets],
                                  output_inds=phys)
    return np.asarray(data).reshape(-1)


def dense_expectation(arrays, terms, normalized=False):
    """Exact sum of <G> over the terms from the dense state."""
    Lx, Ly = len(arrays), len(arrays[0])
    psi = to_dense(arrays)
    dims = [np.asarray(arrays[i][j]).shape[-1] for i in range(Lx) for j in range(Ly)]
    psi_t = psi.reshape(dims)
    nrm = np.vdot(psi, psi)
    tot = 0.0
    for where, G in terms.items():
        tsites = (tuple(where),) if is_lone_coo(where) else tuple(map(tuple, where))
        ax = [i * Ly + j for i, j in tsites]
        dg = [dims[a] for a in ax]
        g = np.asarray(G).reshape(dg + dg)
        gpsi = np.tensordot(g, psi_t, axes=(list(range(len(ax), 2 * len(ax))), ax))
        gpsi = np.moveaxis(gpsi, list(range(len(ax))), ax)
        tot = tot + np.vdot(psi_t.reshape(-1), gpsi.reshape(-1))
    return tot / nrm if normalized else tot
