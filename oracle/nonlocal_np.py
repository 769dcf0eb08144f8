"""numpy restatement of quimb_b200/nonlocal_gates.py: ``MatrixProductOperator.
from_dense``, ``gate_with_submpo`` / ``gate_nonlocal`` with the 'direct',
'dm' and 'zipup' compressions of a sub-range of the chain, the controlled
MPO of ``Gate.build_mpo`` and the 'auto-mps' / 'nonlocal' circuit driver, for
(l, p, r) site lists and (l, r, u, d) MPO sites.

Gap sites (inside the span, without an MPO tensor) carry the reference's
identity string: a dense delta[w, v] delta[o, p] tensor for 'direct' and
'dm', and the two-index identity node of enforce_1d_like for the zip-up
gauge, whose spanning tree is ``quimb_b200.mpo_compress.ladder_tree_span``
(host control logic, checked against the reference's get_tree_span by
oracle/make_golden_nonlocal.py).
"""

import numpy as np

from oracle import decomp_np as dnp
from oracle import mpo_compress_np as mnp
from oracle import tebd_np as tnp
from quimb_b200.mpo_compress import ladder_tree_span

_MODE = {"direct": "rsum2", "dm": "rsum1", "zipup": "rsum2"}


# ---------------------------------------------------------------- from_dense ---
def from_dense(G, dims=2, sites=None, cutoff=1e-10, cutoff_mode="rsum2", max_bond=None):
    G = np.asarray(G)
    if isinstance(dims, (int, np.integer)):
        ng = int(round(np.log(G.size) / np.log(dims) / 2))
        dims = (int(dims),) * ng
    dims = tuple(dims)
    ng = len(dims)
    sites = tuple(range(ng)) if sites is None else tuple(sites)
    order = sorted(range(ng), key=lambda k: sites[k])
    T = G.reshape(*dims, *dims)
    inds = [("u", k) for k in range(ng)] + [("d", k) for k in range(ng)]
    opts = dnp.parse_truncation_opts(max_bond, cutoff, cutoff_mode, None)
    out = []
    for n, k in enumerate(order[:-1]):
        rest = order[n + 1:]
        right = [("u", j) for j in rest] + [("d", j) for j in rest]
        left = [ix for ix in inds if ix not in right]
        perm = [inds.index(ix) for ix in left + right]
        Tp = np.transpose(T, perm)
        ls = Tp.shape[:len(left)]
        rs = Tp.shape[len(left):]
        lt, _, rt = dnp.svd_truncated(Tp.reshape(int(np.prod(ls)), -1),
                                      absorb=dnp.get_U_sVH, **opts)
        lt = lt.reshape(*ls, -1)
        T = rt.reshape(-1, *rs)
        inds = [("b", n)] + right
        w = lt[None] if n == 0 else lt                   # (b', u, d, b)
        out.append(np.ascontiguousarray(w.transpose(0, 3, 1, 2)))
    w = T.reshape(1, 1, *T.shape) if ng == 1 else T[:, None]
    out.append(np.ascontiguousarray(w))
    return out, sorted(sites)


def controlled_mpo(G, qubits, controls, dims=None):
    """Gate.build_mpo with controls: (G - 1) on the targets, |1><1| on the
    controls (bonds carried past), plus the identity, by direct sum."""
    qubits, controls = list(qubits), list(controls)
    if dims is None:
        dims = (2,) * len(qubits)
    size = int(np.prod(dims))
    Gm = np.asarray(G).reshape(size, size)
    tmpo, tsites = from_dense(Gm - np.eye(size), dims, qubits)
    dt = tmpo[0].dtype
    p1 = np.diag([0.0, 1.0]).astype(dt)
    allsites = sorted(qubits + controls)
    out, k = [], 0
    for m, s in enumerate(allsites):
        if s in tsites:
            w = tmpo[k]
            k += 1
        else:
            D = tmpo[k - 1].shape[1] if 0 < k < len(tsites) else 1
            w = np.eye(D, dtype=dt)[:, :, None, None] * p1
        d = w.shape[2]
        ident = np.eye(d, dtype=dt).reshape(1, 1, d, d)
        (l1, r1), (l2, r2) = w.shape[:2], ident.shape[:2]
        if m == 0:
            z = np.concatenate([w, ident], axis=1)
        elif m == len(allsites) - 1:
            z = np.concatenate([w, ident], axis=0)
        else:
            z = np.zeros((l1 + l2, r1 + r2, d, d), dtype=dt)
            z[:l1, :r1] = w
            z[l1:, r1:] = ident
        out.append(z)
    return out, allsites


# ------------------------------------------------------------- the sub-ladder ---
def _seed(A):
    r = A[-1].shape[2]
    return np.eye(r, dtype=A[0].dtype).reshape(r, 1, r)


def _dense_gap(D, d, dt):
    """delta[w, v] delta[o, p] as an (l, r, o, p) MPO site."""
    return np.einsum("wv,op->wvop", np.eye(D, dtype=dt), np.eye(d, dtype=dt))


def _flip_w(w):
    return w.T if w.ndim == 2 else w.transpose(1, 0, 2, 3)


def direct(A, W, opts, canonize=True):
    return mnp.direct(A, W, opts, canonize)


def dm(A, W, opts):
    """mpo_compress_np.dm with the open end bonds: the first environment
    traces over (l, o), the right environment starts from delta."""
    L = len(A)
    envs = [None] * L
    E = None
    for i in range(L - 1):
        if E is None:
            T = mnp._product(A[0], W[0]).reshape(-1, A[0].shape[2], W[0].shape[1])
            E = np.einsum("obv,oBV->bvBV", T, T.conj(), optimize=True)
        else:
            X = np.einsum("awAW,apb->wAWpb", E, A[i], optimize=True)
            X = np.einsum("wAWpb,wvop->AWbvo", X, W[i], optimize=True)
            X = np.einsum("AWbvo,WVoP->AbvPV", X, W[i].conj(), optimize=True)
            E = np.einsum("AbvPV,APB->bvBV", X, A[i].conj(), optimize=True)
        envs[i + 1] = E
    out = [None] * L
    R = _seed(A)
    for i in range(L - 1, -1, -1):
        Y = np.einsum("apb,bvk,wvop->awok", A[i], R, W[i], optimize=True)
        la, lw, o, k = Y.shape
        if i == 0:
            out[0] = Y.reshape(la * lw, o, k)
            break
        Z = np.einsum("awAW,awok->AWok", envs[i], Y, optimize=True)
        rho = np.einsum("AWok,AWOK->okOK", Z, Y.conj(), optimize=True).reshape(o * k, o * k)
        U, _, _ = mnp._split(rho, method="eigh", **opts)
        U = U.reshape(o, k, -1)
        out[i] = U.transpose(2, 0, 1)
        R = np.einsum("awok,okn->awn", Y, U.conj(), optimize=True)
    return out


def _inds(L, n, W):
    i = n % L
    if n < L:
        return (("a", i - 1), ("p", i), ("a", i))
    if W[i].ndim == 2:
        return (("w", i - 1), ("w", i))
    return (("w", i - 1), ("w", i), ("o", i), ("p", i))


def zipup(A, W, gaps, opts, open_ends, rev=False, canonize=True):
    """``W[i]`` for a gap site i is the (D, D) identity; after the gauge a
    general matrix."""
    L = len(A)
    A, W = list(A), list(W)
    if canonize:
        T = A + W
        seq = ladder_tree_span(L, [a.shape[2] for a in A[:-1]], [w.shape[1] for w in W[:-1]],
                               [a.shape[1] for a in A], 0 if rev else L - 1, gaps=gaps,
                               open_ends=open_ends, rung_between=True)
        for n1, n2 in seq:
            T[n1], T[n2] = dnp.tensor_canonize_bond(T[n1], _inds(L, n1, W), T[n2],
                                                    _inds(L, n2, W))
        A, W = T[:L], T[L:]
    if rev:
        A = [a.transpose(2, 1, 0) for a in reversed(A)]
        W = [_flip_w(w) for w in reversed(W)]
    ts = [None] * L
    Us = _seed(A)
    for i in range(L - 1, -1, -1):
        if W[i].ndim == 2:
            C = np.einsum("bvk,apb,wv->awpk", Us, A[i], W[i], optimize=True)
        else:
            C = np.einsum("bvk,apb,wvop->awok", Us, A[i], W[i], optimize=True)
        la, lw, o, k = C.shape
        if i == 0:
            ts[0] = C.reshape(la * lw, o, k)
            break
        left, _, right = mnp._split(C.reshape(la * lw, o * k), **opts)
        ts[i] = right.reshape(-1, o, k)
        Us = left.reshape(la, lw, -1)
    return mnp._flip_mps(ts) if rev else ts


def canonicalize(sites, si, sf):
    """Left-canonical left of si, right-canonical right of sf (from scratch)."""
    s = [np.array(a) for a in sites]
    for i in range(si):
        tnp.left_canonize_site(s, i)
    for i in range(len(s) - 1, sf, -1):
        tnp.right_canonize_site(s, i)
    return s


def gate_with_submpo(sites, mpo, where, method="direct", max_bond=None, cutoff=1e-10,
                     cutoff_mode=None, transpose=False, normalize=False, sweep_reverse=False,
                     canonize=True):
    """Returns (new sites, centre)."""
    present = sorted(where)
    si, sf = present[0], present[-1]
    L = len(sites)
    s = canonicalize(sites, si, sf)
    A = s[si:sf + 1]
    Wp = [np.asarray(w) for w in mpo]
    if transpose:
        Wp = [w.transpose(0, 1, 3, 2) for w in Wp]
    dt = np.result_type(*A, *Wp)
    A = [a.astype(dt) for a in A]
    W, gaps, k = [], [], 0
    for i, site in enumerate(range(si, sf + 1)):
        if site == present[k]:
            W.append(Wp[k].astype(dt))
            k += 1
        else:
            D = Wp[k - 1].shape[1]
            gaps.append(i)
            W.append(np.eye(D, dtype=dt) if method == "zipup"
                     else _dense_gap(D, A[i].shape[1], dt))
    opts = dict(max_bond=max_bond, cutoff=cutoff, cutoff_mode=cutoff_mode or _MODE[method])
    if method == "zipup":
        out = zipup(A, W, gaps, opts, (si > 0, sf < L - 1), rev=sweep_reverse,
                    canonize=canonize)
    else:
        if sweep_reverse:
            A, W = mnp._flip(A, W)
        out = direct(A, W, opts, canonize) if method == "direct" else dm(A, W, opts)
        if sweep_reverse:
            out = mnp._flip_mps(out)
    c = sf if sweep_reverse else si
    if normalize:
        out[c - si] = out[c - si] / np.linalg.norm(out[c - si])
    s[si:sf + 1] = [np.ascontiguousarray(x) for x in out]
    return s, c


def gate_nonlocal(sites, G, where, dims=None, **kw):
    if dims is None:
        dims = tuple(sites[i].shape[1] for i in where)
    mpo, _ = from_dense(G, dims, where)
    return gate_with_submpo(sites, mpo, where, **kw)


def gate_controlled(sites, G, qubits, controls, **kw):
    dims = tuple(sites[i].shape[1] for i in qubits)
    mpo, allsites = controlled_mpo(G, qubits, controls, dims)
    return gate_with_submpo(sites, mpo, allsites, **kw)


# ------------------------------------------------------------ circuit driver ---
def apply_circuit(sites, gates, contract="auto-mps", **opts):
    """CircuitMPS with gate_contract 'auto-mps' or 'nonlocal': gate entries
    ``(G, where)`` or ``(G, where, controls)``."""
    s = [np.array(a) for a in sites]
    opts.setdefault("cutoff", 1e-10)
    swap_opts = {k: v for k, v in opts.items() if k in ("max_bond", "cutoff", "cutoff_mode")}
    for g in gates:
        G, where = g[0], tuple(g[1])
        controls = tuple(g[2]) if len(g) > 2 else ()
        if controls:
            s, _ = gate_controlled(s, G, list(where), list(controls), **opts)
        elif len(where) == 1:
            i = where[0]
            s[i] = np.einsum("apb,op->aob", s[i], np.asarray(G))
        elif len(where) == 2 and contract == "auto-mps":
            tnp.gate_with_auto_swap(s, np.asarray(G), where, **swap_opts)
        else:
            s, _ = gate_nonlocal(s, G, where, **opts)
    return s
