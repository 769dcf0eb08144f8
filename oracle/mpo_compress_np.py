"""numpy restatement of MPO-MPS application with compression, the four methods
of quimb_b200/mpo_compress.py ('direct', 'dm', 'zipup', 'zipup-first'), for
(l, p, r) site lists and (l, r, u, d) MPO sites.  Splits are those of
oracle/decomp_np.py; the zip-up gauge uses the spanning tree of
``quimb_b200.mpo_compress.ladder_tree_span`` (host control logic, checked
against the reference's get_tree_span by oracle/make_golden_mpo_compress.py).
"""

import numpy as np

from oracle import decomp_np as dnp
from quimb_b200.mpo_compress import ladder_tree_span

_MODE = {"direct": "rsum2", "dm": "rsum1", "zipup": "rsum2", "zipup-first": "rsum2"}


def _prepare(sites, mpo, transpose):
    A = [np.asarray(a) for a in sites]
    W = [np.asarray(w) for w in mpo]
    if transpose:
        W = [w.transpose(0, 1, 3, 2) for w in W]
    dt = np.result_type(*A, *W)
    return [a.astype(dt) for a in A], [w.astype(dt) for w in W]


def _flip(A, W):
    return ([a.transpose(2, 1, 0) for a in reversed(A)],
            [w.transpose(1, 0, 2, 3) for w in reversed(W)])


def _flip_mps(A):
    return [a.transpose(2, 1, 0) for a in reversed(A)]


def _product(a, w):
    t = np.einsum("apb,wvop->awobv", a, w, optimize=True)
    l, wl, o, r, wr = t.shape
    return t.reshape(l * wl, o, r * wr)


def _split(mat, method="svd", absorb="left", max_bond=None, cutoff=1e-10,
           cutoff_mode="rsum2", renorm=None):
    opts = dnp.parse_truncation_opts(max_bond, cutoff, cutoff_mode, renorm)
    if method == "eigh":
        return dnp.eigh_truncated(mat, absorb=None, positive=1, **opts)
    _, ab = dnp.parse_method_absorb("svd", absorb, True)
    return dnp.svd_truncated(mat, absorb=ab, **opts)


def _left_canonize_site(s, i):
    l, d, r = s[i].shape
    q, _, rr = dnp.qr_stabilized(s[i].reshape(l * d, r))
    s[i] = q.reshape(l, d, -1)
    s[i + 1] = np.tensordot(rr, s[i + 1], axes=(1, 0))


def _direct_sweep(s, opts):
    """compress_between(i - 1, i, absorb='left', reduced='right')."""
    for i in range(len(s) - 1, 0, -1):
        l, d, r = s[i].shape
        tc, _, nb = _split(s[i].reshape(l, d * r), **opts)
        s[i] = nb.reshape(-1, d, r)
        s[i - 1] = np.tensordot(s[i - 1], tc, axes=(2, 0))


def direct(A, W, opts, canonize=True):
    out = [_product(A[0], W[0])]
    for i in range(1, len(A)):
        out.append(_product(A[i], W[i]))
        if canonize:
            _left_canonize_site(out, i - 1)
    _direct_sweep(out, opts)
    return out


def _inds(L, n):
    i = n % L
    return (("a", i - 1), ("p", i), ("a", i)) if n < L else \
        (("w", i - 1), ("w", i), ("o", i), ("p", i))


def canonize_around(A, W, root):
    L = len(A)
    T = list(A) + list(W)
    seq = ladder_tree_span(L, [a.shape[2] for a in A[:-1]], [w.shape[1] for w in W[:-1]],
                           [a.shape[1] for a in A], root)
    for n1, n2 in seq:
        T[n1], T[n2] = dnp.tensor_canonize_bond(T[n1], _inds(L, n1), T[n2], _inds(L, n2))
    return T[:L], T[L:]


def zipup(A, W, opts, rev=False, canonize=True):
    L = len(A)
    if canonize:
        A, W = canonize_around(A, W, 0 if rev else L - 1)
    if rev:
        A, W = _flip(A, W)
    ts = [None] * L
    Us = np.ones((1, 1, 1), dtype=A[0].dtype)
    for i in range(L - 1, -1, -1):
        C = np.einsum("bvk,apb,wvop->awok", Us, A[i], W[i], optimize=True)
        la, lw, o, k = C.shape
        if i == 0:
            ts[0] = C.reshape(la * lw, o, k)
            break
        left, _, right = _split(C.reshape(la * lw, o * k), **opts)
        ts[i] = right.reshape(-1, o, k)
        Us = left.reshape(la, lw, -1)
    return _flip_mps(ts) if rev else ts


def dm(A, W, opts, spectra=None):
    """``spectra``: a list that receives every reduced density matrix's
    eigenvalues (descending) and its Frobenius norm."""
    L = len(A)
    envs = [None] * L
    E = None
    for i in range(L - 1):
        if E is None:
            T = _product(A[0], W[0]).reshape(W[0].shape[2], A[0].shape[2], W[0].shape[1])
            E = np.einsum("obv,oBV->bvBV", T, T.conj(), optimize=True)
        else:
            X = np.einsum("awAW,apb->wAWpb", E, A[i], optimize=True)
            X = np.einsum("wAWpb,wvop->AWbvo", X, W[i], optimize=True)
            X = np.einsum("AWbvo,WVoP->AbvPV", X, W[i].conj(), optimize=True)
            E = np.einsum("AbvPV,APB->bvBV", X, A[i].conj(), optimize=True)
        envs[i + 1] = E
    out = [None] * L
    R = np.ones((1, 1, 1), dtype=A[0].dtype)
    for i in range(L - 1, -1, -1):
        Y = np.einsum("apb,bvk->apvk", A[i], R, optimize=True)
        Y = np.einsum("apvk,wvop->awok", Y, W[i], optimize=True)
        la, lw, o, k = Y.shape
        if i == 0:
            out[0] = Y.reshape(la * lw, o, k)
            break
        Z = np.einsum("awAW,awok->AWok", envs[i], Y, optimize=True)
        rho = np.einsum("AWok,AWOK->okOK", Z, Y.conj(), optimize=True)
        rho = rho.reshape(o * k, o * k)
        if spectra is not None:
            spectra.append((np.linalg.eigvalsh(rho)[::-1], np.linalg.norm(rho)))
        U, _, _ = _split(rho, method="eigh", **opts)
        U = U.reshape(o, k, -1)
        out[i] = U.transpose(2, 0, 1)
        R = np.einsum("awok,okn->awn", Y, U.conj(), optimize=True)
    return out


def gate_with_mpo(sites, mpo, method="direct", max_bond=None, cutoff=1e-10, cutoff_mode=None,
                  transpose=False, normalize=False, sweep_reverse=False, canonize=True,
                  max_bond_oversample=None, cutoff_oversample=None, spectra=None):
    """MatrixProductState.gate_with_mpo on host arrays: sites (l, p, r), MPO
    sites (l, r, u, d) with size-1 outer bonds at the ends.  ``spectra``: see
    :func:`dm`."""
    method = "zipup-first" if method == "zipup-oversample" else method
    A, W = _prepare(sites, mpo, transpose)
    L = len(A)
    opts = dict(max_bond=max_bond, cutoff=cutoff, cutoff_mode=cutoff_mode or _MODE[method])
    if method == "zipup-first":
        if max_bond_oversample is None:
            mbo = None if max_bond is None else 2 * max_bond
        elif isinstance(max_bond_oversample, float):
            mbo = round(max_bond * max_bond_oversample)
        else:
            mbo = int(max_bond_oversample)
        if cutoff_oversample is None:
            cutoff_oversample = cutoff / 10 if max_bond is None else cutoff
        out = zipup(A, W, dict(opts, max_bond=mbo, cutoff=cutoff_oversample),
                    rev=not sweep_reverse, canonize=canonize)
        out = _flip_mps(out) if sweep_reverse else out
        _direct_sweep(out, opts)
        out = _flip_mps(out) if sweep_reverse else out
    elif method == "zipup":
        out = zipup(A, W, opts, rev=sweep_reverse, canonize=canonize)
    else:
        if sweep_reverse:
            A, W = _flip(A, W)
        out = direct(A, W, opts, canonize) if method == "direct" else dm(A, W, opts, spectra)
        if sweep_reverse:
            out = _flip_mps(out)
    if normalize:
        c = L - 1 if sweep_reverse else 0
        out[c] = out[c] / np.linalg.norm(out[c])
    return [np.ascontiguousarray(x) for x in out]


# ---------------------------------------------------- gauge-invariant views ---
def dense(sites):
    """The state vector of an (l, p, r) site list."""
    v = np.ones((1, 1))
    for a in sites:
        l, d, r = a.shape
        v = (v @ a.reshape(l, d * r)).reshape(-1, r)
    return v.reshape(-1)


def schmidt_values(sites):
    """Singular values of every bond (i, i + 1), from a left-canonicalised
    copy swept back with SVDs."""
    s = [np.array(a, dtype=np.result_type(a.dtype, np.float64)) for a in sites]
    for i in range(len(s) - 1):
        _left_canonize_site(s, i)
    out = [None] * (len(s) - 1)
    for i in range(len(s) - 1, 0, -1):
        l, d, r = s[i].shape
        U, S, VH = np.linalg.svd(s[i].reshape(l, d * r), full_matrices=False)
        s[i] = VH.reshape(-1, d, r)
        s[i - 1] = np.tensordot(s[i - 1], U * S, axes=(2, 0))
        out[i - 1] = S
    return out
