"""numpy restatement of quimb_b200/observables.py (MPS observables of
open-boundary (l, p, r) site lists): numpy QR / SVD for the centre moves and
Schmidt values, explicit einsum for every reduced density matrix.  Site lists
are lists of numpy arrays, modified in place where the device version is."""

import functools
import numbers
import operator

import numpy as np

_einsum = functools.partial(np.einsum, optimize=True)


def _qr_stab(x):
    q, r = np.linalg.qr(x)
    sg = np.where(np.real(np.diag(r)) < 0, -1.0, 1.0)
    return q * sg[None, :], r * sg[:, None]


def left_canonize_site(sites, i):
    l, d, r = sites[i].shape
    q, R = _qr_stab(sites[i].reshape(l * d, r))
    sites[i] = q.reshape(l, d, -1)
    sites[i + 1] = _einsum("ab,bpr->apr", R, sites[i + 1])


def right_canonize_site(sites, i):
    l, d, r = sites[i].shape
    q, R = _qr_stab(sites[i].reshape(l, d * r).T)
    sites[i] = q.T.reshape(-1, d, r)
    sites[i - 1] = _einsum("lpa,ba->lpb", sites[i - 1], R)


def count_canonized(sites):
    L = len(sites)

    def isid(x):
        single = x.dtype in (np.float32, np.complex64)
        rtol, atol = (1e-5, 1e-6) if single else (1e-9, 1e-11)
        return np.allclose(x, np.eye(x.shape[0]), rtol=rtol, atol=atol)

    nl = nr = 0
    E = np.eye(sites[0].shape[0])
    for i in range(L - 1):
        E = _einsum("xa,xpy,apb->yb", E, sites[i].conj(), sites[i])
        if not isid(E):
            break
        nl += 1
    E = np.eye(sites[-1].shape[2])
    for j in reversed(range(nl + 1, L)):
        E = _einsum("xpy,apb,yb->xa", sites[j].conj(), sites[j], E)
        if not isid(E):
            break
        nr += 1
    return nl, nr


def canonicalize(sites, where, info=None):
    w = (where,) if isinstance(where, numbers.Integral) else tuple(where)
    i, j = min(w), max(w)
    info = {} if info is None else info
    info.setdefault("cur_orthog", "calc")
    cur = info["cur_orthog"]
    if isinstance(cur, str):
        lo, ro = count_canonized(sites)
        cur = (lo, len(sites) - ro - 1)
    cmin, cmax = (cur, cur) if isinstance(cur, numbers.Integral) else (min(cur), max(cur))
    if i > cmin:
        for k in range(cmin, i):
            left_canonize_site(sites, k)
    else:
        i = min(j, cmin)
    if j < cmax:
        for k in range(cmax, j, -1):
            right_canonize_site(sites, k)
    else:
        j = max(i, cmax)
    info["cur_orthog"] = (i, j)
    return info


def rho_dense(sites, where, EL=None, ER=None):
    """rho[(p...), (q...)] of ``where`` (in its order) with everything outside
    the span contracted through EL / ER [bra, ket] (identity when None)."""
    w = (where,) if isinstance(where, numbers.Integral) else tuple(where)
    lo, hi = min(w), max(w)
    a = sites[lo].shape[0]
    EL = np.eye(a) if EL is None else EL
    T = EL.T[None, None]                          # T[P, Q, ket bond, bra bond]
    for k in range(lo, hi + 1):
        B = sites[k]
        if k in w:
            T = _einsum("PQax,apb,xqy->PpQqby", T, B, B.conj())
            T = T.reshape(T.shape[0] * T.shape[1], T.shape[2] * T.shape[3], *T.shape[4:])
        else:
            T = _einsum("PQax,asb,xsy->PQby", T, B, B.conj())
    ER = np.eye(T.shape[2]) if ER is None else ER
    rho = _einsum("PQby,yb->PQ", T, ER)
    dims = [sites[k].shape[1] for k in sorted(w)]
    order = [sorted(w).index(x) for x in w]
    n, D = len(w), rho.shape[0]
    return rho.reshape(dims + dims).transpose(order + [n + o for o in order]).reshape(D, D)


def partial_trace_to_dense_canonical(sites, where, normalized=True, info=None):
    canonicalize(sites, where, info)
    rho = rho_dense(sites, where)
    return rho / np.trace(rho) if normalized else rho


def local_expectation_canonical(sites, G, where, normalized=True, info=None):
    rho = partial_trace_to_dense_canonical(sites, where, normalized, info)
    return np.trace(np.asarray(G).reshape(rho.shape) @ rho)


def _w(k):
    return (k,) if isinstance(k, numbers.Integral) else tuple(k)


def compute_local_expectation(sites, terms, normalized=True, return_all=False,
                              method="canonical", info=None, inplace=False):
    if method == "canonical":
        info = {} if info is None else info
        if not inplace:
            sites, info = list(sites), info.copy()
        cur = info.get("cur_orthog", "calc")
        if isinstance(cur, tuple):
            items = sorted(terms.items(), key=lambda kv: abs(min(_w(kv[0])) - cur[0]))
        else:
            items = sorted(terms.items(), key=lambda kv: min(_w(kv[0])))
        ex = {k: local_expectation_canonical(sites, G, _w(k), normalized, info)
              for k, G in items}
    else:
        L = len(sites)
        left, right = {}, {}
        E = np.eye(1)
        for i in range(L - 1):
            E = _einsum("xa,xpy,apb->yb", E, sites[i].conj(), sites[i])
            left[i + 1] = E
        E = np.eye(1)
        for i in range(L - 1, 0, -1):
            E = _einsum("xpy,apb,yb->xa", sites[i].conj(), sites[i], E)
            right[i - 1] = E
        nf = _einsum("xpy,apb,yb->", sites[0].conj(), sites[0], right.get(0, np.eye(1)))
        ex = {}
        for k, G in terms.items():
            w = _w(k)
            rho = rho_dense(sites, w, left.get(min(w)), right.get(max(w)))
            x = np.trace(np.asarray(G).reshape(rho.shape) @ rho)
            ex[k] = x / nf if normalized else x
    return ex if return_all else functools.reduce(operator.add, ex.values())


def singular_values(sites, i, info=None, method="svd"):
    if not 0 < i < len(sites):
        raise ValueError(f"Need 0 < i < {len(sites)}, got i={i}.")
    canonicalize(sites, i, info)
    l, d, r = sites[i].shape
    x = sites[i].reshape(l, d * r)
    if method == "svd":
        return np.linalg.svd(x, compute_uv=False)
    g = x @ x.conj().T if l <= d * r else x.conj().T @ x
    ev = np.linalg.eigvalsh(g)[::-1]
    return np.sqrt(np.clip(ev, 0.0, None))


def schmidt_values(sites, i, info=None, method="svd"):
    return singular_values(sites, i, info, method) ** 2


def entropy(sites, i, info=None, method="svd"):
    S = schmidt_values(sites, i, info, method)
    S = S[S > 0.0]
    return np.sum(-S * np.log2(S))


def schmidt_gap(sites, i, info=None, method="svd"):
    S = schmidt_values(sites, i, info, method)
    return S[0] if len(S) == 1 else S[0] - S[1]


def spin_operator(label, S=0.5):
    D = int(2 * S + 1)
    op = np.zeros((D, D), dtype=complex)
    ms = np.linspace(S, -S, D)
    if label.lower() in "xy":
        for k in range(D - 1):
            c = 0.5 * (S * (S + 1) - ms[k] * ms[k + 1]) ** 0.5
            op[k, k + 1] = -1j * c if label.lower() == "y" else c
            op[k + 1, k] = 1j * c if label.lower() == "y" else c
    else:
        op[np.arange(D), np.arange(D)] = ms
    return np.real_if_close(op)


def magnetization(sites, i, direction="Z", info=None):
    canonicalize(sites, i, info)
    rho = rho_dense(sites, (i,))
    return np.sum(spin_operator(direction, (sites[i].shape[1] - 1) / 2) * rho)


def _overlap(bra, ket):
    E = np.ones((1, 1))
    for A, B in zip(bra, ket):
        E = _einsum("xa,xpy,apb->yb", E, A.conj(), B)
    return E.reshape(())[()]


def correlation(sites, A, i, j, B=None):
    B = A if B is None else B

    def gate(s, G, k):
        s = list(s)
        s[k] = _einsum("qp,lpr->lqr", G, s[k])
        return s

    pA = gate(sites, A, i)
    pB = gate(sites, B, j)
    pAB = gate(pA, B, j)
    return _overlap(sites, pAB) - _overlap(sites, pA) * _overlap(sites, pB)


def _ops(d):
    """Pauli X, Y, Z for d = 2, the spin-1 operators for d = 3."""
    S = (d - 1) / 2
    return {c: spin_operator(c, S) * (2 if d == 2 else 1) for c in "XYZ"}


def terms_for(label, L, d):
    """The term dictionaries of the fixture cases (tests/golden/observables.*),
    by label: 'X' / 'Z' on every site, 'heis' on every bond, 'far' three
    non-adjacent pairs."""
    o = _ops(d)
    if label in ("X", "Y", "Z"):
        return {(i,): o[label] for i in range(L)}
    if label == "heis":
        h = np.real_if_close(sum(np.kron(o[c], o[c]) for c in "XYZ"))
        return {(i, i + 1): h for i in range(L - 1)}
    if label == "far":
        return {(0, 3): np.kron(o["Z"], o["Z"]), (1, 4): np.kron(o["X"], o["Z"]),
                (L - 4, L - 1): np.kron(o["Z"], o["X"])}
    raise KeyError(label)
