"""MPS observables on the device: orthogonality-centre tracking, reduced
density matrices, local expectations, Schmidt values, entanglement entropy,
magnetisation and correlators of open-boundary (l, p, r) site lists.

Mirrors, at array level, quimb's

  count_canonized / calc_current_orthog_center  tn1d/core.py:1571-1626
  canonicalize (tracked centre)                 tn1d/core.py:1096-1189, :351
  singular_values                               tn1d/core.py:1472-1506
  magnetization, schmidt_values, entropy,
  schmidt_gap                                   tn1d/core.py:2605-2725
  partial_trace_to_dense_canonical,
  local_expectation_canonical,
  compute_local_expectation ('canonical' and
  'envs')                                       tn1d/core.py:2827-3165
  correlation                                   tn1d/core.py:699-741

``info["cur_orthog"]`` records the orthogonality centre as the reference
records it, so a sweep over sorted sites moves the centre one site at a time.

Every reduced density matrix ends in one ``qb_rdm_reduce``
(csrc/rdm.cu): rho[m, n] = sum_{a, b} U[a, m, b] conj(V[a, n, b]), a
reduction with a tiny output and a summed extent of chi_l chi_r that the
contraction engine pads to a 32 x 32 tile and splits.  U is formed on the
contraction engine:

  contiguous sites     U = V = theta, the block of the sites (chi, D, chi)
  non-contiguous sites X[P, Q, a, a'] carried over the span (sites in the
                       gaps traced, open sites adding to P and Q), then
                       U = Y[a', (P Q p), b] = sum_a X A, V = A of the last
                       site, and one permute to ((P p), (Q q))
  method='envs'        the same with the left / right norm environments
                       folded into the first / last step

All results are device Arrays; the only value read back is the identity
test of the ``"calc"`` centre.
"""

import ctypes
import functools
import numbers
import operator

import numpy as np
import torch

from . import _lib, ops, tebd
from .array import Array
from .contract import _WIDE, contract_pair, convert
from .mps import compute_left_environments, compute_right_environments, norm_step, \
    norm_step_right
from .split import array_svals

# the widest operand of qb_rdm_reduce: M, N <= 64
RDM_MAX_DIM = 64


# ------------------------------------------------------------- the kernel ---
def rdm_reduce(U, V, out=None):
    """out[m, n] = sum_{a, b} U[a, m, b] conj(V[a, n, b]) through
    ``qb_rdm_reduce``: U (n1, M, n2) and V (n1, N, n2) torch tensors of one
    dtype, any strides; float32 / complex64 are widened, the result is fp64 /
    c128 (M, N), written into ``out`` (a contiguous (M, N) tensor) if given."""
    if U.dtype != V.dtype:
        raise TypeError(f"rdm_reduce: dtype mismatch {U.dtype} vs {V.dtype}")
    if U.dtype in _WIDE:
        alias = U is V
        U = convert(U, _WIDE[U.dtype])
        V = U if alias else convert(V, _WIDE[V.dtype])
    n1, M, n2 = U.shape
    if V.shape[0] != n1 or V.shape[2] != n2:
        raise ValueError(f"rdm_reduce: U {tuple(U.shape)} and V {tuple(V.shape)} differ "
                         "in the summed extents")
    N = V.shape[1]
    lib = _lib.load()
    if out is None:
        out = torch.empty((M, N), dtype=U.dtype, device=U.device)
    elif out.shape != (M, N) or out.dtype != U.dtype or not out.is_contiguous():
        raise ValueError(f"rdm_reduce: out must be a contiguous ({M}, {N}) {U.dtype} tensor")
    need = int(lib.qb_rdm_workspace(n1, M, N, n2))
    if need < 0:
        _lib.check(need, "qb_rdm_workspace")
    ws = torch.empty(need, dtype=torch.uint8, device=U.device) if need else None
    us = (ctypes.c_int64 * 3)(*U.stride())
    vs = (ctypes.c_int64 * 3)(*V.stride())
    rc = lib.qb_rdm_reduce(_lib.qb_dtype(U.dtype), n1, M, N, n2, U.data_ptr(), us,
                           V.data_ptr(), vs, out.data_ptr(),
                           None if ws is None else ws.data_ptr(), need, _lib.stream_ptr())
    _lib.check(rc, "qb_rdm_reduce")
    return out


def _plain(A):
    """The torch tensor of an Array with any lazy conjugation applied."""
    return ops.materialize(A).t if A.cj else A.t


# ----------------------------------------------------------- site handling ---
def _prepare(sites):
    """Device (l, p, r) arrays with open boundaries, converted in place."""
    if not len(sites):
        raise ValueError("empty MPS")
    for k, a in enumerate(sites):
        a = ops.asarray(a)
        if a.ndim != 3:
            raise ValueError("sites must be (l, p, r) arrays")
        if np.dtype(a.dtype).kind not in "fc":
            raise TypeError(f"unsupported dtype {a.dtype}")
        sites[k] = a
    if sites[0].shape[0] != 1 or sites[-1].shape[2] != 1:
        raise ValueError("open boundaries only (first left and last right bond of "
                         "dimension 1)")
    return sites


def _where(where):
    return (int(where),) if isinstance(where, numbers.Integral) else tuple(int(w) for w in where)


# ----------------------------------------------------- orthogonality centre ---
def _is_identity(x):
    """count_canonized's isidentity: allclose to eye with the reference's
    tolerances per dtype (one value read back)."""
    single = x.t.dtype in _WIDE
    rtol, atol = (1e-5, 1e-6) if single else (1e-9, 1e-11)
    eye = ops.eye(x.shape[0], dtype=x.dtype, device=x.device)
    return ops.allclose(x, eye, rtol=rtol, atol=atol)


def mps_count_canonized(sites):
    """``(num_can_l, num_can_r)``: how many sites from the left are left
    isometries and, after those, how many from the right are right isometries
    (count_canonized, tn1d/core.py:1571-1614)."""
    sites = _prepare(sites)
    L = len(sites)
    nl = nr = 0
    E = None
    for i in range(L - 1):
        A = sites[i]
        if E is None:
            E = ops.eye(A.shape[0], dtype=A.dtype, device=A.device)
        E = norm_step(E, A)
        if not _is_identity(E):
            break
        nl += 1
    E = None
    for j in reversed(range(nl + 1, L)):
        A = sites[j]
        if E is None:
            E = ops.eye(A.shape[2], dtype=A.dtype, device=A.device)
        E = norm_step_right(E, A)
        if not _is_identity(E):
            break
        nr += 1
    return nl, nr


def mps_calc_current_orthog_center(sites):
    """``(lo, hi)``: the sites around which the MPS is orthogonal
    (calc_current_orthog_center, tn1d/core.py:1616-1626)."""
    lo, ro = mps_count_canonized(sites)
    return lo, len(sites) - ro - 1


def mps_canonicalize(sites, where, info=None):
    """Move the orthogonality centre to site(s) ``where`` (an int, or the
    range min(where) .. max(where)), in place, starting from
    ``info["cur_orthog"]`` (``"calc"``, a site, or an inclusive (min, max)
    pair; default ``"calc"``) and moving only the sites between it and
    ``where`` (canonicalize, tn1d/core.py:1096-1189).  Records the new range
    in ``info["cur_orthog"]`` and returns ``sites``."""
    sites = _prepare(sites)
    w = _where(where)
    i, j = min(w), max(w)
    if info is None:
        info = {}
    info.setdefault("cur_orthog", "calc")
    cur = info["cur_orthog"]
    if isinstance(cur, str) and cur == "calc":
        cur = mps_calc_current_orthog_center(sites)
    if cur is None:
        tebd.left_canonize(sites, 0, i)
        tebd.right_canonize(sites, len(sites) - 1, j)
    else:
        if isinstance(cur, numbers.Integral):
            cmin = cmax = int(cur)
        else:
            cmin, cmax = min(cur), max(cur)
        if i > cmin:
            for k in range(cmin, i):
                tebd.left_canonize_site(sites, k)
        else:
            i = min(j, cmin)
        if j < cmax:
            for k in range(cmax, j, -1):
                tebd.right_canonize_site(sites, k)
        else:
            j = max(i, cmax)
    info["cur_orthog"] = (i, j)
    return sites


# ------------------------------------------------- reduced density matrices ---
def _cast(x, dt):
    return x if x is None or x.dtype == dt else x.astype(dt)


def _rho(sites, where, EL=None, ER=None):
    """rho[(p...), (q...)] of the sites ``where`` (in that order), with the
    left / right norm environments EL[bra, ket], ER[bra, ket] around the span
    (None: an isometry, i.e. the identity).  Not normalised; the sites' dtype
    widened to fp64 / c128."""
    L = len(sites)
    if len(set(where)) != len(where) or not all(0 <= w < L for w in where):
        raise ValueError(f"invalid sites {where} for an MPS of {L} sites")
    ws = sorted(where)
    span = list(sites[ws[0]:ws[-1] + 1])
    dt = np.result_type(*[x.dtype for x in span + [EL, ER] if x is not None])
    span, EL, ER = ([_cast(x, dt) for x in span], _cast(EL, dt), _cast(ER, dt))
    dims = [sites[w].shape[1] for w in ws]
    D = int(np.prod(dims))
    if ws == list(range(ws[0], ws[-1] + 1)):
        if D > RDM_MAX_DIM:
            raise NotImplementedError(
                f"reduced density matrix of dimension {D}: qb_rdm_reduce takes "
                f"operands up to {RDM_MAX_DIM} wide")
        theta = span[0]
        tt = _plain(theta)
        for B in span[1:]:
            l, p, _ = tt.shape
            tt = contract_pair(tt, [0, 1, 2], B.t, [2, 3, 4], [0, 1, 3, 4], conj_b=B.cj)
            tt = tt.reshape(l, p * B.shape[1], B.shape[2])
        U = tt
        if EL is not None:
            U = contract_pair(EL.t, [5, 0], U, [0, 1, 2], [5, 1, 2], conj_a=EL.cj)
        if ER is not None:
            U = contract_pair(U, [0, 1, 2], ER.t, [6, 2], [0, 1, 6], conj_b=ER.cj)
        rho = rdm_reduce(U, tt)
    else:
        rho = _rho_transfer(span, [w - ws[0] for w in ws], dims, EL, ER)
    rho = Array(rho)
    if list(where) != ws:
        # the reference's index order is that of ``where``
        k = len(ws)
        order = [ws.index(w) for w in where]
        rho = ops.materialize(
            rho.reshape(*(dims + dims)).transpose(*(order + [k + o for o in order])))
        rho = rho.reshape(D, D)
    return rho


def _rho_transfer(span, opened, dims, EL, ER):
    """rho of the non-contiguous open sites ``opened`` (positions in the
    ``span`` of sites) by the transfer form: cost linear in the span."""
    # labels: a ket / a' bra left bond, s physical, b / b' right bonds, P / Q
    # the open physical indices collected so far (ket / bra)
    a, a_, s, b, b_, P, Q, q = range(8)
    DP = int(np.prod(dims[:-1]))
    d_last = dims[-1]
    if DP * DP * d_last > RDM_MAX_DIM:
        raise NotImplementedError(
            f"non-contiguous reduced density matrix: the last step needs a "
            f"{DP * DP * d_last}-wide operand, qb_rdm_reduce takes up to {RDM_MAX_DIM}")
    A = span[0]
    At = _plain(A)
    T = At if EL is None else contract_pair(EL.t, [a_, a], At, [a, s, b], [a_, s, b],
                                            conj_a=EL.cj)
    # X[p, q, b, b'] after the first open site
    X = contract_pair(T, [a_, P, b], At, [a_, Q, b_], [P, Q, b, b_], conj_b=True)
    for k in range(1, len(span) - 1):
        At = _plain(span[k])
        np_, nq = X.shape[0], X.shape[1]
        T = contract_pair(X, [P, Q, a, a_], At, [a, s, b], [P, Q, a_, s, b])
        if k in opened:
            X = contract_pair(T, [P, Q, a_, s, b], At, [a_, q, b_], [P, s, Q, q, b, b_],
                              conj_b=True)
            d = At.shape[1]
            X = X.reshape(np_ * d, nq * d, X.shape[4], X.shape[5])
        else:
            X = contract_pair(T, [P, Q, a_, s, b], At, [a_, s, b_], [P, Q, b, b_],
                              conj_b=True)
    At = _plain(span[-1])
    l, d, r = At.shape
    Y = contract_pair(X, [P, Q, a, a_], At, [a, s, b], [a_, P, Q, s, b])
    if ER is not None:
        Y = contract_pair(Y, [a_, P, Q, s, b], ER.t, [b_, b], [a_, P, Q, s, b_], conj_b=ER.cj)
    Y = Y.reshape(l, DP * DP * d, r)
    rho = rdm_reduce(Y, At)                                 # [(P, Q, p), q]
    rho = rho.reshape(DP, DP, d, d).permute(0, 2, 1, 3)     # [P, p, Q, q]
    return ops.materialize(Array(rho)).t.reshape(DP * d, DP * d)


def mps_partial_trace_to_dense_canonical(sites, where, normalized=True, info=None):
    """Dense reduced density matrix of the site(s) ``where`` (D x D, D the
    product of their physical dimensions, indices in the order of ``where``):
    the centre is moved onto ``where`` in place first and recorded in
    ``info`` (partial_trace_to_dense_canonical, tn1d/core.py:2827-2877).
    ``normalized`` divides by the trace."""
    sites = _prepare(sites)
    w = _where(where)
    mps_canonicalize(sites, w, info=info)
    dt = np.result_type(*[sites[k].dtype for k in range(min(w), max(w) + 1)])
    rho = _rho(sites, w).astype(dt, copy=False)
    if normalized:
        rho = rho / ops.trace(rho)
    return rho


def mps_local_expectation_canonical(sites, G, where, normalized=True, info=None):
    """``trace(G @ rho)`` of the reduced density matrix of ``where``
    (local_expectation_canonical, tn1d/core.py:2879-2911)."""
    rho = mps_partial_trace_to_dense_canonical(sites, where, normalized=normalized, info=info)
    G = ops.asarray(G).reshape(rho.shape)
    return ops.trace(ops.matmul(G, rho))


def _sum(values):
    return functools.reduce(operator.add, values)


def mps_compute_local_expectation(sites, terms, normalized=True, return_all=False,
                                  method="canonical", info=None, inplace=False):
    """Many local expectations at once (compute_local_expectation,
    tn1d/core.py:3089-3165).  ``terms`` maps a site tuple to its operator;
    returns their sum, or with ``return_all`` a dict of 0-d device Arrays.

    ``method='canonical'`` moves the centre from ``info["cur_orthog"]``
    through the terms sorted as the reference sorts them, on a copy of the
    list (and of ``info``) unless ``inplace``.  ``method='envs'`` builds the
    left and right norm environments once and uses no canonical form."""
    if method == "canonical":
        if info is None:
            info = {}
        if inplace:
            psi = sites
        else:
            psi = list(sites)
            info = info.copy()
        _prepare(psi)
        cur = info.get("cur_orthog", "calc")
        if isinstance(cur, tuple):
            items = sorted(terms.items(), key=lambda kv: abs(min(_where(kv[0])) - cur[0]))
        else:
            items = sorted(terms.items(), key=lambda kv: min(_where(kv[0])))
        expecs = {where: mps_local_expectation_canonical(psi, G, _where(where),
                                                         normalized=normalized, info=info)
                  for where, G in items}
    elif method == "envs":
        expecs = _local_expectation_envs(list(sites), terms, normalized)
    else:
        raise ValueError(f"Unrecognized method: {method}, should be one of: "
                         "'canonical', 'envs'.")
    return expecs if return_all else _sum(expecs.values())


def _local_expectation_envs(psi, terms, normalized):
    """compute_local_expectation_via_envs (tn1d/core.py:2998-3087)."""
    psi = _prepare(psi)
    left = compute_left_environments(psi, shape="lpr")
    right = compute_right_environments(psi, shape="lpr")
    nfactor = None
    if normalized:
        A = psi[0]
        E = right[0] if 0 in right else ops.eye(A.shape[2], dtype=A.dtype, device=A.device)
        nfactor = norm_step_right(E, A).reshape(())
    expecs = {}
    for where, G in terms.items():
        w = _where(where)
        lo, hi = min(w), max(w)
        dt = np.result_type(*[psi[k].dtype for k in range(lo, hi + 1)])
        rho = _rho(psi, w, left.get(lo), right.get(hi)).astype(dt, copy=False)
        G = ops.asarray(G).reshape(rho.shape)
        x = ops.trace(ops.matmul(G, rho))
        expecs[where] = x / nfactor if normalized else x
    return expecs


# ---------------------------------------------------------- Schmidt values ---
def mps_singular_values(sites, i, info=None, method="svd"):
    """Singular values of the bond (i - 1, i), the centre moved to site i in
    place (singular_values, tn1d/core.py:1472-1506); ``method`` 'svd' or
    'eig'."""
    sites = _prepare(sites)
    L = len(sites)
    if not 0 < i < L:
        raise ValueError(f"Need 0 < i < {L}, got i={i}.")
    mps_canonicalize(sites, i, info=info)
    A = sites[i]
    l, d, r = A.shape
    return array_svals(A.reshape(l, d * r), method=method)


def mps_schmidt_values(sites, i, info=None, method="svd"):
    """Squared singular values of the bond (i - 1, i) (schmidt_values,
    tn1d/core.py:2637-2666)."""
    return mps_singular_values(sites, i, info=info, method=method) ** 2


def mps_entropy(sites, i, info=None, method="svd"):
    """-sum S log2 S over the Schmidt values S > 0 of the bond (i - 1, i)
    (entropy, tn1d/core.py:2668-2695); a 0-d device Array."""
    S = mps_schmidt_values(sites, i, info=info, method=method).t
    pos = S > 0.0
    terms = torch.where(pos, S * torch.log2(torch.where(pos, S, torch.ones_like(S))),
                        torch.zeros_like(S))
    return Array(-terms.sum())


def mps_schmidt_gap(sites, i, info=None, method="svd"):
    """S[0] - S[1] of the Schmidt values of the bond (i - 1, i), or S[0] if
    there is one (schmidt_gap, tn1d/core.py:2697-2725)."""
    S = mps_schmidt_values(sites, i, info=info, method=method)
    if S.shape[0] == 1:
        return S[0]
    return S[0] - S[1]


# ----------------------------------------------------- spin and correlators ---
def spin_operator(label, S=0.5):
    """Spin-S operator 'X', 'Y' or 'Z' as a host array, built as
    quimb.gen.operators.spin_operator builds it (complex, then real if the
    imaginary part vanishes)."""
    D = int(2 * S + 1)
    op = np.zeros((D, D), dtype=complex)
    ms = np.linspace(S, -S, D)
    label = label.lower()
    if label in {"x", "y"}:
        for k in range(D - 1):
            c = 0.5 * (S * (S + 1) - (ms[k] * ms[k + 1])) ** 0.5
            op[k, k + 1] = -1.0j * c if label == "y" else c
            op[k + 1, k] = 1.0j * c if label == "y" else c
    elif label == "z":
        for k in range(D):
            op[k, k] = ms[k]
    else:
        raise ValueError(f"Label '{label}' not understood, should be one of "
                         "'X', 'Y', 'Z'.")
    return np.real_if_close(op)


def mps_magnetization(sites, i, direction="Z", info=None):
    """sum_{p, q} T[.., p, ..] O[p, q] conj(T[.., q, ..]) at the centre moved to
    site i, O the spin-(d - 1)/2 operator of ``direction`` (magnetization,
    tn1d/core.py:2605-2634: unnormalised, O contracted as the reference
    contracts it)."""
    sites = _prepare(sites)
    mps_canonicalize(sites, i, info=info)
    d = sites[i].shape[1]
    rho = _rho(sites, (i,)).astype(sites[i].dtype, copy=False)
    O = ops.asarray(spin_operator(direction, S=(d - 1) / 2), device=rho.device)
    return ops.einsum("pq,pq->", O, rho)


def mps_correlation(sites, A, i, j, B=None):
    """``<A(i) B(j)> - <A(i)> <B(j)>`` for single sites i != j, unnormalised
    (correlation, tn1d/core.py:699-741); works on copies of the list."""
    if not (isinstance(i, numbers.Integral) and isinstance(j, numbers.Integral)) or i == j:
        raise NotImplementedError("mps_correlation: single sites i != j only")
    if B is None:
        B = A
    psi = _prepare(list(sites))
    pA = list(psi)
    tebd.gate_single(pA, A, i)
    cA = tebd.mps_overlap_array(psi, pA)
    pB = list(psi)
    tebd.gate_single(pB, B, j)
    cB = tebd.mps_overlap_array(psi, pB)
    tebd.gate_single(pA, B, j)
    cAB = tebd.mps_overlap_array(psi, pA)
    return cAB - cA * cB
