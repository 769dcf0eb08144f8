"""GPU tier: every kernel route of the QR and SVD against exact and bounded
oracles (``tests/decomp_oracle.py``).

The library reports which kernels a QR or SVD takes (``linalg.route_qr`` /
``linalg.route_svd``: panel instantiations, aggregation, TSQR, Jacobi stream
groups, the sweep graph, the epilogue, the host-layer transposes).  The route
search asks it for the cheapest grid shape that reaches each route, and every
route is run through:

(a) the exact dyadic oracle, for every absorb mode and cutoff mode it serves;
(b) sentinel buffers on the raw C ABI: NaN-padded input, outputs pre-filled
    with a bit pattern that must survive outside the declared regions;
(c) a repeated call, bit-identical (first-call graph capture against replay);
(d) rank deficiency: exact zero and duplicated columns.

Further: the mpmath oracle at small n, the exponent range 2^+-1000 and
subnormal input, column blocks 2^520 apart, NaN / Inf input, and two
subprocess runs with the Jacobi switches that are read once per process.
"""

import ctypes
import os
import sys
import textwrap
import zlib

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from quimb_b200 import _lib, linalg
from tests import decomp_oracle as do
from tests.test_gpu_p2p import run_process_group

pytestmark = pytest.mark.gpu

SENT = 0x7FF8DEADBEEF0001
KEYS = do.QR_KEYS + do.SVD_KEYS
ABSORB_ALL = (100, 2, -1, -10, -11, 0, -12, 12, 1, 10, 11)
# quimb's absorb code -> (powers of s on the left / right factor, which exist)
_PLAN = {100: (0, 0, 1, 1), 2: (0, 0, 0, 0), -1: (1, 0, 1, 1), -10: (1, 0, 1, 0),
         -11: (0, 0, 0, 1), 0: (.5, .5, 1, 1), -12: (.5, 0, 1, 0), 12: (0, .5, 0, 1),
         1: (0, 1, 1, 1), 10: (0, 0, 1, 0), 11: (0, 1, 0, 1)}


@pytest.fixture(scope="module")
def routes():
    return do.search_routes()


@pytest.fixture(scope="module")
def routes3():
    """Shapes of at least three rows and columns with the same route report
    (rank deficiency, truncation and sentinel checks need them)."""
    return do.search_routes(min_cols=3)


def _id(key):
    return "-".join(str(k) for k in key)


def _rng(*salt):
    return np.random.default_rng(zlib.crc32(repr(salt).encode()))


def _dev(x):
    return qb.asarray(np.ascontiguousarray(x))


def _np(a):
    return None if a is None else a.to_numpy()


def _qr(A, **kw):
    Q, R = linalg.qr(_dev(A), stabilized=True, **kw)
    return _np(Q), _np(R)


def _svd(A):
    U, s, VH = linalg.svd(_dev(A))
    return _np(U), _np(s), _np(VH)


def _check_trunc(A, code, left, s, right, s_exact, nk, scale=1.0):
    """svd_trunc factors of mode `code` against the exact spectrum."""
    lp, rp, wl, wr = _PLAN[code]
    n = A.shape[1]
    sk = s_exact[:nk] * scale
    if code in (100, 2):
        assert s.shape == (nk,)
        es = np.abs(s - sk).max(initial=0.0)
        assert es <= do.bound(n) * s_exact[0] * scale + do.C * n * do.TINY
    if not (wl and wr):
        for f in (left, right):
            if f is not None and f.size:
                assert np.all(np.isfinite(f))
        if left is not None and lp == 0:
            do.check_orthonormal_cols(left[:, sk > 0], n, "left isometry")
        if right is not None and rp == 0:
            do.check_orthonormal_cols(right[sk > 0].T, n, "right isometry")
        return
    mid = s if code == 100 else np.ones(nk)
    rec = (left * mid) @ right
    # best rank-nk approximation: |A - rec| = sqrt(sum of the dropped s^2)
    drop = float(np.sqrt(np.sum((s_exact[nk:] * scale) ** 2)))
    err = np.linalg.norm(A - rec)
    tol = do.bound(n) * np.linalg.norm(A) + do.C * n * do.TINY
    assert abs(err - drop) <= tol + 1e-8 * drop, (err, drop)
    for f, p, side in ((left, lp, "left"), (right, rp, "right")):
        if p == 0:
            do.check_orthonormal_cols(f if side == "left" else f.T, n, side)


# ------------------------------------------------------------ route coverage
def test_route_search_covers_every_decomposition_route(routes):
    lines = [f"{_id(k):34s} {routes[k][0]} {routes[k][1]} absorb={routes[k][2]}"
             for k in KEYS if k in routes]
    print("\n" + "\n".join(lines))
    missing = [k for k in KEYS if k not in routes]
    assert not missing, f"routes no grid shape reaches: {missing}"


# ------------------------------------------------------------------- QR routes
@pytest.mark.parametrize("key", do.QR_KEYS, ids=_id)
def test_qr_route_exact_oracle(routes, key):
    assert key in routes, f"no grid shape reaches {key}"
    (m, n), dt, _, r = routes[key]
    assert linalg.route_qr((m, n), dt) == r
    rng = _rng("qr", key)
    if dt == torch.complex128:
        A = rng.standard_normal((m, n)) + 1j * rng.standard_normal((m, n))
        Q, R = _qr(A)
        k = min(m, n)
        assert np.abs(Q @ R - A).max() <= do.bound(n) * np.abs(A).sum(1).max()
        assert np.abs(Q.conj().T @ Q - np.eye(k)).max() <= do.bound(n)
        assert np.all(np.abs(np.diag(R).imag) == 0) and np.all(np.diag(R).real >= 0)
        return
    A, Q0, R0, kappa = do.qr_case(m, n, rng)
    Q, R = _qr(A)
    do.check_qr(A, Q, R, kappa=kappa, Q0=Q0, R0=R0)
    _, R2 = _qr(A, want_q=False)
    np.testing.assert_array_equal(R2, R)
    Q3, R3 = _qr(A)
    assert np.array_equal(Q3, Q) and np.array_equal(R3, R), "repeated call differs"


@pytest.mark.parametrize("key", do.QR_KEYS, ids=_id)
def test_qr_route_rank_deficient(routes3, key):
    (m, n), dt, _, _ = routes3[key]
    if dt != torch.float64:
        pytest.skip("real routes")
    rng = _rng("qr-rank", key)
    A, *_ = do.qr_case(m, n, rng)
    A[:, 0] = 0.0                       # exact zero column
    A[:, min(m, n) - 1] = A[:, 1]       # duplicated column (inside the panel range)
    Q, R = _qr(A)
    do.check_qr(A, Q, R)


def _padded_dev(nelem, fill_bits=None, fill=float("nan"), pad=4096):
    buf = torch.empty(nelem + 2 * pad, dtype=torch.float64, device="cuda")
    if fill_bits is None:
        buf.fill_(fill)
    else:
        buf.view(torch.int64).fill_(fill_bits)
    return buf, buf[pad:pad + nelem]


def _sent_intact(buf, lo, hi, pad=4096):
    bits = buf.view(torch.int64).cpu().numpy()
    keep = np.ones(bits.size, bool)
    keep[pad + lo:pad + hi] = False
    return bool(np.all(bits[keep] == SENT))


@pytest.mark.parametrize("key", [k for k in do.QR_KEYS if k[1] == "panel" or k[1] == "aggregated"],
                         ids=_id)
def test_qr_raw_abi_sentinels(routes3, key):
    """qb_qr_stab on a NaN-padded input writes exactly Q (m x k) and R (k x n)."""
    (m, n), _, _, r = routes3[key]
    kern = r["kernels"][0]
    m, n = kern["shape"]
    k = min(m, n)
    A, *_ = do.qr_case(m, n, _rng("qr-sent", key))
    lib = _lib.load()
    xb, X = _padded_dev(m * n)
    X.copy_(torch.from_numpy(A.reshape(-1)))
    qb_, Q = _padded_dev(m * k, SENT)
    rb_, R = _padded_dev(k * n, SENT)
    need = lib.qb_qr_workspace(_lib.QB_F64, m, n)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    rc = lib.qb_qr_stab(_lib.QB_F64, m, n, X.data_ptr(), Q.data_ptr(), R.data_ptr(), 1,
                        ws.data_ptr(), need, _lib.stream_ptr())
    _lib.check(rc, "qb_qr_stab")
    torch.cuda.synchronize()
    assert _sent_intact(qb_, 0, m * k) and _sent_intact(rb_, 0, k * n)
    do.check_qr(A, Q.cpu().numpy().reshape(m, k), R.cpu().numpy().reshape(k, n))


# ------------------------------------------------------------------ SVD routes
def _svd_case_for(key, m, n, kind="separated"):
    mm, nn = max(m, n), min(m, n)
    A, U0, s, V0 = do.svd_case(mm, nn, kind, _rng("svd", key, kind))
    if m < n:                            # wide: A^T = V0 s U0^T
        return A.T.copy(), V0, s, U0
    return A, U0, s, V0


@pytest.mark.parametrize("key", do.SVD_KEYS, ids=_id)
def test_svd_route_exact_oracle(routes, key):
    assert key in routes, f"no grid shape reaches {key}"
    (m, n), dt, absorb, r = routes[key]
    assert linalg.route_svd((m, n), dt, absorb) == r
    if dt == torch.complex128:
        rng = _rng("svd-c", key)
        A = rng.standard_normal((m, n)) + 1j * rng.standard_normal((m, n))
        U, s, VH = _svd(A)
        ref = np.linalg.svd(A, compute_uv=False)
        assert np.abs(s - ref).max() <= do.bound(max(m, n)) * ref[0]
        assert np.abs((U * s) @ VH - A).max() <= do.bound(max(m, n)) * ref[0]
        return
    kinds = ("separated", "clusters", "zeros", "graded", "gap") if min(m, n) >= 3 else ("separated",)
    for kind in kinds:
        A, U0, s_ex, V0 = _svd_case_for(key, m, n, kind)
        if absorb is None:
            U, s, VH = _svd(A)
            do.check_svd(A, U, s, VH, s_ex, U0, V0)
            U2, s2, VH2 = _svd(A)
            assert np.array_equal(U2, U) and np.array_equal(VH2, VH), "repeated call differs"
            continue
        k = min(m, n)
        cuts = [(-1.0, 4, -1)]
        if kind == "gap":
            r0 = max(1, k // 3)
            cuts += [(2.0 ** -10, 1, -1), (2.0 ** -10, 2, -1), (2.0 ** -30, 3, -1),
                     (2.0 ** -40, 4, -1), (2.0 ** -15, 5, -1), (2.0 ** -25, 6, -1),
                     (-1.0, 4, max(1, r0 - 1))]
        for cutoff, mode, mb in cuts:
            info = {"error": None}
            left, s, right = (_np(t) for t in linalg.svd_trunc(
                _dev(A), cutoff, mode, mb, absorb, 0, info))
            nk, err = do.keep_rule(s_ex, cutoff, mode, mb)
            assert info["n_keep"] == nk, (kind, cutoff, mode, info["n_keep"], nk)
            assert abs(info["error"] - err) <= do.bound(k) * s_ex[0] + 1e-12 * err
            _check_trunc(A, absorb, left, s, right, s_ex, nk)
            again = [_np(t) for t in linalg.svd_trunc(_dev(A), cutoff, mode, mb, absorb, 0)]
            for x, y in zip((left, s, right), again):
                assert (x is None and y is None) or np.array_equal(x, y), "repeated call differs"


@pytest.mark.parametrize("key", [k for k in do.SVD_KEYS if k[1] in ("epilogue", "groups")],
                         ids=_id)
def test_svd_trunc_raw_abi_sentinels(routes3, key):
    """qb_svd_trunc writes U (m x nk), S (nk) and VH (nk x n) and nothing
    past the kept rank; the input sits in a NaN-padded buffer."""
    (m, n), _, absorb, r = routes3[key]
    m, n = r["kernel_shape"]
    code = r["absorb"]
    if n < 2:
        pytest.skip("needs a truncation")
    A, _, s_ex, _ = _svd_case_for(key, m, n)
    mb = n // 2
    lib = _lib.load()
    xb, X = _padded_dev(m * n)
    X.copy_(torch.from_numpy(A.reshape(-1)))
    ub, U = _padded_dev(m * n, SENT)
    sb, S = _padded_dev(n, SENT)
    vb, VH = _padded_dev(n * n, SENT)
    need = lib.qb_svd_workspace(_lib.QB_F64, m, n)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    nk, err, nnull = ctypes.c_int64(0), ctypes.c_double(0.0), ctypes.c_int64(0)
    sw = ctypes.c_int(0)
    rc = lib.qb_svd_trunc(_lib.QB_F64, m, n, X.data_ptr(), -1.0, 4, mb, code, 0,
                          U.data_ptr(), S.data_ptr(), VH.data_ptr(), ctypes.byref(nk),
                          ctypes.byref(err), ctypes.byref(nnull), ws.data_ptr(), need,
                          ctypes.byref(sw), _lib.stream_ptr())
    _lib.check(rc, "qb_svd_trunc")
    torch.cuda.synchronize()
    k = nk.value
    assert k == mb
    _, _, wl, wr = _PLAN[code]
    assert _sent_intact(ub, 0, m * k if wl else 0), "U written outside m x nk"
    assert _sent_intact(vb, 0, k * n if wr else 0), "VH written outside nk x n"
    assert _sent_intact(sb, 0, k if code in (100, 2) else 0), "S written outside nk"


@pytest.mark.parametrize("key", [k for k in do.SVD_KEYS if k[1] != "complex"], ids=_id)
def test_svd_route_rank_deficient_isometries(routes3, key):
    """Zero and duplicated columns: the kept null directions are completed, so
    the isometric factors stay isometries."""
    (m, n), _, absorb, _ = routes3[key]
    A, *_ = _svd_case_for(key, m, n)
    A = A.copy()
    A[:, 0] = 0.0
    A[:, 1] = A[:, 2]
    for code in (100, -1, 1):
        left, s, right = (_np(t) for t in linalg.svd_trunc(_dev(A), -1.0, 4, -1, code, 0))
        k = min(m, n)
        if code in (100, 1):
            do.check_orthonormal_cols(left, k, "left")
        if code in (100, -1):
            do.check_orthonormal_cols(right.T, k, "right")
        rec = (left * s) @ right if code == 100 else left @ right
        assert np.linalg.norm(A - rec) <= do.bound(k) * np.linalg.norm(A)


# --------------------------------------------------------------- mpmath oracle
@pytest.mark.parametrize("key", [k for k in KEYS if k[1] != "complex"], ids=_id)
def test_route_against_mpmath(routes3, key):
    """Random (not dyadic) matrices on each route's shape of at least three
    columns, where that shape is small enough for mpmath at 40 digits."""
    pytest.importorskip("mpmath")
    (m, n), _, absorb, _ = routes3[key]
    if min(m, n) > 48 or m * n * min(m, n) > 400_000:
        pytest.skip(f"{(m, n)} is too large for the mpmath oracle")
    A = _rng("mp", key).standard_normal((m, n))
    s_mp = do.mp_svd(A)
    k = min(m, n)
    if key[0] == "qr":
        Q, R = _qr(A)
        do.check_qr(A, Q, R)
        # wide input: the leading k x k block of R is the QR of A[:, :k]
        R_mp = do.mp_qr_r(A[:, :k])
        kappa = s_mp[0] / s_mp[-1]
        assert np.abs(R[:, :k] - R_mp).max() <= do.bound(max(m, n)) * kappa * np.abs(R_mp).max()
        return
    if absorb is None:
        U, s, VH = _svd(A)
        do.check_svd(A, U, s, VH)
    else:
        _, s, _ = linalg.svd_trunc(_dev(A), -1.0, 4, -1, 2, 0)
        s = _np(s)
        left, sm, right = (_np(t) for t in linalg.svd_trunc(_dev(A), -1.0, 4, -1, absorb, 0))
        _check_trunc(A, absorb, left, sm, right, s_mp, k)
    assert np.abs(s - s_mp).max() <= do.bound(max(m, n)) * s_mp[0]


# -------------------------------------------------------------- exponent range
EXPS = (2, -2, 300, -300, 520, -520, 600, -600, 1000, -1000, -1070)


def _stored(A, k):
    """A 2^k as float64 (rounded when subnormal), that matrix times 2^-k (the
    oracle's input: exact, since scaling up by 2^-k is exact), and one unit
    in the last place of a subnormal, in those scaled-back units."""
    As = np.ldexp(A, k)
    return As, np.ldexp(As, -k), np.ldexp(do.TINY, -k)


@pytest.mark.parametrize("k", EXPS)
def test_qr_exponent_range(k):
    for (m, n) in ((200, 48), (4096, 160)):
        A, Q0, R0, kappa = do.qr_case(m, n, _rng("qr-exp", m, k))
        As, Ab, ulp = _stored(A, k)
        Q, R = _qr(As)
        assert np.all(np.isfinite(Q)) and np.all(np.isfinite(R))
        Rb = np.ldexp(R, -k)
        if np.array_equal(Ab, A):
            do.check_qr(Ab, Q, Rb, kappa=kappa, Q0=Q0, R0=R0)
            continue
        # subnormal storage: the oracle of the matrix as stored; each entry of
        # R is rounded once more (half an ulp) when it is scaled back
        q, r = np.linalg.qr(Ab)
        sg = np.where(np.diag(r) < 0, -1.0, 1.0)
        r = r * sg[:, None]
        do.check_qr(Ab, Q, Rb, floor=np.sqrt(m) * n * ulp)
        kap = np.linalg.cond(r)
        assert np.abs(Rb - r).max() <= do.bound(n) * kap * np.abs(r).max() + ulp


@pytest.mark.parametrize("k", EXPS)
def test_svd_exponent_range(k):
    m, n = 300, 64
    A, U0, s_ex, V0 = do.svd_case(m, n, "separated", _rng("svd-exp", k))
    As, Ab, ulp = _stored(A, k)
    exact = np.array_equal(Ab, A)
    s_ref = s_ex if exact else np.linalg.svd(Ab, compute_uv=False)
    floor = np.sqrt(m) * n * ulp
    U, s, VH = _svd(As)
    assert np.all(np.isfinite(s))
    sb = np.ldexp(s, -k)
    assert np.abs(sb - s_ref).max() <= do.bound(n) * s_ref[0] + ulp
    if exact:
        do.check_svd(Ab, U, sb, VH, s_ex, U0, V0)
    else:
        do.check_svd(Ab, U, sb, VH, s_ref, floor=floor)
    for code in ABSORB_ALL:
        info = {"error": None}
        cut = np.ldexp(0.5 * (s_ref[n // 2] + s_ref[n // 2 + 1]), k)   # absolute, caller's units
        left, s, right = (_np(t) for t in linalg.svd_trunc(_dev(As), cut, 1, -1, code, 0, info))
        nk = n // 2 + 1
        assert info["n_keep"] == nk, (code, info["n_keep"])
        # the reference rule in the caller's units (its squares overflow or
        # underflow as the reference's do)
        err = float(np.sqrt(np.sum(np.ldexp(s_ref[nk:], k) ** 2)))
        if err == 0.0 or not np.isfinite(err):
            assert info["error"] == err
        else:
            assert abs(np.ldexp(info["error"] - err, -k)) <= do.bound(n) * s_ref[0] + n * ulp
        for f in (left, s, right):
            assert f is None or np.all(np.isfinite(f))
        lp, rp, wl, wr = _PLAN[code]
        if lp == 0 and wl:
            do.check_orthonormal_cols(left, n, "left isometry")
        if rp == 0 and wr:
            do.check_orthonormal_cols(right.T, n, "right isometry")
        if wl and wr:
            rec = np.ldexp((left * s) @ right if code == 100 else left @ right, -k)
            best = float(np.sqrt(np.sum(s_ref[nk:] ** 2)))
            assert np.linalg.norm(Ab - rec) <= best + do.bound(n) * s_ref[0] * np.sqrt(n) + floor


@pytest.mark.parametrize("k", EXPS)
def test_eigh_exponent_range(k):
    n = 96
    rng = _rng("eigh-exp", k)
    V = do.to_float(do.isometry(n, n, rng))
    w = np.arange(-n // 2, n - n // 2, dtype=np.float64)        # exact, distinct
    A = (V * w) @ V.T
    As, Ab, ulp = _stored(A, k)
    w_ref = w if np.array_equal(Ab, A) else np.linalg.eigvalsh(Ab)
    wd, vd = linalg.eigh(_dev(As))
    wd, vd = np.ldexp(_np(wd), -k), _np(vd)
    assert np.all(np.isfinite(wd)) and np.all(np.isfinite(vd))
    assert np.abs(wd - w_ref).max() <= do.bound(n) * np.abs(w_ref).max() * 4 + 2 * ulp
    do.check_orthonormal_cols(vd, n, "eigenvectors")
    assert np.linalg.norm(Ab @ vd - vd * wd) <= do.bound(n) * 4 * np.abs(w_ref).max() * np.sqrt(n) \
        + n * ulp


@pytest.mark.xfail(torch.cuda.is_available(), strict=True,
                   reason="the Householder panel's dlarfg sums squares without scaling: "
                   "columns 2^520 below the largest underflow there, and Q (so U) "
                   "loses orthogonality (1.2e-11 measured at 256 x 64)")
def test_svd_column_blocks_2_520_apart():
    """Two column blocks whose scales differ by 2^520: the Jacobi iteration
    converges (a pair it does not rotate is not flagged either) and the
    factors meet the bounds relative to the large block."""
    m, n = 256, 64
    A, *_ = do.svd_case(m, n, "separated", _rng("mixed"))
    A[:, n // 2:] = np.ldexp(A[:, n // 2:], -520)
    for B in (A, np.ldexp(A, 300)):
        U, s, VH = _svd(B)
        do.check_svd(B, U, s, VH)
        ref = np.linalg.svd(B, compute_uv=False)
        assert np.abs(s - ref).max() <= do.bound(n) * ref[0]


# ------------------------------------------------------------ non-finite input
@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf], ids=["nan", "inf", "-inf"])
@pytest.mark.parametrize("col", ["first", "middle", "last"])
def test_nonfinite_input(bad, col):
    m, n = 200, 96
    A = _rng("nf", col).standard_normal((m, n))
    c = {"first": 0, "middle": n // 2, "last": n - 1}[col]
    A[m // 3, c] = bad
    for fn in (lambda x: linalg.svd(x), lambda x: linalg.svd_trunc(x, 1e-3, 4, -1, 0, 0),
               lambda x: qb.array_split(x, method="svd", cutoff=1e-10),
               lambda x: linalg.svd(qb.asarray(np.ascontiguousarray(A.T)))):
        with pytest.raises(ValueError, match="NaN or Inf"):
            fn(_dev(A))
    S = A[:n] + A[:n].T
    with pytest.raises(ValueError, match="NaN or Inf"):
        linalg.eigh(_dev(S))
    _, R = _qr(A)
    assert not np.all(np.isfinite(R)), "QR returned an all-finite R from non-finite input"


# ------------------------------------------------------------- process switches
_SCRIPT = textwrap.dedent("""
    import sys, numpy as np
    sys.path.insert(0, {root!r})
    import quimb_b200 as qb
    from quimb_b200 import linalg
    from tests import decomp_oracle as do
    out = {{}}
    for n in (512, 1024):
        A, *_ = do.svd_case(n + 64, n, "clusters", np.random.default_rng(n))
        for code in (100, -1, 1, 2):
            l, s, r = linalg.svd_trunc(qb.asarray(A), -1.0, 4, -1, code, 0)
            for name, t in (("l", l), ("s", s), ("r", r)):
                if t is not None:
                    out[f"{{n}}_{{code}}_{{name}}"] = t.to_numpy()
    np.savez({path!r}, **out)
""")


def _run_switched(tmp_path, env_extra):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    path = str(tmp_path / f"out_{len(env_extra)}_{'_'.join(env_extra)}.npz")
    env = dict(os.environ, **env_extra)
    rc, _, err = run_process_group([sys.executable, "-c", _SCRIPT.format(root=root, path=path)],
                                   timeout=600, env=env)
    assert rc == 0, err[-3000:]
    return dict(np.load(path))


def test_process_switches_graph_and_accumulate(tmp_path):
    base = _run_switched(tmp_path, {})
    for n in (512, 1024):
        assert linalg.route_svd((n + 64, n))["graph_sweeps"] > 0
    nograph = _run_switched(tmp_path, {"QB_JAC_GRAPH": "0"})
    assert base.keys() == nograph.keys()
    for key in base:
        assert np.array_equal(base[key], nograph[key]), f"QB_JAC_GRAPH=0 changed {key}"
    acc = _run_switched(tmp_path, {"QB_SVD_ACCUMULATE": "1"})
    for n in (512, 1024):
        A, _, s_ex, _ = do.svd_case(n + 64, n, "clusters", np.random.default_rng(n))
        for code in (100, -1, 1, 2):
            get = lambda nm: acc.get(f"{n}_{code}_{nm}")   # noqa: E731
            _check_trunc(A, code, get("l"), get("s"), get("r"), s_ex, n)
