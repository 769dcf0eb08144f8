"""GPU tier: MPS observables (``quimb_b200.observables``) and the
``qb_rdm_reduce`` kernel.

The host layer is checked against what the unmodified reference computed
(tests/golden/observables.*) and against the numpy oracle
(oracle/observables_np.py) at larger sizes; the raw kernel against a numpy
einsum, for bitwise reproducibility across streams and graph replay, for
NaN / Inf propagation, its error codes and its launch count."""

import ctypes
import warnings

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from quimb_b200 import _lib, observables as obs
from oracle import observables_np as onp
from oracle.observables_np import terms_for
from tests.conftest import load_golden
from tests.test_gpu_mps_sample import rand_mps

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------- helpers ---
def _host_sites(data, meta, name, prefix=None):
    L = meta["states"][name]["L"]
    key = prefix or f"{name}__site"
    return [np.ascontiguousarray(data[f"{key}{i}"]) for i in range(L)]


def _np(x):
    return np.asarray(x.to_numpy() if hasattr(x, "to_numpy") else x)


def _close(got, want, tol=1e-10):
    got, want = _np(got), np.asarray(want)
    scale = max(1.0, float(np.max(np.abs(want), initial=0.0)))
    assert got.shape == want.shape, (got.shape, want.shape)
    np.testing.assert_allclose(got, want, rtol=0, atol=tol * scale)


def _info(x):
    return tuple(x) if isinstance(x, list) else x


def run_golden_case(data, meta, k, case):
    """One fixture case on the device layer; asserts values, the recorded
    centre and (inplace) the site arrays."""
    name = case["state"]
    pre = f"case{k}__"
    sites = _host_sites(data, meta, name)
    L, d = meta["states"][name]["L"], meta["states"][name]["d"]
    kind = case["kind"]
    if kind == "schmidt":
        psi, info = [qb.asarray(a) for a in sites], {}
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", FutureWarning)
            for i in range(1, L):
                S = _np(qb.mps_schmidt_values(psi, i, info=info, method=case["method"]))
                ref = data[pre + f"S{i}"]
                np.testing.assert_allclose(S, ref, rtol=0, atol=1e-12 * ref[0])
                _close(qb.mps_entropy(psi, i, info=info, method=case["method"]),
                       data[pre + "entropy"][i - 1])
                _close(qb.mps_schmidt_gap(psi, i, info=info, method=case["method"]),
                       data[pre + "gap"][i - 1])
        assert info["cur_orthog"] == tuple(case["cur_orthog"])
    elif kind == "rho":
        psi, info = [qb.asarray(a) for a in sites], {}
        where = tuple(case["where"])
        D_P = int(np.prod([d] * (len(where) - 1)))
        contiguous = list(where) == list(range(where[0], where[-1] + 1))
        too_wide = (d ** len(where) > 64) if contiguous else (D_P * D_P * d > 64)
        if too_wide:
            with pytest.raises(NotImplementedError):
                qb.mps_partial_trace_to_dense_canonical(psi, where, case["normalized"], info)
            return
        rho = qb.mps_partial_trace_to_dense_canonical(psi, where, case["normalized"], info)
        _close(rho, data[pre + "rho"])
        assert info["cur_orthog"] == tuple(case["cur_orthog"])
    elif kind == "expec":
        if case["start"] is not None:
            sites = [np.ascontiguousarray(data[pre + f"in{i}"]) for i in range(L)]
        terms = terms_for(case["terms"], L, d)
        info = None if case["info"] is None else {"cur_orthog": _info(case["info"]["cur_orthog"])} \
            if "cur_orthog" in case["info"] else {}
        psi = [qb.asarray(a) for a in sites]
        before = [_np(a).copy() for a in psi]
        info_before = None if info is None else dict(info)
        got = qb.mps_compute_local_expectation(
            psi, terms, return_all=case["return_all"], method=case["method"], info=info,
            inplace=case["inplace"])
        if case["return_all"]:
            assert [list(k) for k in got] == case["keys"]
            vals = [got[tuple(k)] for k in case["keys"]]
        else:
            vals = [got]
        _close(np.array([complex(_np(v)) for v in vals]), data[pre + "values"])
        if "cur_orthog_after" in case:
            assert info["cur_orthog"] == _info(case["cur_orthog_after"])
        if case["inplace"]:
            for i in range(L):
                _close(psi[i], data[pre + f"out{i}"])
        else:
            assert info == info_before
            for a, b in zip(psi, before):
                assert np.array_equal(_np(a), b)
    elif kind == "mag":
        psi, info = [qb.asarray(a) for a in sites], {}
        vals = [complex(_np(qb.mps_magnetization(psi, case["site"], c, info=info)))
                for c in "XYZ"]
        _close(np.array(vals), data[pre + "values"])
        assert info["cur_orthog"] == tuple(case["cur_orthog"])
    elif kind == "corr":
        Z, X = onp.spin_operator("Z") * 2, onp.spin_operator("X") * 2
        psi = [qb.asarray(a) for a in sites]
        c = qb.mps_correlation(psi, Z, case["i"], case["j"], B=X if case["B"] else None)
        _close(complex(_np(c)), data[pre + "value"])
    else:
        raise AssertionError(kind)


# ------------------------------------------------------------------ golden ---
def test_golden_matches_reference():
    data, meta = load_golden("observables")
    for k, case in enumerate(meta["cases"]):
        run_golden_case(data, meta, k, case)


def test_correlation_docstring_values():
    data, meta = load_golden("observables")
    psi = _host_sites(data, meta, "ghz")
    Z, X = onp.spin_operator("Z") * 2, onp.spin_operator("X") * 2
    assert complex(_np(qb.mps_correlation(psi, Z, 0, 1))) == pytest.approx(1.0, abs=1e-12)
    assert complex(_np(qb.mps_correlation(psi, Z, 0, 1, B=X))) == pytest.approx(0.0, abs=1e-12)
    for i, j in ((0, 0), ((0, 1), 2)):
        with pytest.raises(NotImplementedError):
            qb.mps_correlation(psi, Z, i, j)


def test_singular_values_bond_range():
    psi = rand_mps(6, 4, 2, np.float64, 1)
    for i in (0, 6):
        with pytest.raises(ValueError):
            qb.mps_singular_values(psi, i)


# ------------------------------------------------------------------ oracle ---
def check_against_oracle(L, chi, d, dtype, seed, tol=1e-10):
    host = rand_mps(L, chi, d, dtype, seed)
    psi = [qb.asarray(a) for a in host]
    ref = [a.copy() for a in host]
    terms = {(i,): onp.spin_operator("Z", (d - 1) / 2) for i in range(L)}
    terms.update({(i, i + 1): np.kron(onp.spin_operator("X", (d - 1) / 2),
                                      onp.spin_operator("X", (d - 1) / 2))
                  for i in range(0, L - 1, 3)})
    for method in ("canonical", "envs"):
        got = qb.mps_compute_local_expectation(psi, terms, return_all=True, method=method)
        want = onp.compute_local_expectation(ref, terms, return_all=True, method=method)
        _close(np.array([complex(_np(got[k])) for k in want]), np.array(list(want.values())),
               tol)
    info, oinfo = {}, {}
    for where in ((L // 2,), (1, 4), (2, 3, 4)):
        _close(qb.mps_partial_trace_to_dense_canonical(psi, where, info=info),
               onp.partial_trace_to_dense_canonical(ref, where, info=oinfo), tol)
        assert info == oinfo
    for i in range(1, L, 7):
        S = _np(qb.mps_schmidt_values(psi, i, info=info))
        So = onp.schmidt_values(ref, i, info=oinfo)
        np.testing.assert_allclose(S, So, rtol=0, atol=1e-12 * So[0] if tol < 1e-8 else tol)
        _close(qb.mps_entropy(psi, i, info=info), onp.entropy(ref, i, info=oinfo), tol)
    return psi


@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
@pytest.mark.parametrize("d", [2, 3])
def test_matches_oracle_large(dtype, d):
    check_against_oracle(40, 128, d, dtype, seed=10 + d)


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
def test_single_precision_keeps_dtype(dtype):
    host = rand_mps(12, 16, 2, dtype, 4)
    psi = [qb.asarray(a) for a in host]
    ref = [a.astype(np.complex128 if np.dtype(dtype).kind == "c" else np.float64)
           for a in host]
    rho = qb.mps_partial_trace_to_dense_canonical(psi, (3, 4))
    assert rho.dtype == np.dtype(dtype)
    _close(rho, onp.partial_trace_to_dense_canonical(ref, (3, 4)), 1e-5)
    S = qb.mps_schmidt_values(psi, 6)
    _close(S, onp.schmidt_values(ref, 6), 1e-5)


def test_sweep_moves_centre_once_per_site(monkeypatch):
    """A sorted sweep of all one-site terms from a known centre moves the
    centre L - 1 times; from "calc" on a random state, one full
    canonicalisation (L - 1 moves) more."""
    from quimb_b200 import tebd
    L = 9
    calls = {"n": 0}
    for name in ("left_canonize_site", "right_canonize_site"):
        fn = getattr(tebd, name)

        def counted(sites, i, fn=fn):
            calls["n"] += 1
            return fn(sites, i)
        monkeypatch.setattr(tebd, name, counted)
    host = rand_mps(L, 8, 2, np.float64, 2)
    Z = onp.spin_operator("Z") * 2
    terms = {(i,): Z for i in range(L)}
    psi = [qb.asarray(a) for a in host]
    qb.mps_compute_local_expectation(psi, terms, return_all=True)
    assert calls["n"] == 2 * (L - 1)
    psi = [qb.asarray(a) for a in host]
    info = {}
    qb.mps_canonicalize(psi, 0, info=info)
    calls["n"] = 0
    qb.mps_compute_local_expectation(psi, terms, return_all=True, info=info)
    assert calls["n"] == L - 1
    assert info["cur_orthog"] == (0, 0)          # the caller's info is not updated
    qb.mps_compute_local_expectation(psi, terms, info=info, inplace=True)
    assert info["cur_orthog"] == (L - 1, L - 1)


# -------------------------------------------------------------- raw kernel ---
RAW_SHAPES = [(1, 1, 1, 1), (7, 3, 3, 5), (33, 64, 64, 17), (1024, 2, 2, 1024), (5, 8, 2, 9)]


def _rand(rng, shape, cplx):
    x = rng.standard_normal(shape)
    if cplx:
        x = x + 1j * rng.standard_normal(shape)
    return x


def _ref(U, V):
    return np.einsum("amb,anb->mn", U, V.conj())


@pytest.mark.parametrize("shape", RAW_SHAPES)
@pytest.mark.parametrize("cplx", [False, True])
def test_raw_kernel_matches_einsum(shape, cplx):
    n1, M, N, n2 = shape
    rng = np.random.default_rng(sum(shape))
    U = _rand(rng, (n1, M, n2), cplx)
    V = _rand(rng, (n1, N, n2), cplx)
    bound = np.einsum("amb,anb->mn", np.abs(U), np.abs(V))
    Ut, Vt = torch.from_numpy(U).cuda(), torch.from_numpy(V).cuda()
    got = obs.rdm_reduce(Ut, Vt).cpu().numpy()
    assert np.all(np.abs(got - _ref(U, V)) <= 1e-13 * bound + 1e-300)
    if M == N:
        # U aliasing V: loaded once, same bits as two distinct copies
        alias = obs.rdm_reduce(Ut, Ut).cpu().numpy()
        assert np.all(np.abs(alias - _ref(U, U)) <= 1e-13 * np.einsum(
            "amb,anb->mn", np.abs(U), np.abs(U)) + 1e-300)
        two = obs.rdm_reduce(Ut, Ut.clone()).cpu().numpy()
        assert np.array_equal(alias.view(np.uint8), two.view(np.uint8))
    # permuted, non-contiguous views of the same values
    Up = torch.from_numpy(np.ascontiguousarray(U.transpose(2, 0, 1))).cuda().permute(1, 2, 0)
    Vp = torch.from_numpy(np.ascontiguousarray(V.transpose(1, 2, 0))).cuda().permute(2, 0, 1)
    gp = obs.rdm_reduce(Up, Vp).cpu().numpy()
    assert np.all(np.abs(gp - _ref(U, V)) <= 1e-13 * bound + 1e-300)


def test_raw_kernel_strided_slices():
    rng = np.random.default_rng(3)
    big = torch.from_numpy(_rand(rng, (42, 10, 32), True)).cuda()
    U, V = big[::3, 1:7:2, ::4], big[1::3, 0:4, 1::4]        # (14, 3, 8), (14, 4, 8)
    want = _ref(U.cpu().numpy(), V.cpu().numpy())
    got = obs.rdm_reduce(U, V).cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-12)


def _bits(x):
    return x.cpu().numpy().view(np.uint8).copy()


def test_raw_kernel_bitwise_reproducible():
    rng = np.random.default_rng(5)
    U = torch.from_numpy(_rand(rng, (700, 4, 900), True)).cuda()
    V = torch.from_numpy(_rand(rng, (700, 4, 900), True)).cuda()
    alone = _bits(obs.rdm_reduce(U, V))
    # after unrelated work
    junk = torch.randn(2048, 2048, dtype=torch.float64, device="cuda")
    _ = junk @ junk
    assert np.array_equal(_bits(obs.rdm_reduce(U, V)), alone)
    # on a second stream
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        out = obs.rdm_reduce(U, V)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(out), alone)
    # inside a replayed CUDA graph
    from quimb_b200.contract import capture_graph
    graph, out, _scratch = capture_graph(lambda: obs.rdm_reduce(U, V))
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert np.array_equal(_bits(out), alone)


def test_raw_kernel_propagates_nan_and_inf():
    rng = np.random.default_rng(6)
    U = _rand(rng, (300, 3, 200), False)
    V = _rand(rng, (300, 2, 200), False)
    U[17, 1, 33] = np.nan
    V[250, 0, 199] = np.inf
    got = obs.rdm_reduce(torch.from_numpy(U).cuda(), torch.from_numpy(V).cuda()).cpu().numpy()
    assert np.isnan(got[1]).all()
    assert not np.isfinite(got[:, 0]).any()
    assert np.isfinite(got[[0, 2], 1]).all()


def _call(dtype, n1, M, N, n2, U, us, V, vs, out, ws, nbytes):
    lib = _lib.load()
    arr = ctypes.c_int64 * 3
    return lib.qb_rdm_reduce(dtype, n1, M, N, n2, U, None if us is None else arr(*us), V,
                             None if vs is None else arr(*vs), out, ws, nbytes,
                             _lib.stream_ptr())


def test_raw_kernel_error_codes_launch_nothing():
    x = torch.zeros(4096, dtype=torch.complex128, device="cuda")
    p = x.data_ptr()
    ws_need = _lib.load().qb_rdm_workspace(1024, 2, 2, 1024)
    assert ws_need > 0
    F, C = _lib.QB_F64, _lib.QB_C128
    s = (4, 2, 1)
    n0 = _lib.launch_count()
    for rc, args in (
        (-1, (_lib.QB_F32, 1, 2, 2, 1, p, s, p, s, p, None, 0)),
        (-2, (F, 1, 65, 2, 1, p, s, p, s, p, None, 0)),
        (-2, (F, 1, 2, 0, 1, p, s, p, s, p, None, 0)),
        (-3, (F, 0, 2, 2, 1, p, s, p, s, p, None, 0)),
        (-3, (F, 1, 2, 2, 0, p, s, p, s, p, None, 0)),
        (-4, (F, 1, 2, 2, 1, None, s, p, s, p, None, 0)),
        (-4, (C, 1, 2, 2, 1, p + 8, s, p, s, p, None, 0)),
        (-4, (F, 1, 2, 2, 1, p, None, p, s, p, None, 0)),
        (-4, (F, 1, 2, 2, 1, p, s, p, s, None, None, 0)),
        (-6, (F, 1024, 2, 2, 1024, p, s, p, s, p, p, ws_need - 1)),
        (-6, (F, 1024, 2, 2, 1024, p, s, p, s, p, None, ws_need)),
    ):
        assert _call(*args) == rc, args
        assert _lib.last_error()
    assert _lib.launch_count() == n0
    assert _lib.load().qb_rdm_workspace(1, 65, 1, 1) == -2
    assert _lib.load().qb_rdm_workspace(0, 1, 1, 1) == -3


@pytest.mark.parametrize("shape", [(7, 3, 3, 5), (1024, 2, 2, 1024)])
def test_raw_kernel_at_most_two_launches(shape):
    n1, M, N, n2 = shape
    U = torch.randn(n1, M, n2, dtype=torch.float64, device="cuda")
    n0 = _lib.launch_count()
    obs.rdm_reduce(U, U)
    assert 1 <= _lib.launch_count() - n0 <= 2
