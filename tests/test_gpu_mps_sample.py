"""GPU tier: batched MPS sampling (``mps_sample`` / ``mps_sample_configuration``
and the ``qb_sample_select`` kernel).

The reference's draws are the doubles of ``rng.random((C, L))`` in row-major
order, so configurations are compared EXACTLY: against what the unmodified
reference yielded (tests/golden/sample.*) and against the numpy oracle
(oracle/sample_np.py) at larger sizes, each time with the oracle's margin
(distance of every uniform from every cdf boundary) asserted well above
rounding.  The raw kernel is checked to the bit against a numpy restatement
of its arithmetic."""

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from quimb_b200 import _lib, mps, tebd as tb
from oracle import sample_np
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------- helpers ---
def _golden_sites(data, meta, name):
    info = meta[name]
    n = info["L"]
    return [np.ascontiguousarray(mps.site_lpr(data[f"{name}__site{i}"], lay, i, n).to_numpy())
            for i, lay in enumerate(info["layouts"])]


def _device(sites):
    return [qb.asarray(a) for a in sites]


def rand_mps(L, chi, d, dtype, seed):
    """Random open-boundary (l, p, r) host arrays with ragged bonds <= chi."""
    rng = np.random.default_rng(seed)
    bonds = [1]
    for i in range(1, L):
        b = min(chi, d ** min(i, 12), d ** min(L - i, 12))
        if 2 < b:
            b -= int(rng.integers(0, min(b - 1, 6)))
        bonds.append(b)
    bonds.append(1)
    out = []
    for i in range(L):
        shape = (bonds[i], d, bonds[i + 1])
        x = rng.standard_normal(shape)
        if np.dtype(dtype).kind == "c":
            x = x + 1j * rng.standard_normal(shape)
        out.append((x / np.sqrt(bonds[i] * d)).astype(dtype))
    return out


def _dense(sites):
    v = np.ones((1, 1))
    for a in sites:
        l, d, r = a.shape
        v = (v @ a.reshape(l, d * r)).reshape(-1, r)
    return v.reshape(-1)


# ------------------------------------------------------------------ golden ---
def test_golden_matches_reference():
    data, meta = load_golden("sample")
    for k, case in enumerate(meta["cases"]):
        assert min(case["margins"]) > 1e-9, case
        sites = _device(_golden_sites(data, meta, case["state"]))
        before = [s.to_numpy().copy() for s in sites]
        parts = []
        if case["kind"] == "configuration":
            cfg, om = tb.mps_sample_configuration(sites, seed=case["seed"])
            assert isinstance(cfg, list) and all(type(x) is int for x in cfg)
            assert isinstance(om, float)
            parts.append((np.array([cfg]), np.array([om])))
        elif case["kind"] == "sample":
            parts.append(tb.mps_sample(sites, case["C"][0], seed=case["seed"]))
        else:
            # two consecutive calls on one Generator continue its stream
            rng = np.random.default_rng(case["seed"])
            for c in case["C"]:
                parts.append(tb.mps_sample(sites, c, seed=rng))
        for j, (cfgs, oms) in enumerate(parts):
            key = f"case{k}__part{j}"
            assert cfgs.dtype == np.int64 and oms.dtype == np.float64
            np.testing.assert_array_equal(cfgs, data[key + "__configs"], err_msg=key)
            np.testing.assert_allclose(oms, data[key + "__omegas"], rtol=1e-12, atol=0)
        for a, b in zip(sites, before):
            assert np.array_equal(a.to_numpy(), b)


def test_device_generator_seed():
    """A quimb_b200.random.default_rng generator is unwrapped to its numpy
    Generator and advanced like one."""
    sites = rand_mps(8, 6, 2, np.float64, seed=1)
    g = qb.random.default_rng(4)
    c1, o1 = tb.mps_sample(_device(sites), 30, seed=g)
    c2, o2 = tb.mps_sample(_device(sites), 30, seed=g)
    rng = np.random.default_rng(4)
    r1, q1, m1 = sample_np.sample(sites, 30, seed=rng)
    r2, q2, m2 = sample_np.sample(sites, 30, seed=rng)
    assert min(m1, m2) > 1e-9
    np.testing.assert_array_equal(c1, r1)
    np.testing.assert_array_equal(c2, r2)
    np.testing.assert_allclose(np.concatenate([o1, o2]), np.concatenate([q1, q2]), rtol=1e-12)


# ------------------------------------------------------------------ oracle ---
def check_against_oracle(L, chi, C, dtype, d, seed, rtol=1e-12):
    sites = rand_mps(L, chi, d, dtype, seed)
    cfgs, oms = tb.mps_sample(_device(sites), C, seed=seed + 100)
    rc, ro, margin = sample_np.sample(sites, C, seed=seed + 100)
    assert margin > 1e-11, margin
    np.testing.assert_array_equal(cfgs, rc)
    np.testing.assert_allclose(oms, ro, rtol=rtol, atol=0)


@pytest.mark.parametrize("dtype,d", [(np.float64, 2), (np.complex128, 2),
                                     (np.float64, 4), (np.complex128, 4)])
def test_matches_oracle_large(dtype, d):
    # both sides are fp64 GEMMs with different summation orders: the
    # selected row of an outcome of probability p carries a relative rounding
    # error of about eps * sqrt(chi / p), and omega multiplies 40 of them (the
    # worst of the 4 x 4096 samples measured 1.2e-12 on the H100)
    check_against_oracle(40, 256, 4096, dtype, d, seed=7 + d, rtol=4e-12)


def test_omega_is_normalised_amplitude_squared():
    sites = rand_mps(10, 8, 2, np.complex128, seed=21)
    dev = _device(sites)
    cfgs, oms = tb.mps_sample(dev, 40, seed=3)
    psi = _dense(sites)
    norm2 = np.vdot(psi, psi).real
    for cfg, om in zip(cfgs, oms):
        amp = tb.mps_amplitude(dev, cfg)
        np.testing.assert_allclose(om, abs(amp) ** 2 / norm2, rtol=1e-12)


def test_chunked_run_is_identical(monkeypatch):
    sites = _device(rand_mps(12, 32, 2, np.float64, seed=5))
    c1, o1 = tb.mps_sample(sites, 1000, seed=9)
    # at most 32 * 2 * 8 bytes of W per sample: chunks of at least 37 samples
    monkeypatch.setattr(tb, "SAMPLE_CHUNK_BYTES", 37 * 512 + 100)
    c2, o2 = tb.mps_sample(sites, 1000, seed=9)
    np.testing.assert_array_equal(c1, c2)
    np.testing.assert_allclose(o1, o2, rtol=1e-14, atol=0)


@pytest.mark.parametrize("factor", [1e200, 1e-200])
def test_badly_scaled_state_gives_the_same_samples(factor):
    sites = rand_mps(10, 8, 2, np.complex128, seed=11)
    c0, o0 = tb.mps_sample(_device(sites), 300, seed=2)
    scaled = [a.copy() for a in sites]
    scaled[4] = scaled[4] * factor
    dev = _device(scaled)
    before = [s.to_numpy().copy() for s in dev]
    c1, o1 = tb.mps_sample(dev, 300, seed=2)
    np.testing.assert_array_equal(c0, c1)
    np.testing.assert_allclose(o0, o1, rtol=1e-12)
    for a, b in zip(dev, before):
        assert a.to_numpy().tobytes() == b.tobytes()


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
def test_single_precision_is_widened(dtype):
    sites = rand_mps(9, 8, 2, dtype, seed=13)
    cfgs, oms = tb.mps_sample(_device(sites), 200, seed=6)
    wide = [a.astype(np.result_type(a.dtype, np.float64)) for a in sites]
    rc, ro, margin = sample_np.sample(wide, 200, seed=6)
    assert margin > 1e-9
    np.testing.assert_array_equal(cfgs, rc)
    np.testing.assert_allclose(oms, ro, rtol=1e-12)


def test_argument_errors_and_empty_request():
    sites = rand_mps(5, 4, 2, np.float64, seed=2)
    with pytest.raises(TypeError):
        tb.mps_sample([qb.asarray(np.ones(a.shape, dtype=np.int64)) for a in sites], 3)
    periodic = [np.ones((2, 2, 2)) for _ in range(4)]
    with pytest.raises(ValueError):
        tb.mps_sample(_device(periodic), 3)
    n0 = qb.launch_count()
    cfgs, oms = tb.mps_sample(_device(sites), 0, seed=1)
    assert qb.launch_count() == n0
    assert cfgs.shape == (0, 5) and cfgs.dtype == np.int64
    assert oms.shape == (0,) and oms.dtype == np.float64
    zero = [np.zeros_like(a) for a in sites]
    with pytest.raises(ValueError):
        tb.mps_sample(_device(zero), 4, seed=1)


def test_qudits_and_product_state():
    check_against_oracle(9, 20, 500, np.complex128, 3, seed=31)
    bits = [0, 1, 1, 0, 1, 0, 0, 1]
    prod = []
    for b in bits:
        x = np.zeros((1, 2, 1))
        x[0, b, 0] = 1.0
        prod.append(x)
    cfgs, oms = tb.mps_sample(_device(prod), 50, seed=1)
    assert (cfgs == np.array(bits)).all()
    assert (oms == 1.0).all()


# ------------------------------------------------------------ raw C ABI -----
def select_reference(W, u, omega):
    """numpy restatement of qb_sample_select's arithmetic, bit for bit."""
    C, d, r = W.shape
    a2 = W.real * W.real + W.imag * W.imag if np.iscomplexobj(W) else W * W
    nb = -(-r // 32)
    pad = np.zeros((C, d, nb * 32))
    pad[:, :, :r] = a2
    lanes = pad.reshape(C, d, nb, 32)
    acc = np.zeros((C, d, 32))
    for b in range(nb):
        acc = acc + lanes[:, :, b, :]
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, :, idx ^ o]
    pi = acc[:, :, 0]
    cfg = np.full(C, -1, dtype=np.int64)
    om = np.full(C, np.nan)
    V = np.zeros((C, r), dtype=W.dtype)
    for c in range(C):
        tot = np.sum(pi[c])
        if not (tot > 0 and np.isfinite(tot) and 0.0 <= u[c] < 1.0):
            continue
        p = pi[c] / tot
        cdf = np.cumsum(p)
        cdf /= cdf[-1]
        x = int(np.sum(cdf <= u[c]))
        cfg[c] = x
        om[c] = omega[c] * p[x]
        s = np.sqrt(pi[c, x])
        if np.iscomplexobj(W):
            V[c] = W[c, x].real / s + 1j * (W[c, x].imag / s)
        else:
            V[c] = W[c, x] / s
    return cfg, om, V


_GUARD = 64


def _guarded(n, dtype, fill):
    """Device buffer of n elements inside sentinel guards."""
    buf = torch.full((n + 2 * _GUARD,), fill, dtype=dtype, device="cuda") \
        if not dtype.is_complex else \
        torch.full((n + 2 * _GUARD,), complex(fill, fill), dtype=dtype, device="cuda")
    return buf, buf[_GUARD:_GUARD + n]


def run_select(W, u, omega, ldu=1, ldc=1, expect_rc=0):
    """qb_sample_select on device copies of host arrays; checks that nothing
    outside the outputs (guards, the unused strides of u / config) moved."""
    C, d, r = W.shape
    tdt = torch.complex128 if np.iscomplexobj(W) else torch.float64
    Wd = torch.from_numpy(np.ascontiguousarray(W)).cuda()
    ub, uv = _guarded(max((C - 1) * ldu + 1, 1), torch.float64, -7.0)
    if C:
        uv[::ldu] = torch.from_numpy(np.asarray(u, dtype=np.float64)).cuda()
    cb, cv = _guarded(max((C - 1) * ldc + 1, 1), torch.int64, -12345)
    ob, ov = _guarded(C, torch.float64, 0.0)
    ov.copy_(torch.from_numpy(np.asarray(omega, dtype=np.float64)).cuda())
    vb, vv = _guarded(C * r, tdt, 99.0)
    snap = [x.cpu().clone() for x in (ub, cb, ob, vb)]
    rc = _lib.load().qb_sample_select(
        _lib.QB_C128 if tdt.is_complex else _lib.QB_F64, C, d, r, Wd.data_ptr(),
        uv.data_ptr(), ldu, cv.data_ptr(), ldc, ov.data_ptr(), vv.data_ptr(),
        _lib.stream_ptr())
    torch.cuda.synchronize()
    assert rc == expect_rc, _lib.last_error()
    after = [x.cpu() for x in (ub, cb, ob, vb)]
    g = slice(None, _GUARD), slice(-_GUARD, None)
    for s, a in zip(snap, after):
        for sl in g:
            assert torch.equal(s[sl], a[sl])
    assert torch.equal(snap[0], after[0])                        # u is read only
    cfull = after[1][_GUARD:-_GUARD]
    if ldc > 1 and C:
        mask = torch.ones_like(cfull, dtype=torch.bool)
        mask[::ldc] = False
        assert (cfull[mask] == -12345).all()
    if rc != 0:
        for s, a in zip(snap, after):
            assert torch.equal(s, a)
        return None
    cfg = cfull[::ldc].numpy().copy() if C else np.empty(0, np.int64)
    om = after[2][_GUARD:-_GUARD].numpy().copy()
    V = after[3][_GUARD:-_GUARD].numpy().reshape(C, r).copy()
    return cfg, om, V


def _assert_bits(got, want):
    cfg, om, V = got
    rc, ro, rv = want
    np.testing.assert_array_equal(cfg, rc)
    assert np.array_equal(om.view(np.int64)[~np.isnan(om)], ro.view(np.int64)[~np.isnan(ro)])
    assert np.array_equal(np.isnan(om), np.isnan(ro))
    assert V.tobytes() == rv.tobytes()


def _rand_W(rng, C, d, r, cplx):
    W = rng.standard_normal((C, d, r))
    if cplx:
        W = W + 1j * rng.standard_normal((C, d, r))
    return W


def test_raw_select_cdf_boundary_and_zero_probabilities():
    # pi = [1, 1, 1, 1]: cdf = [.25, .5, .75, 1] exactly; u on a boundary
    # picks the next outcome (searchsorted side='right')
    W = np.ones((5, 4, 1))
    u = np.array([0.0, 0.25, 0.5, 0.75, 0.7499999999999999])
    got = run_select(W, u, np.ones(5))
    assert got[0].tolist() == [0, 1, 2, 3, 2]
    _assert_bits(got, select_reference(W, u, np.ones(5)))
    # zero-probability outcomes are never chosen, even at u = 0 or on their
    # (repeated) cdf value
    W = np.zeros((4, 5, 3))
    W[:, 1] = 1.0
    W[:, 3] = 1.0
    u = np.array([0.0, 0.5, 0.4999999, 0.9999999999])
    got = run_select(W, u, np.full(4, 0.5))
    assert got[0].tolist() == [1, 3, 1, 3]
    _assert_bits(got, select_reference(W, u, np.full(4, 0.5)))


@pytest.mark.parametrize("d", [1, 2, 37])
@pytest.mark.parametrize("r", [1, 31, 33, 1000])
@pytest.mark.parametrize("cplx", [False, True])
def test_raw_select_bits(d, r, cplx):
    rng = np.random.default_rng(d * 1000 + r + cplx)
    C = 70
    W = _rand_W(rng, C, d, r, cplx) * 10.0 ** rng.integers(-3, 3, (C, 1, 1))
    u = rng.random(C)
    om = rng.random(C)
    _assert_bits(run_select(W, u, om), select_reference(W, u, om))


def test_raw_select_strided_bad_rows_and_limits():
    rng = np.random.default_rng(3)
    C, d, r = 40, 3, 45
    W = _rand_W(rng, C, d, r, True)
    W[5] = 0.0                       # zero row: sum(pi) == 0
    W[9, 1, 7] = np.nan              # NaN row
    W[11, 0, 0] = np.inf             # infinite row
    u = rng.random(C)
    u[13] = 1.0                      # never drawn: outside [0, 1)
    om = np.ones(C)
    got = run_select(W, u, om, ldu=5, ldc=3)
    want = select_reference(W, u, om)
    _assert_bits(got, want)
    for c in (5, 9, 11, 13):
        assert got[0][c] == -1 and np.isnan(got[1][c]) and not got[2][c].any()
    # d above the shared-memory layout: rejected, nothing written
    assert run_select(np.ones((3, 257, 2)), np.zeros(3), np.ones(3), expect_rc=-3) is None
    assert "257" in _lib.last_error()
    assert run_select(np.ones((0, 2, 2)), np.zeros(0), np.ones(0)) is not None


def test_raw_select_row_alone_equals_row_in_batch():
    rng = np.random.default_rng(17)
    C, d, r = 4096, 2, 200
    W = _rand_W(rng, C, d, r, True)
    u = rng.random(C)
    om = rng.random(C)
    cfg, o, V = run_select(W, u, om)
    for c in (0, 1234, C - 1):
        c1, o1, v1 = run_select(W[c:c + 1], u[c:c + 1], om[c:c + 1])
        assert c1[0] == cfg[c] and o1.tobytes() == o[c:c + 1].tobytes()
        assert v1.tobytes() == V[c:c + 1].tobytes()


def test_sampling_loop_launch_count(monkeypatch):
    sites = _device(rand_mps(11, 16, 2, np.complex128, seed=8))
    psi, _ = tb._sample_prepare(sites)
    row_bytes = max(a.shape[1] * a.shape[2] for a in psi) * 16
    C, L = 400, len(psi)
    for budget in (1 << 30, 100 * row_bytes):
        monkeypatch.setattr(tb, "SAMPLE_CHUNK_BYTES", budget)
        want_chunks = -(-C // min(C, budget // row_bytes))
        dev = psi[0].t.device
        u = torch.from_numpy(np.random.default_rng(1).random((C, L))).to(dev)
        cfg = torch.empty((C, L), dtype=torch.int64, device=dev)
        om = torch.ones(C, dtype=torch.float64, device=dev)
        n0 = qb.launch_count()
        n_chunks = tb._sample_chunks(psi, u, cfg, om)
        assert n_chunks == want_chunks
        assert qb.launch_count() - n0 == 2 * L * n_chunks
