"""GPU tier of PEPS local expectations (quimb_b200/peps_expec.py,
csrc/plaquette.cu): the term kernel against numpy einsum, the whole path
against what the unmodified reference computed (tests/golden/peps_expec.*),
against the numpy oracle (oracle/peps_expec_np.py) at sizes the fixtures do
not reach (5x5 and 4x6 with D = 3 and boundaries of 12-16, where the numpy
oracle still runs in seconds), and against the dense state; the device path
alone at 6x6, D = 4, chi = 64 with a bound on its peak allocation.

Tolerance rule (as tests/test_gpu_boundary_oracle.py): a truncated boundary
is a deterministic function of the input only while every kept rank is
decided away from rounding, so the oracle's smallest recorded relative gap
must be at least 1e-6 (the seeds are chosen so); the device is then held to
the oracle at 1e-8 relative on the sum and on every ``return_all`` entry.
Single-precision PEPS are widened on entry and held to the widened oracle."""

import itertools

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from oracle import peps_expec_np as pe
from quimb_b200 import _lib
from quimb_b200 import peps_expec as px
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu

MIN_GAP = 1e-6
TOL = 1e-8


def _close(got, want, tol):
    got, want = complex(got), complex(want)
    assert abs(got - want) <= tol * max(1.0, abs(want)), (got, want)


# --------------------------------------------------------------- fixtures ---
def golden_state(data, meta, name):
    st = meta["states"][name]
    arrays = [[data[f"{name}__site{i}_{j}"] for j in range(st["Ly"])] for i in range(st["Lx"])]
    keys = [tuple(k[0]) if len(k) == 1 else tuple(map(tuple, k)) for k in st["keys"]]
    terms = {k: data[f"{name}__G{n}"] for n, k in enumerate(keys)}
    return arrays, terms, keys


def _ref_tol(st):
    return 2e-5 if st["dtype"] in ("complex64", "float32") else 1e-10


def test_golden_matches_reference():
    data, meta = load_golden("peps_expec")
    for rec in meta["runs"]:
        st = meta["states"][rec["state"]]
        arrays, terms, keys = golden_state(data, meta, rec["state"])
        dev = [[qb.asarray(a) for a in row] for row in arrays]
        got = qb.peps_compute_local_expectation(dev, terms, **rec["kw"])
        tol = _ref_tol(st)
        if rec["kw"].get("return_all"):
            assert set(got) == set(keys)
            for where, (e, n) in zip(keys, rec["values"]):
                _close(got[where][0], complex(*e), tol)
                if n is None:
                    assert got[where][1] is None
                else:
                    _close(got[where][1], complex(*n), tol)
        else:
            _close(got, complex(*rec["value"]), tol)
            if st["dtype"] in ("float64", "float32"):
                assert isinstance(got, float)


def test_golden_normalize():
    data, meta = load_golden("peps_expec")
    for name, st in meta["states"].items():
        arrays, _, _ = golden_state(data, meta, name)
        for rec in st["normalize"]:
            mb = rec["max_bond"]
            out = qb.peps_normalize([[qb.asarray(a) for a in row] for row in arrays],
                                    max_bond=mb, cutoff=0.0)
            tol = _ref_tol(st)
            for i, j in itertools.product(range(st["Lx"]), range(st["Ly"])):
                want = data[f"{name}__norm{mb}_site{i}_{j}"]
                got = out[i][j].to_numpy()
                assert got.dtype == want.dtype
                np.testing.assert_allclose(got, want, rtol=tol, atol=tol * np.abs(want).max())


# ------------------------------------------------------------- the kernel ---
def _einsum_expec(rho, dims, G, pos):
    """Tr[G rho] over the term sites ``pos`` (others traced) and Tr[rho]."""
    n = len(dims)
    ket = list(range(n))
    bra = [n + s if s in pos else s for s in range(n)]
    gin = [s for s in pos]
    gout = [n + s for s in pos]
    tdims = [dims[s] for s in pos]
    e = np.einsum(G.reshape(tdims + tdims), gout + gin, rho.reshape(dims + dims), ket + bra, [])
    return e, np.trace(rho)


def _rand(rng, shape, cplx):
    x = rng.standard_normal(shape)
    return x + 1j * rng.standard_normal(shape) if cplx else x


def _plaquette_shapes():
    out = []
    for ns in range(1, 7):
        for d in (2, 3, 4):
            if d ** ns <= 64:
                out.append((d,) * ns)
    return out + [(2, 3), (3, 2, 2), (4, 2, 2, 2), (2, 4, 3)]


def _kernel_case(rng, cplx, shapes):
    rhos, items, want = [], [], []
    off = 0
    offsets = []
    for k, dims in enumerate(shapes):
        D = int(np.prod(dims))
        rho = _rand(rng, (D, D), cplx)
        rhos.append(rho.ravel())
        offsets.append(off)
        off += D * D
        subsets = [(s,) for s in range(len(dims))] + list(itertools.combinations(range(len(dims)), 2))
        for pos in subsets:
            dg = int(np.prod([dims[s] for s in pos]))
            G = _rand(rng, (dg, dg), cplx)
            items.append((k, list(dims), G, pos))
            want.append(_einsum_expec(rho, list(dims), G, pos))
    buf = torch.from_numpy(np.concatenate(rhos)).to("cuda")
    return buf, offsets, items, want


@pytest.mark.parametrize("cplx", [False, True])
def test_kernel_against_einsum(cplx):
    rng = np.random.default_rng(1 + cplx)
    buf, offsets, items, want = _kernel_case(rng, cplx, _plaquette_shapes())
    got = px.plaquette_expec(buf, offsets, items)
    assert len(got) == len(want)
    for (e, n), (we, wn) in zip(got, want):
        assert abs(e - we) <= 1e-12 * max(1.0, np.abs(buf.cpu().numpy()).max() * 64)
        assert abs(n - wn) <= 1e-12 * 64 * max(1.0, abs(wn))


@pytest.mark.parametrize("cplx", [False, True])
def test_kernel_single_and_many_terms(cplx):
    rng = np.random.default_rng(7)
    buf, offsets, items, want = _kernel_case(rng, cplx, [(2, 2)])
    one = px.plaquette_expec(buf, offsets, items[:1])
    assert abs(one[0][0] - want[0][0]) <= 1e-12 * 16
    shapes = [_plaquette_shapes()[k % 13] for k in range(1700)]
    buf, offsets, items, want = _kernel_case(rng, cplx, shapes)
    assert len(items) >= 10_000
    got = px.plaquette_expec(buf, offsets, items)
    err = max(abs(e - we) / max(1.0, abs(we)) for (e, _), (we, _) in zip(got, want))
    assert err <= 1e-11


def test_kernel_nonfinite_stays_in_its_term():
    rng = np.random.default_rng(3)
    buf, offsets, items, want = _kernel_case(rng, True, [(2, 2, 2), (3, 3)])
    clean = px.plaquette_expec(buf, offsets, items)
    for bad in (np.nan, np.inf):
        k = 5
        poisoned = list(items)
        G = poisoned[k][2].copy()
        G[0, 0] = bad
        poisoned[k] = poisoned[k][:2] + (G,) + poisoned[k][3:]
        got = px.plaquette_expec(buf, offsets, poisoned)
        for t, ((e, n), (ce, cn)) in enumerate(zip(got, clean)):
            if t == k:
                assert not np.isfinite(e)
            else:
                assert e == ce and n == cn


def test_kernel_bits_repeat_and_side_stream():
    rng = np.random.default_rng(5)
    buf, offsets, items, _ = _kernel_case(rng, True, _plaquette_shapes())
    a = px.plaquette_expec(buf, offsets, items)
    b = px.plaquette_expec(buf, offsets, items)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c = px.plaquette_expec(buf, offsets, items)
    torch.cuda.current_stream().wait_stream(side)
    for x, y, z in zip(a, b, c):
        assert x[0] == y[0] == z[0] and x[1] == y[1] == z[1]


def test_kernel_rejects_without_launch():
    import ctypes
    lib = _lib.load()
    rho = torch.zeros(64 * 64 + 1, dtype=torch.float64, device="cuda")
    G = torch.zeros(16 * 16, dtype=torch.float64, device="cuda")
    out = torch.zeros(2, dtype=torch.float64, device="cuda")
    ddev = torch.zeros(_lib.QB_PLAQ_DESC_WORDS, dtype=torch.int64, device="cuda")

    def call(row, dtype=_lib.QB_F64, rho_ptr=None, n=1):
        table = np.array(row + [1] * (12 - len(row)), dtype=np.int64)
        return lib.qb_plaquette_expec(
            dtype, n, table.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), ddev.data_ptr(),
            rho.data_ptr() if rho_ptr is None else rho_ptr, rho.numel(), G.data_ptr(),
            G.numel(), out.data_ptr(), _lib.stream_ptr())

    n0 = qb.launch_count()
    assert call([0, 0, 2, 2, 0, 1, 2, 2]) == 0
    assert qb.launch_count() == n0 + 1
    n0 = qb.launch_count()
    ok = [0, 0, 2, 2, 0, 1, 2, 2]
    bad = [  # (descriptor row, dtype, rho pointer, n_terms, expected code)
        (ok, _lib.QB_C64, None, 1, -1),
        (ok, _lib.QB_F64, None, -1, -2),
        ([0, 0, 7, 1, 0, 0], _lib.QB_F64, None, 1, -3),          # 7 sites
        ([0, 0, 2, 2, 1, 0, 2, 2], _lib.QB_F64, None, 1, -3),    # positions reversed
        ([0, 0, 2, 2, 0, 0, 2, 2], _lib.QB_F64, None, 1, -3),    # a site twice
        ([0, 0, 3, 1, 0, 0, 4, 4, 5], _lib.QB_F64, None, 1, -3), # D = 80
        ([2, 0, 3, 1, 0, 0, 4, 4, 4], _lib.QB_F64, None, 1, -3), # rho overrun
        ([0, 250, 2, 2, 0, 1, 2, 2], _lib.QB_F64, None, 1, -3),  # G overrun
        (ok, _lib.QB_F64, rho.data_ptr() + 4, 1, -4),            # misaligned
    ]
    for row, dt, ptr, n, rc in bad:
        assert call(row, dt, ptr, n) == rc, (row, dt, n)
    assert qb.launch_count() == n0


# -------------------------------------------------------- the whole path ---
def check_against_oracle(Lx, Ly, D, d, seed, dtype, chi, terms_kw, first_contract,
                         normalized=True):
    arrays = pe.rand_peps(Lx, Ly, D, d, seed, dtype)
    terms = pe.heis_terms(Lx, Ly, d, seed=seed, **terms_kw)
    terms = {k: np.asarray(v, dtype=np.result_type(dtype, np.float64)) for k, v in terms.items()}
    want, trace = pe.compute_local_expectation(arrays, terms, chi, cutoff=0.0,
                                               normalized=normalized, return_all=True,
                                               first_contract=first_contract, per_term=False)
    assert pe.min_gap(trace) >= MIN_GAP, pe.min_gap(trace)
    dev = [[qb.asarray(a) for a in row] for row in arrays]
    got = qb.peps_compute_local_expectation(dev, terms, chi, cutoff=0.0, normalized=normalized,
                                            return_all=True, first_contract=first_contract)
    assert list(got) == list(want)
    for where in want:
        _close(got[where][0], want[where][0], TOL)
        if normalized:
            _close(got[where][1], want[where][1], TOL)
    total = qb.peps_compute_local_expectation(dev, terms, chi, cutoff=0.0, normalized=normalized,
                                              first_contract=first_contract)
    ref = sum((e / n if normalized else e) for e, n in want.values())
    _close(total, ref, TOL)
    return trace


@pytest.mark.parametrize("first_contract", ["x", "y"])
def test_oracle_5x5_d3_chi16_complex(first_contract):
    check_against_oracle(5, 5, 3, 2, 21, np.complex128, 16, dict(field=0.3, nnn=0.5, long=0.2),
                         first_contract)


@pytest.mark.parametrize("first_contract", ["x", "y"])
def test_oracle_4x6_d3_chi12_real(first_contract):
    check_against_oracle(4, 6, 3, 2, 22, np.float64, 12, dict(field=0.2, nnn=0.4, long=0.3),
                         first_contract, normalized=False)


def test_6x6_d4_chi64_memory():
    """At 6x6, D = 4, chi = 64 (complex128, diagonal and 1 x 3 terms) every
    plaquette's env . ket network is cut site by site: the call stays within
    a few GB (a K-hub tree would hold 69 GB for one 2 x 2 plaquette).  The
    numpy oracle takes too long here to sit in this tier; the values are
    held to be finite and the local norms positive."""
    arrays = pe.rand_peps(6, 6, 4, 2, 21, np.complex128)
    arrays = [[a / np.sqrt(a.size / 2) for a in row] for row in arrays]
    terms = pe.heis_terms(6, 6, 2, seed=21, field=0.3, nnn=0.5, long=0.2)
    dev = [[qb.asarray(a) for a in row] for row in arrays]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got = qb.peps_compute_local_expectation(dev, terms, 64, cutoff=0.0, normalized=True,
                                            return_all=True)
    peak = torch.cuda.max_memory_allocated() - base
    print(f"6x6 D=4 chi=64: peak allocation {peak / 2**30:.2f} GiB")
    assert peak < 8 * 2**30
    assert set(got) == set(terms)
    for e, n in got.values():
        assert np.isfinite(e) and np.isfinite(n) and n.real > 0


def test_oracle_complex64_widened():
    check_against_oracle(4, 5, 3, 2, 23, np.complex64, 16, dict(field=0.3, nnn=0.2), None)


def test_dense_state_without_truncation():
    arrays = pe.rand_peps(3, 4, 2, 2, 31, np.complex128)
    terms = pe.heis_terms(3, 4, 2, field=0.3, nnn=0.5, long=0.2, seed=31)
    dev = [[qb.asarray(a) for a in row] for row in arrays]
    for normalized in (False, True):
        for fc in ("x", "y"):
            got = qb.peps_compute_local_expectation(dev, terms, 256, cutoff=0.0,
                                                    normalized=normalized, first_contract=fc)
            _close(got, pe.dense_expectation(arrays, terms, normalized), 1e-10)


@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_normalize_against_oracle(dtype):
    """The normalized PEPS matches the oracle; its boundary norm at the same
    chi is nfact / |nfact|: 1 for a real state, a phase of modulus 1 when
    truncation leaves the complex nfact slightly off the real axis (as in
    the reference, which scales the ket by the complex nfact ** (-1/2N))."""
    arrays = pe.rand_peps(5, 5, 3, 2, 41, dtype)
    want, _ = pe.normalize(arrays, max_bond=32, cutoff=0.0)
    dev = [[qb.asarray(a) for a in row] for row in arrays]
    out = qb.peps_normalize(dev, max_bond=32, cutoff=0.0)
    for r1, r2 in zip(out, want):
        for a, b in zip(r1, r2):
            np.testing.assert_allclose(a.to_numpy(), b, rtol=1e-10, atol=1e-10 * np.abs(b).max())
    n = qb.contract_boundary(qb.peps_norm_tensors(out)[0], 5, 5, 32, cutoff=0.0,
                             layer_tags=("KET", "BRA"))
    assert abs(abs(n) - 1) <= 1e-10
    if dtype == np.float64:
        assert abs(n - 1) <= 1e-10
