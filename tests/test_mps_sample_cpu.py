"""CPU tier of batched MPS sampling: the numpy oracle against what the
unmodified reference yielded, and the host layer of ``mps_sample`` (seeding,
canonicalisation, widening, chunking, pointer / stride plumbing of
``qb_sample_select``) run against a numpy emulation of the C ABI.  The test
bodies are those of tests/test_gpu_mps_sample.py; the raw-kernel and
launch-count tests need the device and are not repeated here."""

import numpy as np
import pytest

from oracle import sample_np
from tests import test_gpu_mps_sample as gpu
from tests.abi_emulator import _NP, _flat, emulated_abi
from tests.conftest import load_golden
from quimb_b200 import _lib


def _emulated_sample_select(emu, dtype, C, d, r, W, u, ldu, config, ldc, omega, V, stream):
    """numpy version of qb_sample_select (csrc/sample.cu), same contract."""
    if dtype not in (_lib.QB_F64, _lib.QB_C128):
        return emu._fail(-1, "qb_sample_select: dtype must be QB_F64 or QB_C128")
    if C < 0:
        return emu._fail(-2, "qb_sample_select: C < 0")
    if not 1 <= d <= 256:
        return emu._fail(-3, f"qb_sample_select: physical dimension d = {d} outside [1, 256]")
    if r < 1:
        return emu._fail(-4, "qb_sample_select: r < 1")
    if C == 0:
        return 0
    emu._tick("qb_sample_select")
    Wv = _flat(W, C * d * r, _NP[dtype]).reshape(C, d, r)
    uv = _flat(u, (C - 1) * ldu + 1, np.float64)[::ldu]
    cv = _flat(config, (C - 1) * ldc + 1, np.int64)[::ldc]
    ov = _flat(omega, C, np.float64)
    Vv = _flat(V, C * r, _NP[dtype]).reshape(C, r)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        pi = np.sum(np.abs(Wv) ** 2, axis=2)
        tot = pi.sum(axis=1)
        ok = (tot > 0) & np.isfinite(tot) & (uv >= 0) & (uv < 1)
        p = pi / tot[:, None]
        cdf = np.cumsum(p, axis=1)
        cdf /= cdf[:, -1:]
        x = np.where(ok, np.sum(cdf <= uv[:, None], axis=1), -1)
        rows = np.arange(C)
        xs = np.where(ok, x, 0)
        ov[...] = np.where(ok, ov * p[rows, xs], np.nan)
        cv[...] = x
        Vv[...] = np.where(ok[:, None], Wv[rows, xs] / np.sqrt(pi[rows, xs])[:, None], 0)
    return 0


@pytest.fixture
def emulator():
    with emulated_abi() as emu:
        emu.qb_sample_select = lambda *a: _emulated_sample_select(emu, *a)
        yield emu


def _lpr(x, lay):
    """(l, p, r) view of a site array in the reference's layout ``lay``."""
    for c in "lpr":
        if c not in lay:
            x = x[..., None]
            lay += c
    return np.transpose(x, [lay.index(c) for c in "lpr"])


def test_oracle_matches_reference():
    data, meta = load_golden("sample")
    for k, case in enumerate(meta["cases"]):
        info = meta[case["state"]]
        n = info["L"]
        psi = sample_np.prepare([_lpr(data[f"{case['state']}__site{i}"], lay)
                                 for i, lay in enumerate(info["layouts"])])
        rng = np.random.default_rng(case["seed"])
        for j, C in enumerate(case["C"]):
            key = f"case{k}__part{j}"
            cfgs, oms, margin = sample_np.sample_uniforms(psi, rng.random((C, n)))
            assert margin == pytest.approx(case["margins"][j], rel=1e-6)
            assert margin > 1e-9
            np.testing.assert_array_equal(cfgs, data[key + "__configs"])
            np.testing.assert_allclose(oms, data[key + "__omegas"], rtol=1e-12, atol=0)
            # the probabilities are those of the normalised state
            assert (oms > 0).all() and (oms <= 1).all()


def test_emu_golden(emulator):
    gpu.test_golden_matches_reference()
    assert emulator.calls["qb_sample_select"] > 0


def test_emu_device_generator_seed(emulator):
    gpu.test_device_generator_seed()


@pytest.mark.parametrize("dtype,d", [(np.float64, 2), (np.complex128, 2),
                                     (np.float64, 4), (np.complex128, 4)])
def test_emu_matches_oracle(emulator, dtype, d):
    gpu.check_against_oracle(16, 24, 300, dtype, d, seed=7 + d)


def test_emu_omega_is_normalised_amplitude_squared(emulator):
    gpu.test_omega_is_normalised_amplitude_squared()


def test_emu_chunked_run_is_identical(emulator, monkeypatch):
    gpu.test_chunked_run_is_identical(monkeypatch)
    assert emulator.calls["qb_sample_select"] > 12 * 20      # 12 sites, >= 20 chunks


@pytest.mark.parametrize("factor", [1e200, 1e-200])
def test_emu_badly_scaled_state(emulator, factor):
    gpu.test_badly_scaled_state_gives_the_same_samples(factor)


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
def test_emu_single_precision_is_widened(emulator, dtype):
    gpu.test_single_precision_is_widened(dtype)


def test_emu_argument_errors_and_empty_request(emulator):
    gpu.test_argument_errors_and_empty_request()


def test_emu_qudits_and_product_state(emulator):
    gpu.test_qudits_and_product_state()
