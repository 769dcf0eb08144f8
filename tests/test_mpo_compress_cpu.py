"""CPU tier of MPO application with compression: the numpy oracle against what
the unmodified reference computed, and the host layer (the four methods'
contraction and split sequences, the zip-up gauge, orientation, dtype and
argument handling) run against a numpy emulation of the C ABI.  The test
bodies are those of tests/test_gpu_mpo_compress.py."""

import numpy as np
import pytest

from oracle import mpo_compress_np as onp
from tests import test_gpu_mpo_compress as gpu
from tests.abi_emulator import emulated_abi
from tests.conftest import load_golden


@pytest.fixture
def emulator():
    with emulated_abi() as emu:
        yield emu


def test_oracle_matches_reference():
    data, meta = load_golden("mpo_compress")
    methods = set()
    for k, case in enumerate(meta["cases"]):
        A, W = gpu._inputs(data, meta, case)
        got = onp.gate_with_mpo(A, W, **gpu._kwargs(case))
        assert [x.shape[2] for x in got[:-1]] == case["bonds"]
        vec = data[f"case{k}__vec"]
        np.testing.assert_allclose(onp.dense(got), vec, rtol=0,
                                   atol=1e-10 * np.max(np.abs(vec)))
        for i, s in enumerate(onp.schmidt_values(got)):
            ref = data[f"case{k}__S{i}"]
            np.testing.assert_allclose(s, ref, rtol=0, atol=1e-10 * ref[0])
        methods.add(case["method"])
    assert methods == set(gpu.METHODS)


def test_fixtures_truncate_in_the_zipup_gauge():
    """Without the reference's pseudo-canonical gauge the zip-up fixtures are
    not reproduced: they pin the gauge, not just the method."""
    data, meta = load_golden("mpo_compress")
    worst = 0.0
    for k, case in enumerate(meta["cases"]):
        if case["method"] != "zipup" or case.get("max_bond") is None:
            continue
        A, W = gpu._inputs(data, meta, case)
        got = onp.gate_with_mpo(A, W, canonize=False, **gpu._kwargs(case))
        vec = data[f"case{k}__vec"]
        worst = max(worst, np.max(np.abs(onp.dense(got) - vec)) / np.max(np.abs(vec)))
    assert worst > 1e-3


def test_emu_golden(emulator):
    gpu.test_golden_matches_reference()
    assert emulator.calls["qb_contract_pair"] > 0


@pytest.mark.parametrize("method", gpu.METHODS)
def test_emu_matches_oracle(emulator, method):
    gpu.check_against_oracle(12, 16, 3, 2, np.complex128, method, seed=5)


@pytest.mark.parametrize("method", gpu.METHODS)
def test_emu_untruncated_equals_mpo_apply(emulator, method):
    gpu.test_untruncated_equals_mpo_apply(method)


@pytest.mark.parametrize("method", gpu.METHODS)
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_emu_canonical_form_and_info(emulator, method, sweep_reverse):
    gpu.test_canonical_form_and_info(method, sweep_reverse)


@pytest.mark.parametrize("method", gpu.METHODS)
def test_emu_inputs_unchanged(emulator, method):
    gpu.test_inputs_unchanged(method)


@pytest.mark.parametrize("method", gpu.METHODS)
@pytest.mark.parametrize("L", [1, 2])
def test_emu_short_chains(emulator, method, L):
    gpu.test_short_chains(method, L)


@pytest.mark.parametrize("method", gpu.METHODS)
def test_emu_split_opts_override_defaults(emulator, method):
    gpu.test_split_opts_override_defaults(method)


def test_emu_mixed_dtypes_promote(emulator):
    gpu.test_mixed_dtypes_promote()


def test_emu_argument_errors(emulator):
    gpu.test_argument_errors()
