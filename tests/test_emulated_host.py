"""CPU tier: the product's HOST LAYER (tree executor, einsum/tensordot label
logic, split drivers, complex embedding, Lanczos, MPS / DMRG2 drivers) run
against ``tests/abi_emulator.py`` -- a numpy emulation of the kernel-launching
C-ABI entry points -- and checked against the same oracle / golden vectors as
the GPU tier.  The test bodies ARE the ``-m gpu`` parity tests (imported
below, minus their module-level gpu mark): what changes is only who serves the
ABI calls.  This validates pointer / stride / label / option plumbing of the
Python layer without a device; it makes no statement about the CUDA kernels.
"""

import importlib

import pytest

from tests.abi_emulator import emulated_abi

# tests that need a real device (CUDA graphs, streams, kernel-specific
# tolerances or engines) or are too large for the CPU tier's time budget
_SKIP = {
    "test_gpu_contract": {
        "test_full_size_properties_chi1024",
        # assert the launch count of the int8 engine's kernel sequence
        "test_int8_engine_matches_oracle",
        "test_int8_engine_badly_scaled_and_accumulate",
        "test_native_single_precision_engine",
        # int8 engine edges: device tensors and the engine's own error bound
        "test_int8_engine_ragged_edges",
        "test_int8_engine_k_limit",
        "test_int8_engine_nonfinite_inputs",
        "test_int8_engine_extreme_exponents",
    },
    "test_gpu_tree_circuit": {"test_cuda_graph_replay_of_a_tree"},
    # spawns worker processes on the real device
    "test_gpu_mps_dmrg": {"test_bond_sharded_eigensolve_two_ranks_one_gpu",
                          # CUDA graph capture needs a device
                          "test_chain_plans_replay_as_cuda_graphs"},
    "test_gpu_split": set(),
    "test_gpu_split2": set(),
    "test_gpu_zzz_split3": set(),
    # asserts the launch count of the real engine
    "test_gpu_zzz_stream": {"test_stream_engine_gate_application"},
    "test_gpu_boundary": set(),
    "test_gpu_tebd": set(),
    "test_gpu_linop": set(),
    # allocates on the device directly
    "test_gpu_zz_edge_cases": {"test_zero_extent_contraction_into_a_strided_output"},
    "test_gpu_compressed": set(),
    # raw C-ABI calls on device buffers, and subprocesses on the real device
    "test_gpu_decomp_routes": {"test_qr_raw_abi_sentinels", "test_svd_trunc_raw_abi_sentinels",
                               "test_process_switches_graph_and_accumulate"},
}


@pytest.fixture(autouse=True)
def _emulator():
    with emulated_abi() as emu:
        yield emu


def _reexport():
    for modname, skip in _SKIP.items():
        mod = importlib.import_module(f"tests.{modname}")
        for name, obj in vars(mod).items():
            if name.startswith("test_") and callable(obj) and name not in skip:
                globals()[f"test_emu__{modname[9:]}__{name[5:]}"] = obj
            elif type(obj).__name__ == "FixtureFunctionDefinition" or hasattr(
                    obj, "_pytestfixturefunction"):
                globals()[name] = obj            # module-level fixtures travel along


_reexport()


def test_emu_blocked_qr_svd_for_tall_matrices(monkeypatch):
    """m > 16384 rows goes through the blocked (TSQR) host composition; the
    limit is lowered here so the logic runs at test size."""
    import numpy as np
    import quimb_b200 as qb
    from quimb_b200 import linalg
    monkeypatch.setattr(linalg, "_QR_MAX_ROWS", 48)
    rng = np.random.default_rng(0)
    for m, n in [(100, 20), (200, 24), (97, 16)]:
        x = rng.standard_normal((m, n))
        Q, R = linalg.qr(qb.asarray(x), stabilized=True)
        q, r = Q.to_numpy(), R.to_numpy()
        np.testing.assert_allclose(q @ r, x, atol=1e-12)
        np.testing.assert_allclose(q.T @ q, np.eye(n), atol=1e-12)
        assert np.all(np.diag(r) >= 0) and np.allclose(np.tril(r, -1), 0)
        _, R2 = linalg.qr(qb.asarray(x), stabilized=True, want_q=False)
        np.testing.assert_allclose(R2.to_numpy(), r, atol=1e-12)
        U, s, VH = (t.to_numpy() for t in linalg.svd(qb.asarray(x)))
        np.testing.assert_allclose(s, np.linalg.svd(x, compute_uv=False), rtol=1e-12)
        np.testing.assert_allclose((U * s) @ VH, x, atol=1e-12)
    z = rng.standard_normal((120, 10)) + 1j * rng.standard_normal((120, 10))
    Q, R = linalg.qr(qb.asarray(z))
    np.testing.assert_allclose(Q.to_numpy() @ R.to_numpy(), z, atol=1e-12)
    with pytest.raises(ValueError):
        linalg.qr(qb.asarray(rng.standard_normal((100, 60))))


def test_emu_inplace_arithmetic_updates_storage_and_refuses_widening():
    """ADVICE r01: += / -= / *= / /= mutate the array's own storage (views and
    aliases see the update, as numpy's do) and raise on a dtype-widening result."""
    import numpy as np
    import quimb_b200 as qb
    x = qb.asarray(np.arange(6.0).reshape(2, 3))
    row = x[0]
    row += 10.0
    np.testing.assert_array_equal(x.to_numpy(), [[10.0, 11.0, 12.0], [3.0, 4.0, 5.0]])
    alias = x
    x *= 2.0
    assert alias is x
    np.testing.assert_array_equal(alias.to_numpy()[1], [6.0, 8.0, 10.0])
    x -= qb.asarray(np.ones((2, 3)))
    x /= 2.0
    np.testing.assert_array_equal(x.to_numpy(), [[9.5, 10.5, 11.5], [2.5, 3.5, 4.5]])
    with pytest.raises(TypeError):
        x += 1j                       # real storage cannot take a complex result
    z = qb.asarray(np.array([1 + 1j, 2 - 1j])).conj()      # lazy conjugation flag
    z += 1.0
    np.testing.assert_allclose(z.to_numpy(), [2 - 1j, 3 + 1j])
