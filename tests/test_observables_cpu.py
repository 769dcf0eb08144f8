"""CPU tier of the MPS observables: the numpy oracle against what the
unmodified reference computed, and the host layer (centre tracking, the three
reduced-density-matrix routes, pointer / stride / dtype plumbing of
``qb_rdm_reduce``) run against a numpy emulation of the C ABI.  The test
bodies are those of tests/test_gpu_observables.py; the raw-kernel tests need
the device and are not repeated here."""

import ctypes

import numpy as np
import pytest

from oracle import observables_np as onp
from oracle.observables_np import terms_for
from tests import test_gpu_observables as gpu
from tests.abi_emulator import _NP, _addr, _flat, emulated_abi
from tests.conftest import load_golden
from quimb_b200 import _lib


def _strided(ptr, shape, strides, dtype):
    dt = np.dtype(dtype)
    extent = 1 + sum((n - 1) * s for n, s in zip(shape, strides))
    return np.lib.stride_tricks.as_strided(
        _flat(ptr, extent, dt), shape=shape, strides=tuple(s * dt.itemsize for s in strides))


def _emulated_rdm_reduce(emu, dtype, n1, M, N, n2, U, us, V, vs, out, ws, ws_bytes, stream):
    """numpy version of qb_rdm_reduce (csrc/rdm.cu), same contract."""
    if dtype not in (_lib.QB_F64, _lib.QB_C128):
        return emu._fail(-1, "qb_rdm_reduce: dtype must be QB_F64 or QB_C128")
    rc = emu._real.qb_rdm_workspace(n1, M, N, n2)
    if rc < 0:
        return emu._fail(int(rc), "qb_rdm_reduce: bad shape")
    align = 15 if dtype == _lib.QB_C128 else 7
    ptrs = [_addr(p) for p in (U, V, out)]
    if any(not p or p & align for p in ptrs) or us is None or vs is None:
        return emu._fail(-4, "qb_rdm_reduce: null or misaligned pointer")
    if rc > 0 and (not _addr(ws) or ws_bytes < rc):
        return emu._fail(-6, "qb_rdm_reduce: workspace too small")
    emu._tick("qb_rdm_reduce", 2 if rc > 0 else 1)
    us, vs = [int(us[i]) for i in range(3)], [int(vs[i]) for i in range(3)]
    u = _strided(U, (n1, M, n2), us, _NP[dtype])
    v = _strided(V, (n1, N, n2), vs, _NP[dtype])
    _flat(out, M * N, _NP[dtype]).reshape(M, N)[...] = np.einsum("amb,anb->mn", u, v.conj())
    return 0


@pytest.fixture
def emulator():
    with emulated_abi() as emu:
        emu.qb_rdm_reduce = lambda *a: _emulated_rdm_reduce(emu, *a)
        emu.qb_rdm_workspace = emu._real.qb_rdm_workspace
        yield emu


def _oracle_case(data, meta, k, case):
    """One fixture case on the oracle."""
    name, pre = case["state"], f"case{k}__"
    sites = gpu._host_sites(data, meta, name)
    L, d = meta["states"][name]["L"], meta["states"][name]["d"]
    kind = case["kind"]
    if kind == "schmidt":
        info = {}
        for i in range(1, L):
            ref = data[pre + f"S{i}"]
            S = onp.schmidt_values(sites, i, info, case["method"])
            np.testing.assert_allclose(S, ref, rtol=0, atol=1e-12 * ref[0])
            gpu._close(onp.entropy(sites, i, info, case["method"]), data[pre + "entropy"][i - 1])
            gpu._close(onp.schmidt_gap(sites, i, info, case["method"]), data[pre + "gap"][i - 1])
        assert info["cur_orthog"] == tuple(case["cur_orthog"])
    elif kind == "rho":
        info = {}
        rho = onp.partial_trace_to_dense_canonical(sites, tuple(case["where"]),
                                                   case["normalized"], info)
        gpu._close(rho, data[pre + "rho"])
        assert info["cur_orthog"] == tuple(case["cur_orthog"])
    elif kind == "expec":
        if case["start"] is not None:
            sites = [data[pre + f"in{i}"].copy() for i in range(L)]
        info = None if case["info"] is None else {
            key: gpu._info(val) for key, val in case["info"].items()}
        got = onp.compute_local_expectation(sites, terms_for(case["terms"], L, d),
                                            return_all=case["return_all"],
                                            method=case["method"], info=info,
                                            inplace=case["inplace"])
        vals = [got[tuple(kk)] for kk in case["keys"]] if case["return_all"] else [got]
        gpu._close(np.array(vals, dtype=complex), data[pre + "values"])
        if "cur_orthog_after" in case:
            assert info["cur_orthog"] == gpu._info(case["cur_orthog_after"])
        if case["inplace"]:
            for i in range(L):
                gpu._close(sites[i], data[pre + f"out{i}"])
    elif kind == "mag":
        info = {}
        vals = [onp.magnetization(sites, case["site"], c, info) for c in "XYZ"]
        gpu._close(np.array(vals, dtype=complex), data[pre + "values"])
    elif kind == "corr":
        Z, X = onp.spin_operator("Z") * 2, onp.spin_operator("X") * 2
        c = onp.correlation(sites, Z, case["i"], case["j"], B=X if case["B"] else None)
        gpu._close(c, data[pre + "value"])


def test_oracle_matches_reference():
    data, meta = load_golden("observables")
    kinds = set()
    for k, case in enumerate(meta["cases"]):
        _oracle_case(data, meta, k, case)
        kinds.add(case["kind"])
    assert kinds == {"schmidt", "rho", "expec", "mag", "corr"}


def test_emu_golden(emulator):
    gpu.test_golden_matches_reference()
    assert emulator.calls["qb_rdm_reduce"] > 0


def test_emu_correlation_docstring_values(emulator):
    gpu.test_correlation_docstring_values()


def test_emu_singular_values_bond_range(emulator):
    gpu.test_singular_values_bond_range()


@pytest.mark.parametrize("dtype,d", [(np.float64, 2), (np.complex128, 3)])
def test_emu_matches_oracle(emulator, dtype, d):
    gpu.check_against_oracle(14, 12, d, dtype, seed=3 + d)


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
def test_emu_single_precision_keeps_dtype(emulator, dtype):
    gpu.test_single_precision_keeps_dtype(dtype)


def test_emu_sweep_moves_centre_once_per_site(emulator, monkeypatch):
    gpu.test_sweep_moves_centre_once_per_site(monkeypatch)


def test_emu_one_reduction_per_contiguous_term(emulator):
    """After the centre move, a contiguous term costs one qb_rdm_reduce; a
    non-contiguous one too (the transfer form ends in a single reduction)."""
    import quimb_b200 as qb
    psi = [qb.asarray(a) for a in gpu.rand_mps(8, 6, 2, np.float64, 8)]
    info = {}
    qb.mps_canonicalize(psi, (2, 3), info=info)
    for where in ((2, 3), (2, 5), (1, 3, 6)):
        n0 = emulator.calls["qb_rdm_reduce"]
        qb.mps_partial_trace_to_dense_canonical(psi, where, info=info)
        assert emulator.calls["qb_rdm_reduce"] - n0 == 1


def test_emu_non_contiguous_order_and_limits(emulator):
    """``where`` out of order gives rho in that order; operands wider than 64
    raise NotImplementedError."""
    import quimb_b200 as qb
    host = gpu.rand_mps(9, 6, 2, np.complex128, 9)
    for where in ((5, 1), (4, 0, 2)):
        got = qb.mps_partial_trace_to_dense_canonical([qb.asarray(a) for a in host], where)
        want = onp.partial_trace_to_dense_canonical([a.copy() for a in host], where)
        gpu._close(got, want)
    for where in ((0, 1, 2, 3, 4, 5, 6), (0, 2, 4, 6)):
        with pytest.raises(NotImplementedError):
            qb.mps_partial_trace_to_dense_canonical([qb.asarray(a) for a in host], where)


def test_emu_inplace_false_leaves_caller_untouched(emulator):
    import quimb_b200 as qb
    host = gpu.rand_mps(7, 5, 2, np.complex128, 11)
    psi = [qb.asarray(a) for a in host]
    ids = [id(a) for a in psi]
    before = [a.to_numpy().copy() for a in psi]
    info = {"cur_orthog": "calc"}
    terms = terms_for("heis", 7, 2)
    for method in ("canonical", "envs"):
        qb.mps_compute_local_expectation(psi, terms, method=method, info=info)
    assert info == {"cur_orthog": "calc"}
    assert [id(a) for a in psi] == ids
    for a, b in zip(psi, before):
        assert np.array_equal(a.to_numpy(), b)


def test_emu_argument_errors(emulator):
    import quimb_b200 as qb
    psi = [qb.asarray(a) for a in gpu.rand_mps(5, 4, 2, np.float64, 1)]
    with pytest.raises(ValueError):
        qb.mps_compute_local_expectation(psi, {(0,): np.eye(2)}, method="nope")
    with pytest.raises(ValueError):
        qb.mps_partial_trace_to_dense_canonical(psi, (1, 1))
    with pytest.raises(ValueError):
        qb.mps_magnetization(psi, 1, direction="Q")
    arr = ctypes.c_int64 * 3
    assert emulator.qb_rdm_reduce(_lib.QB_F32, 1, 1, 1, 1, 8, arr(1, 1, 1), 8, arr(1, 1, 1),
                                  8, None, 0, None) == -1
