"""CPU tier of DMRG-X: the numpy oracle against what the unmodified reference
computed, and the host layer (environments, dense Heff, selection, sweeps,
errors) run against a numpy emulation of the C ABI.  The test bodies are
those of tests/test_gpu_dmrgx.py."""

import numpy as np
import pytest
import torch

from oracle import dmrgx_np as onp
from quimb_b200 import dmrgx as qdx
from tests import test_gpu_dmrgx as gpu
from tests.abi_emulator import emulated_abi
from tests.conftest import load_golden


@pytest.fixture
def emulator():
    with emulated_abi() as emu:
        yield emu


# ---------------------------------------------------------------- oracle ---
@pytest.mark.parametrize("name", gpu.PINNED)
def test_oracle_pinned(name):
    data, meta = load_golden("dmrgx")
    case = next(c for c in meta["cases"] if c["name"] == name)
    mpo, p0 = gpu.case_inputs(data, case)
    assert onp.mpo_dist2(mpo, onp.mpo_mbl(case["fields"])) < 1e-20
    o = onp.DMRGX(mpo, p0, case["chi"])
    o.opts.update(case["opts"])
    assert abs(o.energies[0] - case["energy0"]) < 1e-12
    assert abs(onp.mps_expec2(p0, mpo) - case["en2_p0"]) < 1e-11 * abs(case["en2_p0"])
    for direction, canonize in case["sweeps"]:
        o.sweep(direction, canonize=canonize)
    np.testing.assert_allclose(np.array(o.local_energies), data[f"{name}__local"],
                               rtol=0, atol=1e-10)
    np.testing.assert_allclose(np.array(o.total_energies), data[f"{name}__total"],
                               rtol=0, atol=1e-10)
    assert gpu.fidelity(onp.mps_dense(o.k), data[f"{name}__state"]) > 1 - 1e-10
    assert min(m for _, _, m, _ in o.decisions) >= meta["min_margin"]
    assert min(g for _, _, _, g in o.decisions) >= meta["min_margin"]


@pytest.mark.parametrize("name", gpu.PROPERTY)
def test_oracle_property(name):
    data, meta = load_golden("dmrgx")
    case = next(c for c in meta["cases"] if c["name"] == name)
    mpo, p0 = gpu.case_inputs(data, case)
    o = onp.DMRGX(mpo, p0, case["chi"], seed=1)
    o.opts.update(case["opts"])
    run = case["run"]
    if isinstance(run, dict):
        assert o.solve(**run)
        energy = o.energy
    else:
        for direction, canonize in run:
            o.sweep(direction, canonize=canonize)
        energy = o.total_energies[-1][-1]
    assert abs(energy - case["energy"]) < 1e-8
    bound = max(1e-8, 1e2 * case["variance"])
    assert gpu.fidelity(onp.mps_dense(o.k), data[f"{name}__state"]) > 1 - bound


def test_oracle_sector_spectrum():
    """The S^z-sector spectrum the GPU tier uses equals the dense MPO's."""
    fields = gpu.rand_fields(6, 4.0, 8)
    H = onp.mpo_dense(onp.mpo_mbl(fields))
    ev = np.linalg.eigvalsh(H)
    psi = np.zeros(64)
    psi[0b010110] = 1.0
    sec = gpu.spectrum(fields, psi)
    for e in sec:
        assert np.min(np.abs(ev - e)) < 1e-12


# ------------------------------------------------------ host layer, emulated ---
@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_env_steps_emulated(emulator, dtype):
    gpu.check_env_steps(dtype)


def test_expec2_golden_emulated(emulator):
    gpu.check_expec2_golden()


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_dense_heff_emulated(emulator, dtype):
    gpu.check_dense_heff(dtype)


@pytest.mark.parametrize("name", gpu.PINNED)
def test_pinned_emulated(emulator, name):
    gpu.check_pinned(name)


@pytest.mark.parametrize("name", ["thresh1", "partial", "complex"])
def test_property_emulated(emulator, name):
    gpu.check_property(name)


def test_errors_emulated(emulator):
    gpu.check_errors()


def test_dmrg1_dmrg2_post_sweep_hook_is_noop(emulator):
    """DMRG1 / DMRG2 keep their results: the hook records nothing."""
    import quimb_b200 as qb
    from oracle import dmrg_np as dm
    d = qb.DMRG2(dm.mpo_heis(6), [4, 8], cutoffs=1e-10, mpo_shape="lrdu", seed=2)
    d.solve(tol=1e-8, max_sweeps=3)
    assert not hasattr(d, "variances")
    assert len(d.energies) == len(d.local_energies)


def test_site_update_host_reads(emulator, monkeypatch):
    """One site update reads only the eigenvalues, the overlaps and, with
    several candidates, their <H^2> (eigh's own internal reads aside); the
    sweep reads its total energies once at the end."""
    reads, state = [], {"on": False}
    for name in ("cpu", "item", "tolist", "__float__"):
        inner = getattr(torch.Tensor, name)

        def wrapped(self, *a, _inner=inner, _name=name, **k):
            if state["on"]:
                reads.append((_name, tuple(self.shape)))
            return _inner(self, *a, **k)
        monkeypatch.setattr(torch.Tensor, name, wrapped)
    inner_eigh = qdx.eigh

    def eigh(x, *a, **k):
        state["on"] = False
        try:
            return inner_eigh(x, *a, **k)
        finally:
            state["on"] = True
    monkeypatch.setattr(qdx, "eigh", eigh)
    updates = []
    inner_update = qdx.DMRGX._update_local_state_1site_dmrgx

    def update(self, i, direction):
        reads.clear()
        state["on"] = True
        try:
            out = inner_update(self, i, direction)
        finally:
            state["on"] = False
        updates.append((self._k[i].shape, list(reads)))
        return out
    monkeypatch.setattr(qdx.DMRGX, "_update_local_state_1site_dmrgx", update)

    data, meta = load_golden("dmrgx")
    case = next(c for c in meta["cases"] if c["name"] == "pin_real")
    mpo, p0 = gpu.case_inputs(data, case)
    d = qdx.DMRGX(gpu._dev(mpo), gpu._dev(p0), case["chi"])
    d.sweep_right()
    several = 0
    for _, rd in updates:
        names = [n for n, _ in rd]
        assert names in (["cpu", "cpu"], ["cpu", "cpu", "cpu"]), rd
        (_, ev), (_, ov) = rd[:2]
        assert len(ev) == 1 and ov == ev
        if len(rd) == 3:
            several += 1
            assert len(rd[2][1]) == 1 and rd[2][1][0] < ev[0]
    assert several > 0
    assert len(updates) == case["L"]
