"""CPU tier of the variational 1D fit: the numpy oracle against what the
unmodified reference computed, and the host layer (contraction and split
sequences, conjugation flags, sweep schedule, environment preparation, host
reads, dtype and argument handling) run against a numpy emulation of the C
ABI.  The test bodies are those of tests/test_gpu_fit.py."""

import numpy as np
import pytest

from oracle import fit_np as onp
from quimb_b200 import fit as qfit
from tests import test_gpu_fit as gpu
from tests.abi_emulator import emulated_abi
from tests.conftest import load_golden


@pytest.fixture
def emulator():
    with emulated_abi() as emu:
        yield emu


class _Count:
    """Counts the calls of a module attribute, passing them through."""

    def __init__(self, monkeypatch, obj, name):
        self.calls = []
        f = getattr(obj, name)

        def wrapped(*a, **k):
            self.calls.append((a, k))
            return f(*a, **k)
        monkeypatch.setattr(obj, name, wrapped)

    def __len__(self):
        return len(self.calls)


def _ladder(L, chi, D, seed, dtype=np.complex128):
    return gpu._dev(gpu.rand_mpo(L, D, 2, dtype, seed + 1)), \
        gpu._dev(gpu.rand_mps(L, chi, 2, dtype, seed))


# ---------------------------------------------------------------- oracle ---
def test_oracle_matches_reference():
    data, meta = load_golden("fit")
    kinds = set()
    for k, case in enumerate(meta["cases"]):
        targets, guess = gpu._case_inputs(data, meta, case)
        kw = gpu._kwargs(case)
        info = {}
        got = onp.fit(targets, guess=guess, info=info, **kw)
        assert info["sweeps"] == case["sweeps"]
        if case.get("property"):
            exact = onp.target_dense(targets, kw.get("transpose", False))
            f = onp.fidelity(onp.dense(got), exact)
            assert f >= case["fidelity_ref"] - meta["property_tol"]
            continue
        assert [x.shape[2] for x in got[:-1]] == case["bonds"]
        vec = data[f"case{k}__vec"]
        np.testing.assert_allclose(onp.dense(got), vec, rtol=0,
                                   atol=1e-10 * np.max(np.abs(vec)))
        for i, s in enumerate(onp.schmidt_values(got)):
            ref = data[f"case{k}__S{i}"]
            np.testing.assert_allclose(s, ref, rtol=0, atol=1e-10 * ref[0])
        bsz = qfit.choose_bsz(case.get("bsz", "auto"), case.get("max_bond"), case.get("cutoff"))
        kinds.add((bsz, case["guess"] == "zipup", len(case["targets"])))
    assert {(2, False, 1), (2, True, 1), (2, False, 2), (1, False, 1), (1, False, 2)} <= kinds


def test_fixtures_pin_bond_expansion_by_property_only():
    """The one-site expansion cases depend on the guess's gauge: a left- and
    a right-canonical copy of the same guess give different results."""
    data, meta = load_golden("fit")
    case = next(c for c in meta["cases"] if c.get("property") and c["guess"] != "zipup")
    targets, guess = gpu._case_inputs(data, meta, case)
    kw = dict(gpu._kwargs(case), tol=0.0, max_iterations=10)
    left, right = [x.copy() for x in guess], [x.copy() for x in guess]
    for i in range(len(guess) - 1):
        onp._qr_site(left, i)
        onp._lq_site(right, len(guess) - 1 - i)
    a = onp.dense(onp.fit(targets, guess=left, **kw))
    b = onp.dense(onp.fit(targets, guess=right, **kw))
    assert np.max(np.abs(a - b)) / np.max(np.abs(a)) > 1e-3


def test_bond_schedule():
    assert qfit.bond_schedule(None, 8, 10, 2, True) == (float("inf"), 8)
    assert qfit.bond_schedule(1000, 8, 3, 1, True) == (1000, 125)
    assert qfit.bond_schedule(6, 8, 10, 1, False) == (6, 6)
    assert qfit.bond_schedule(12, 8, 1, 2, True) == (12, 12)
    with pytest.raises(ValueError):
        qfit.bond_schedule(None, 8, 10, 1, True)
    assert qfit.choose_bsz("auto", 10, None) == 1
    assert qfit.choose_bsz("auto", 10, 1e-10) == 2
    assert qfit.choose_bsz("auto", None, None) == 2
    assert qfit.choose_bsz("auto", None, 0.0) == 1


# --------------------------------------------------------------- emulated ---
def test_emu_golden(emulator):
    gpu.test_golden_matches_reference()
    assert emulator.calls["qb_contract_pair"] > 0


@pytest.mark.parametrize("bsz", [1, 2])
def test_emu_matches_oracle(emulator, bsz):
    gpu.check_against_oracle(12, 16, 3, 2, np.complex128, bsz, seed=5)


def test_emu_untruncated(emulator):
    gpu.test_untruncated_equals_mpo_apply()
    gpu.test_untruncated_sum_equals_mps_add()


@pytest.mark.parametrize("bsz", [1, 2])
@pytest.mark.parametrize("sweep_sequence", ["RL", "LR", "RRL"])
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_emu_canonical_form_and_info(emulator, bsz, sweep_sequence, sweep_reverse):
    gpu.test_canonical_form_and_info(bsz, sweep_sequence, sweep_reverse)


@pytest.mark.parametrize("bsz", [1, 2])
def test_emu_inputs_unchanged(emulator, bsz):
    gpu.test_inputs_unchanged(bsz)


def test_emu_short_chains(emulator):
    gpu.test_short_chains()


def test_emu_same_seed_same_bits(emulator):
    gpu.test_same_seed_same_bits()


def test_emu_mixed_dtypes_promote(emulator):
    gpu.test_mixed_dtypes_promote()


def test_emu_argument_errors(emulator):
    gpu.test_argument_errors()


@pytest.mark.parametrize("bsz", [1, 2])
def test_emu_launch_and_split_sequence(emulator, monkeypatch, bsz):
    """One MPO target, no tol: every environment step and local tensor is a
    fixed number of contraction launches (the partial of one step reused by
    the next step's environment), and every step one split (two-site) or one
    QR move (one-site)."""
    N, sweeps = 9, 3
    mpo, psi = _ladder(N, 6, 3, 20)
    guess = gpu._dev(gpu.full_mps(N, 6, 2, np.complex128, 22))
    cp = _Count(monkeypatch, qfit, "contract_pair")
    sp = _Count(monkeypatch, qfit, "array_split")
    lq = _Count(monkeypatch, qfit.tebd, "left_canonize_site")
    rq = _Count(monkeypatch, qfit.tebd, "right_canonize_site")
    qfit.mps_fit([(mpo, psi)], guess=guess, bsz=bsz, max_iterations=sweeps)
    if bsz == 1:
        # prepare: N - 1 QR moves and environments; a sweep: N - 1 QR moves,
        # 3 launches per local tensor and 1 per environment
        assert len(cp) == 3 * (N - 1) + sweeps * (3 * N + N - 1)
        assert len(lq) + len(rq) == (N - 1) * (1 + sweeps)
        assert len(sp) == 0
    else:
        # prepare: N - 2 environments; a sweep: 5 launches per block, 1 per
        # environment, one split per block
        assert len(cp) == 3 * (N - 2) + sweeps * (5 * (N - 1) + N - 2)
        assert len(sp) == sweeps * (N - 1)
        assert len(lq) + len(rq) == N - 1


def test_emu_conjugation_flags(emulator, monkeypatch):
    """The fitted sites enter the environments through the conjugation flag
    (no conjugated copies): a lazily conjugated guess or target gives the
    result of its materialised conjugate."""
    from quimb_b200 import ops
    N = 7
    mpo, psi = _ladder(N, 5, 3, 30)
    G = gpu._dev(gpu.full_mps(N, 5, 2, np.complex128, 31))
    cp = _Count(monkeypatch, qfit, "contract_pair")
    qfit.mps_fit([(mpo, psi)], guess=G, bsz=2, max_iterations=2)
    # every environment step conjugates the fitted site on load
    assert sum(bool(k.get("conj_a") or k.get("conj_b")) for _, k in cp.calls) == 3 * (N - 2)
    lazy = qfit.mps_fit([(mpo, psi)], guess=[x.conj() for x in G], bsz=2, max_iterations=2)
    eager = qfit.mps_fit([(mpo, psi)], guess=[ops.materialize(x.conj()) for x in G], bsz=2,
                         max_iterations=2)
    for x, y in zip(lazy, eager):
        np.testing.assert_allclose(gpu._np(x), gpu._np(y), rtol=0, atol=1e-13)
    B = gpu._dev(gpu.rand_mps(N, 4, 2, np.complex128, 32))
    lazy = qfit.mps_fit([[x.conj() for x in B]], guess=G, bsz=2, max_iterations=2)
    eager = qfit.mps_fit([[ops.materialize(x.conj()) for x in B]], guess=G, bsz=2,
                         max_iterations=2)
    for x, y in zip(lazy, eager):
        np.testing.assert_allclose(gpu._np(x), gpu._np(y), rtol=0, atol=1e-13)


@pytest.mark.parametrize("seq,its,want", [("RL", 4, 1), ("R", 4, 4), ("RRL", 6, 3),
                                          ("LLR", 3, 2)])
def test_emu_prepare_schedule(emulator, monkeypatch, seq, its, want):
    """Environments are rebuilt on the first sweep and whenever the direction
    repeats (bsz = 2; one-site also whenever the bond is padded)."""
    mpo, psi = _ladder(7, 4, 3, 40)
    prep = _Count(monkeypatch, qfit._Fit, "prepare")
    qfit.mps_fit([(mpo, psi)], max_bond=6, cutoff=1e-10, max_iterations=its,
                 sweep_sequence=seq, seed=1)
    assert len(prep) == want


def test_emu_one_site_expansion_prepares(emulator, monkeypatch):
    """One-site from a guess of bond 2 to max_bond 8: padded (with zeros) on
    the first two sweeps, each of which then rebuilds the environments."""
    mpo, psi = _ladder(8, 4, 3, 50)
    G = gpu._dev(gpu.full_mps(8, 2, 2, np.complex128, 51))
    prep = _Count(monkeypatch, qfit._Fit, "prepare")
    pad = _Count(monkeypatch, qfit.ops, "pad")
    info = {}
    out = qfit.mps_fit([(mpo, psi)], guess=G, max_bond=8, bsz=1, max_iterations=4, info=info)
    assert len(prep) == 2 and len(pad) > 0
    assert max(x.shape[2] for x in out) == 8


@pytest.mark.parametrize("bsz", [1, 2])
@pytest.mark.parametrize("tol", [0.0, 1e-3])
def test_emu_reads_once_per_sweep(emulator, monkeypatch, bsz, tol):
    """``tol > 0``: the convergence measure is read back once per sweep;
    ``tol == 0``: never."""
    mpo, psi = _ladder(8, 6, 3, 60)
    G = gpu._dev(gpu.full_mps(8, 6, 2, np.complex128, 61))
    reads = _Count(monkeypatch, qfit, "_host_read")
    info = {}
    qfit.mps_fit([(mpo, psi)], guess=G, bsz=bsz, tol=tol, max_iterations=20, info=info)
    assert len(reads) == (info["sweeps"] if tol else 0)
    assert (info["max_tdiff"] >= 0) == bool(tol)
