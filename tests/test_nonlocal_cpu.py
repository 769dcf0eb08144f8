"""CPU tier of sub-MPO gate application: the numpy oracle against what the
unmodified reference computed, and the host layer (the MPO split, the
sub-range ladder's contraction and split sequences, gap sites, orientation,
``info`` handling, the circuit driver and argument handling) run against a
numpy emulation of the C ABI.  Several test bodies are those of
tests/test_gpu_nonlocal.py."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import mpo_compress_np as mnp
from oracle import nonlocal_np as onp
from quimb_b200 import mpo_compress, nonlocal_gates as nl, tebd
from tests import test_gpu_nonlocal as gpu
from tests.abi_emulator import emulated_abi
from tests.conftest import load_golden
from tests.test_gpu_mps_sample import rand_mps


@pytest.fixture
def emulator():
    with emulated_abi() as emu:
        yield emu


# ------------------------------------------------------------------ oracle ---
def test_oracle_matches_reference():
    data, meta = load_golden("nonlocal")
    seen = set()
    for k, case in enumerate(meta["cases"]):
        A, G = gpu._inputs(data, meta, case)
        kw = gpu._kwargs(case)
        if case.get("controls"):
            got, c = onp.gate_controlled(A, G, case["where"], case["controls"], **kw)
        else:
            got, c = onp.gate_nonlocal(A, G, case["where"], **kw)
        assert [x.shape[2] for x in got[:-1]] == case["bonds"]
        assert [c, c] == case["cur_orthog"]
        vec = data[f"case{k}__vec"]
        np.testing.assert_allclose(mnp.dense(got), vec, rtol=0,
                                   atol=1e-10 * np.max(np.abs(vec)))
        for i, s in enumerate(mnp.schmidt_values(got)):
            ref = data[f"case{k}__S{i}"]
            np.testing.assert_allclose(s, ref, rtol=0, atol=1e-10 * ref[0])
        seen.add(case["method"])
    assert seen == set(gpu.METHODS)
    assert meta["min_cut_gap"] > 1e-6


def test_oracle_circuit_matches_reference():
    data, meta = load_golden("nonlocal")
    c = meta["circuit"]
    got = onp.apply_circuit(gpu.zero_state(c["N"]), gpu.circuit_gates(data, meta),
                            contract="auto-mps", max_bond=c["max_bond"], cutoff=c["cutoff"])
    assert [x.shape[2] for x in got[:-1]] == c["bonds"]
    np.testing.assert_allclose(mnp.dense(got), data["circ__vec"], rtol=0, atol=1e-10)


def test_fixtures_truncate_in_the_zipup_gauge():
    """Without the sub-range network's pseudo-canonical gauge the truncating
    zip-up fixtures are not reproduced: they pin the gauge, not just the
    method."""
    data, meta = load_golden("nonlocal")
    worst = 0.0
    for k, case in enumerate(meta["cases"]):
        if case["method"] != "zipup" or case.get("max_bond") is None or case.get("controls"):
            continue
        A, G = gpu._inputs(data, meta, case)
        got, _ = onp.gate_nonlocal(A, G, case["where"], canonize=False, **gpu._kwargs(case))
        vec = data[f"case{k}__vec"]
        worst = max(worst, np.max(np.abs(mnp.dense(got) - vec)) / np.max(np.abs(vec)))
    assert worst > 1e-3


def test_default_ladder_tree_span_unchanged():
    """The sub-range options default to the full-chain ladder."""
    args = (6, [2, 4, 5, 4, 2], [3, 3, 3, 3, 3], [2] * 6, 5)
    assert (mpo_compress.ladder_tree_span(*args)
            == mpo_compress.ladder_tree_span(*args, gaps=(), open_ends=(False, False),
                                             rung_between=False))


# ------------------------------------------------------------- host layer ---
def test_emu_golden(emulator):
    gpu.test_golden_matches_reference()
    assert emulator.calls["qb_contract_pair"] > 0


def test_emu_circuit(emulator):
    gpu.test_circuit_matches_reference()


@pytest.mark.parametrize("method", gpu.METHODS)
def test_emu_matches_oracle(emulator, method):
    gpu.check_against_oracle(14, 12, gpu.rand_unitary(8, np.complex128, 2), (11, 2, 6),
                             np.complex128, method, seed=5)


@pytest.mark.parametrize("method", gpu.METHODS)
@pytest.mark.parametrize("where", [(1, 5, 3), (6, 2), (0, 7)])
def test_emu_untruncated_equals_mpo_apply(emulator, method, where):
    gpu.test_untruncated_equals_mpo_apply(method, where)


@pytest.mark.parametrize("name", ["CX", "RZZ", "CX_far", "C2X"])
def test_emu_mpo_from_dense_is_unitary(emulator, name):
    gpu.test_mpo_from_dense_is_unitary(name)


@pytest.mark.parametrize("method", gpu.METHODS)
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_emu_canonical_form_and_info(emulator, method, sweep_reverse):
    gpu.test_canonical_form_and_info(method, sweep_reverse)


@pytest.mark.parametrize("method", gpu.METHODS)
def test_emu_inputs_unchanged(emulator, method):
    gpu.test_inputs_unchanged(method)


@pytest.mark.parametrize("contract", ["auto-mps", "nonlocal"])
def test_emu_apply_circuit_modes_agree(emulator, contract):
    gpu.test_apply_circuit_modes_agree_untruncated(contract)


def test_emu_argument_errors(emulator):
    gpu.test_argument_errors()


class _Count:
    """Counts the ladder's own contraction launches (those of mpo_compress,
    not the splits' internal ones) and its splits."""

    def __init__(self, monkeypatch):
        self.n = {"contract": 0, "split": 0, "canon": 0, "compress": 0, "canon_bond": 0}
        for mod, name, key in ((mpo_compress, "contract_pair", "contract"),
                               (mpo_compress, "array_split", "split"),
                               (mpo_compress, "tensor_canonize_bond", "canon_bond"),
                               (tebd, "left_canonize_site", "canon"),
                               (tebd, "right_compress_site", "compress")):
            monkeypatch.setattr(mod, name, self._wrap(getattr(mod, name), key))

    def _wrap(self, fn, key):
        def f(*a, **k):
            self.n[key] += 1
            return fn(*a, **k)
        return f


@pytest.mark.parametrize("where", [(2, 3), (2, 6), (2, 3, 4), (2, 5, 6), (6, 2, 9)])
@pytest.mark.parametrize("method", ["direct", "dm", "zipup", "zipup-nocanon"])
def test_emu_launch_and_split_counts(emulator, monkeypatch, method, where):
    """Per-method contraction and split counts of one sub-range application
    over N = sf - si + 1 sites, P of them carrying an MPO tensor: a gap site
    costs no product contraction ('direct': an index expansion, one permute
    launch; 'dm': two environment and one carry contraction instead of four
    and two; zip-up without the gauge: one carry contraction instead of
    two)."""
    A = rand_mps(11, 6, 2, np.complex128, 3)
    psi = [qb.asarray(a) for a in A]
    G = gpu.rand_unitary(2 ** len(where), np.complex128, 1)
    mpo, present = qb.mpo_from_dense(G, 2, where)
    si, sf = present[0], present[-1]
    N = sf - si + 1
    gap = [s not in present for s in range(si, sf + 1)]
    info = {"cur_orthog": (si, sf)}
    qb.mps_canonicalize(psi, (si, sf), {})
    count = _Count(monkeypatch)
    emulator.calls.clear()
    kw = dict(canonize=False) if method == "zipup-nocanon" else {}
    out = qb.mps_gate_with_submpo(psi, mpo, where, method=method.split("-")[0], max_bond=5,
                                  info=info, **kw)
    n = count.n
    carry = sum(1 if g else 2 for g in gap)
    if method == "direct":
        assert n["contract"] == N - sum(gap)
        assert n["canon"] == N - 1 and n["compress"] == N - 1
        assert emulator.calls["qb_permute"] >= sum(gap)
    elif method == "dm":
        envs = 2 + sum(2 if g else 4 for g in gap[1:-1])
        assert n["contract"] == envs + carry + 3 * (N - 1)
        assert n["split"] == N - 1
    elif method == "zipup":
        # the gauge leaves a full matrix on every gap site: two contractions
        assert n["canon_bond"] == 2 * N - 2
        assert n["contract"] == 2 * N
        assert n["split"] == N - 1
    else:
        assert n["canon_bond"] == 0
        assert n["contract"] == carry
        assert n["split"] == N - 1
    assert info["cur_orthog"] == (si, si)
    assert len(out) == len(psi)


def test_emu_info_skips_canonicalisation(emulator, monkeypatch):
    """A centre already inside the span costs no QR: consecutive gates on
    overlapping spans canonicalise only between the old and new centre."""
    A = rand_mps(10, 6, 2, np.complex128, 4)
    psi = [qb.asarray(a) for a in A]
    info = {}
    qb.mps_canonicalize(psi, (3, 6), info)
    moves = []
    for name in ("left_canonize_site", "right_canonize_site"):
        fn = getattr(tebd, name)
        monkeypatch.setattr(tebd, name,
                            lambda s, i, fn=fn, name=name: (moves.append((name, i)), fn(s, i)))
    U8 = gpu.rand_unitary(8, np.complex128, 2)
    psi = qb.mps_gate_nonlocal(psi, U8, (6, 3, 4), info=info, max_bond=8, method="dm")
    assert moves == [] and info["cur_orthog"] == (3, 3)
    psi = qb.mps_gate_nonlocal(psi, U8, (5, 8, 7), info=info, max_bond=8, method="dm")
    assert moves == [("left_canonize_site", 3), ("left_canonize_site", 4)]
    assert info["cur_orthog"] == (5, 5)


def test_emu_apply_circuit_default_unchanged(emulator, monkeypatch):
    """The default mode runs two-site gates through gate_with_auto_swap with
    the caller's options, as before, and never reaches the sub-MPO path."""
    calls = []
    monkeypatch.setattr(nl, "mps_gate_with_submpo",
                        lambda *a, **k: calls.append("submpo"))
    psi = [qb.asarray(a) for a in gpu.zero_state(5)]
    tebd.apply_circuit(psi, [(gpu.H, (0,)), (gpu.CX, (0, 4)), (gpu.CX, (3, 1))], max_bond=4)
    assert calls == []
    with pytest.raises(ValueError, match="only one- and two-qubit gates"):
        tebd.apply_circuit(psi, [(gpu.CCX, (0, 2, 4))])


def test_emu_apply_circuit_carries_info(emulator):
    """One info dict across the circuit: a two-site gate by swaps leaves the
    centre inside its span, a sub-MPO gate at its first site."""
    psi = [qb.asarray(a) for a in gpu.zero_state(8)]
    info = {}
    tebd.apply_circuit(psi, [(gpu.H, (q,)) for q in range(8)] + [(gpu.CX, (1, 6))],
                       contract="auto-mps", info=info)
    assert info["cur_orthog"] == (1, 6)
    tebd.apply_circuit(psi, [(gpu.CCX, (7, 2, 4))], contract="auto-mps", info=info)
    assert info["cur_orthog"] == (2, 2)
    tebd.apply_circuit(psi, [(gpu.X, (5,), (0,))], contract="nonlocal", info=info)
    assert info["cur_orthog"] == (0, 0)
