"""CPU tier of successive compression: the numpy oracle against what the
unmodified reference computed, and the host layer (the left-environment and
sweep sequences, the noise draw, conjugation flags, orientation, dtype and
argument handling) run against a numpy emulation of the C ABI, including
``qb_sketch_env`` (emulated below).  Test bodies are shared with
tests/test_gpu_successive.py; the raw-kernel tests need the device."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import successive_np as onp
from quimb_b200 import _lib
from quimb_b200 import successive as sc
from tests import test_gpu_successive as gpu
from tests.abi_emulator import _NP, _addr, _flat, emulated_abi
from tests.conftest import load_golden
from tests.test_gpu_mpo_compress import rand_mpo
from tests.test_gpu_mps_sample import rand_mps


def _strided(ptr, shape, strides, dtype):
    dt = np.dtype(dtype)
    extent = 1 + sum((n - 1) * s for n, s in zip(shape, strides))
    return np.lib.stride_tricks.as_strided(
        _flat(ptr, extent, dt), shape=shape, strides=tuple(s * dt.itemsize for s in strides))


def _emulated_sketch_env(emu, dtype, nB, na, nv, nu, no, np_, LE, les, W, ws, Om, oms, H, hs,
                         stream):
    """numpy version of qb_sketch_env (csrc/sketch.cu), same contract."""
    if dtype not in _NP:
        return emu._fail(-1, "qb_sketch_env: unknown dtype")
    if min(nB, na, nv, nu, no, np_) < 1:
        return emu._fail(-2, "qb_sketch_env: extents must be >= 1")
    align = np.dtype(_NP[dtype]).itemsize - 1
    if any(not _addr(p) or _addr(p) & align for p in (LE, W, Om, H)) or \
            any(s is None for s in (les, ws, oms, hs)):
        return emu._fail(-3, "qb_sketch_env: null or misaligned pointer")
    emu._tick("qb_sketch_env")
    dt = _NP[dtype]
    wide = np.complex128 if np.dtype(dt).kind == "c" else np.float64
    st = [[int(s[i]) for i in range(n)] for s, n in ((les, 3), (ws, 4), (oms, 2), (hs, 4))]
    le = _strided(LE, (nB, na, nv), st[0], dt).astype(wide)
    w = _strided(W, (nv, nu, no, np_), st[1], dt).astype(wide)
    om = _strided(Om, (nB, no), st[2], dt).astype(wide)
    _strided(H, (nB, na, nu, np_), st[3], dt)[...] = np.einsum(
        "Bav,vuop,Bo->Baup", le, w, om).astype(dt)
    return 0


@pytest.fixture
def emulator():
    with emulated_abi() as emu:
        emu.qb_sketch_env = lambda *a: _emulated_sketch_env(emu, *a)
        yield emu


# ------------------------------------------------------------------ oracle ---
def test_oracle_matches_reference():
    data, meta = load_golden("successive")
    methods = set()
    for k, case in enumerate(meta["cases"]):
        A, W = gpu._inputs(data, meta, case)
        got = onp.gate_with_mpo_successive(A, W, **gpu._kwargs(data, meta, case))
        assert [x.shape[2] for x in got[:-1]] == case["bonds"]
        vec = data[f"case{k}__vec"]
        np.testing.assert_allclose(onp.dense(got), vec, rtol=0, atol=1e-10 * np.max(np.abs(vec)))
        for i, s in enumerate(onp.schmidt_values(got)):
            ref = data[f"case{k}__S{i}"]
            np.testing.assert_allclose(s, ref, rtol=0, atol=1e-10 * ref[0])
        methods.add(case["method"])
    assert methods == set(gpu.METHODS)
    assert meta["min_cut_gap"] > 1e-6


def test_fixtures_depend_on_the_noise():
    """Another seed gives another sketch: the fixtures pin the noise rule."""
    data, meta = load_golden("successive")
    k, case = next((k, c) for k, c in enumerate(meta["cases"])
                   if c["method"] == "src" and c["max_bond"] == 6)
    A, W = gpu._inputs(data, meta, case)
    kw = dict(gpu._kwargs(data, meta, case), seed=case["seed"] + 100)
    vec = data[f"case{k}__vec"]
    assert np.max(np.abs(onp.dense(onp.gate_with_mpo_successive(A, W, **kw)) - vec)) > \
        1e-3 * np.max(np.abs(vec))


# ------------------------------------------------------- host layer (ABI) ---
def test_emu_golden(emulator):
    gpu.test_golden_matches_reference()
    assert emulator.calls["qb_sketch_env"] > 0


@pytest.mark.parametrize("method", gpu.METHODS)
def test_emu_matches_oracle(emulator, method):
    gpu.check_against_oracle(10, 12, 2, np.complex128, method, seed=5, mpo="rand")


@pytest.mark.parametrize("method", ["src", "sdc"])
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_emu_exact_when_sketch_covers_the_rank(emulator, method, sweep_reverse):
    gpu.test_exact_when_sketch_covers_the_rank(method, sweep_reverse)


@pytest.mark.parametrize("method", gpu.METHODS)
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_emu_canonical_form_and_info(emulator, method, sweep_reverse):
    gpu.test_canonical_form_and_info(method, sweep_reverse)


@pytest.mark.parametrize("method", ["src", "src-oversample", "srcmps"])
def test_emu_seed_reproducible_and_inputs_unchanged(emulator, method):
    gpu.test_seed_reproducible_and_inputs_unchanged(method)


def test_emu_mixed_dtypes_promote(emulator):
    gpu.test_mixed_dtypes_promote()


def test_emu_argument_errors_and_warnings(emulator):
    gpu.test_argument_errors_and_warnings()


def _counting(monkeypatch):
    """Record every contraction (with its conjugation flags), split and
    noise draw of the successive module."""
    log = []
    cp, split, noise = sc._cp, sc.array_split, sc.noise_host

    def _cp(a, la, b, lb, lc):
        log.append(("cp", bool(a.cj), bool(b.cj)))
        return cp(a, la, b, lb, lc)

    def _split(x, **kw):
        log.append(("split", kw.get("method"), kw.get("absorb"), tuple(x.shape)))
        return split(x, **kw)

    def _noise(rng, k, d, dist):
        x = noise(rng, k, d, dist)
        log.append(("noise", x.shape))
        return x
    monkeypatch.setattr(sc, "_cp", _cp)
    monkeypatch.setattr(sc, "array_split", _split)
    monkeypatch.setattr(sc, "noise_host", _noise)
    return log


def test_emu_src_launches_per_site(emulator, monkeypatch):
    """'src': per site but the last one sketch launch and one GEMM for the
    environment; per site but the first three contractions, one QR
    (method 'qr', absorb 'lorthog') of a (d k_right) x k sketch and one
    contraction closing the right environment with conj(Q) by the flag; two
    contractions at the first site.  Nothing else launches."""
    L, k = 6, 4
    A = rand_mps(L, 5, 2, np.complex128, 1)
    W = rand_mpo(L, 3, 2, np.complex128, 2)
    psi = [qb.asarray(a) for a in A]
    mpo = [qb.asarray(w) for w in W]
    log = _counting(monkeypatch)
    n0 = dict(emulator.calls)
    qb.mps_gate_with_mpo_successive(psi, mpo, k, seed=0)
    calls = {key: emulator.calls[key] - n0.get(key, 0) for key in emulator.calls}
    assert calls["qb_sketch_env"] == L - 1
    cps = [e for e in log if e[0] == "cp"]
    splits = [e for e in log if e[0] == "split"]
    assert len(cps) == (L - 1) + 4 * (L - 1) + 2
    assert [e[1:3] for e in splits] == [("qr", "lorthog")] * (L - 1)
    assert splits[0][3] == (2, k)
    # only the right-environment closures conjugate, and only their Q
    conj = [e for e in cps if e[1] or e[2]]
    assert conj == [("cp", False, True)] * (L - 1)
    assert [e[1] for e in log if e[0] == "noise"] == [(k, 2)] * (L - 1)


def test_emu_noise_drawn_in_sweep_order(emulator, monkeypatch):
    """One (k, d) block per site, in site order; with ``sweep_reverse`` the
    blocks are drawn from the last site backwards.  Each block is what
    ``random.array`` draws from the Generator in turn."""
    dims = [2, 3, 2, 3, 3]
    L, k = len(dims), 3
    rng = np.random.default_rng(0)
    A, W = [], []
    bonds = [1, 2, 3, 3, 2, 1]
    for i, d in enumerate(dims):
        A.append(qb.asarray(rng.standard_normal((bonds[i], d, bonds[i + 1]))))
        W.append(qb.asarray(rng.standard_normal((1 if i == 0 else 2, 1 if i == L - 1 else 2,
                                                 d, d))))
    for rev in (False, True):
        log = _counting(monkeypatch)
        qb.mps_gate_with_mpo_successive(A, W, k, seed=11, sweep_reverse=rev)
        order = dims[::-1] if rev else dims
        assert [e[1] for e in log if e[0] == "noise"] == [(k, d) for d in order[:-1]]
        monkeypatch.undo()
    g = np.random.default_rng(11)
    blocks = [g.standard_normal((k, d)) for d in dims[:-1]]
    g = np.random.default_rng(11)
    assert all(np.array_equal(sc.noise_host(g, k, d, "normal"), b)
               for d, b in zip(dims[:-1], blocks))


def test_emu_noise_modes_agree(emulator):
    L = 6
    psi = [qb.asarray(a) for a in rand_mps(L, 4, 2, np.float64, 3)]
    mpo = [qb.asarray(w) for w in rand_mpo(L, 3, 2, np.float64, 4)]
    outs = [[x.to_numpy() for x in qb.mps_gate_with_mpo_successive(psi, mpo, 4, seed=2,
                                                                   noise_mode=m)]
            for m in sc.NOISE_MODES]
    for o in outs[1:]:
        assert all(np.array_equal(x, y) for x, y in zip(outs[0], o))


def test_emu_sdc_and_srcmps_counts(emulator, monkeypatch):
    """'sdc': per site but the last two contractions and one truncating SVD
    split (absorb 'rfactor'); 'srcmps': three contractions per environment
    and no sketch launch."""
    L = 6
    psi = [qb.asarray(a) for a in rand_mps(L, 4, 2, np.complex128, 3)]
    mpo = [qb.asarray(w) for w in rand_mpo(L, 3, 2, np.complex128, 4)]
    log = _counting(monkeypatch)
    qb.mps_gate_with_mpo_successive(psi, mpo, 4, method="sdc")
    splits = [e[1:3] for e in log if e[0] == "split"]
    assert splits == [(None, "rfactor")] * (L - 1) + [("qr", "lorthog")] * (L - 1)
    assert sum(e[0] == "cp" for e in log) == 2 * (L - 1) + 4 * (L - 1) + 2
    log.clear()
    n0 = emulator.calls["qb_sketch_env"]
    qb.mps_gate_with_mpo_successive(psi, mpo, 4, method="srcmps", seed=1)
    assert emulator.calls["qb_sketch_env"] == n0
    assert sum(e[0] == "cp" for e in log) == 3 * (L - 1) + 4 * (L - 1) + 2


def test_oversample_bond_rule():
    assert sc.oversample_bond(4, None) == 14
    assert sc.oversample_bond(100, None) == 150
    assert sc.oversample_bond(10, 1.5) == 15
    assert sc.oversample_bond(10, 12) == 12
    with pytest.raises(ValueError):
        sc.oversample_bond(10, 0)


def test_emu_kernel_contract(emulator):
    """The host wrapper passes element strides of permuted views."""
    import torch
    g = torch.Generator().manual_seed(0)
    LE = torch.randn((3, 4, 5, 2), generator=g, dtype=torch.float64)[..., 1].permute(0, 1, 2)
    W = torch.randn((2, 2, 3, 5), generator=g, dtype=torch.float64).permute(3, 2, 1, 0)
    Om = torch.randn((2, 3), generator=g, dtype=torch.float64).t()
    H = sc.sketch_env(LE, W, Om)
    np.testing.assert_allclose(H.numpy(), np.einsum("Bav,vuop,Bo->Baup", LE.numpy(),
                                                    W.numpy(), Om.numpy()), rtol=1e-14)
    assert emulator.qb_sketch_env(_lib.QB_F64, 0, 1, 1, 1, 1, 1, 8, None, 8, None, 8, None, 8,
                                  None, None) == -2
