"""GPU tier: the variational 1D fit (``quimb_b200.fit``: ``mps_fit`` and
``mps_gate_with_mpo_fit``).

Checked against what the unmodified reference computed (tests/golden/fit.*:
bond sizes, per-bond singular values and the dense output, all
gauge-independent; one-site fits that pad their bonds by their fidelity with
the exact sum), against the numpy oracle (oracle/fit_np.py) at L = 40,
chi = 128, and against ``tebd.mpo_apply`` / ``tebd.mps_add`` when nothing is
truncated."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import fit_np as onp
from tests.conftest import load_golden
from tests.test_gpu_mpo_compress import heis_lrud, overlap, rand_mpo
from tests.test_gpu_mps_sample import rand_mps

pytestmark = pytest.mark.gpu

_NOT_KW = ("targets", "guess", "bonds", "sweeps", "property", "fidelity_ref")


# ----------------------------------------------------------------- helpers ---
def _np(x):
    return np.asarray(x.to_numpy() if hasattr(x, "to_numpy") else x)


def _dev(x):
    return [qb.asarray(a) for a in x]


def _case_inputs(data, meta, case):
    """(targets, guess) of a fixture case as host arrays: a target is an
    (l, p, r) list or a tuple (mpo, sites) of (l, r, u, d) MPO sites."""
    def sites(name):
        return [np.ascontiguousarray(data[f"{name}__site{i}"])
                for i in range(meta["states"][name]["L"])]

    targets = []
    for t in case["targets"]:
        if t[0] == "mps":
            targets.append(sites(t[1]))
        else:
            L = meta["mpos"][t[1]]["L"]
            targets.append(([np.ascontiguousarray(data[f"{t[1]}__mpo{i}"]) for i in range(L)],
                            sites(t[2])))
    g = case["guess"]
    if g != "zipup":
        g = [np.ascontiguousarray(data[f"{g}__guess{i}"]) for i in range(meta["guesses"][g]["L"])]
    return targets, g


def _dev_targets(targets):
    return [(_dev(t[0]), _dev(t[1])) if isinstance(t, tuple) else _dev(t) for t in targets]


def _kwargs(case):
    return {k: v for k, v in case.items() if k not in _NOT_KW}


def full_mps(L, chi, d, dtype, seed):
    """Random (l, p, r) host arrays with every bond min(chi, d^i, d^(L-i))."""
    rng = np.random.default_rng(seed)
    bonds = [1] + [min(chi, d ** min(i, 30), d ** min(L - i, 30)) for i in range(1, L)] + [1]
    out = []
    for i in range(L):
        shape = (bonds[i], d, bonds[i + 1])
        x = rng.standard_normal(shape)
        if np.dtype(dtype).kind == "c":
            x = x + 1j * rng.standard_normal(shape)
        out.append((x / np.sqrt(bonds[i] * d)).astype(dtype))
    return out


def fidelity(x, y):
    return abs(overlap(x, y)) ** 2 / (overlap(x, x).real * overlap(y, y).real)


def check_golden_case(data, meta, case):
    """One fixture case on the device layer.  A two-site case first checks,
    on the oracle's spectra of the same inputs, that each cut is decided far
    from the device SVD's noise."""
    targets, guess = _case_inputs(data, meta, case)
    kw = _kwargs(case)
    k = meta["cases"].index(case)
    spectra, oinfo = [], {}
    onp.fit(targets, guess=guess, spectra=spectra, info=oinfo, **kw)
    for s, mb, cut, mode in spectra:
        onp.check_svd_margin(s, mb, cut, mode)
    onp.check_tol_margin(oinfo["tdiffs"], kw.get("tol", 0.0))
    info = {}
    out = qb.mps_fit(_dev_targets(targets), guess=guess if guess == "zipup" else _dev(guess),
                     info=info, **kw)
    got = [_np(x) for x in out]
    if case.get("property"):
        # padded one-site fits depend on the QR's completion: the sweeps run
        # and the result are checked by their fidelity only
        exact = onp.target_dense(targets, kw.get("transpose", False))
        f = onp.fidelity(onp.dense(got), exact)
        assert f >= case["fidelity_ref"] - meta["property_tol"], (f, case["fidelity_ref"])
        return
    assert info["sweeps"] == case["sweeps"]
    assert [x.shape[2] for x in got[:-1]] == case["bonds"]
    vec = data[f"case{k}__vec"]
    np.testing.assert_allclose(onp.dense(got), vec, rtol=0, atol=1e-10 * np.max(np.abs(vec)))
    for i, s in enumerate(onp.schmidt_values(got)):
        ref = data[f"case{k}__S{i}"]
        np.testing.assert_allclose(s, ref, rtol=0, atol=1e-10 * ref[0])


def check_against_oracle(L, chi, D, d, dtype, bsz, seed, mpo="rand", max_iterations=4):
    """The device fit against the oracle on one random MPS / MPO at
    ``max_bond = chi``: two-site from the random start, one-site from a guess
    at full bond.  Equal bonds, Schmidt values to 1e-10 of the largest,
    normalised fidelity within 1e-12 of 1; every two-site cut is first checked
    to lie far above the device SVD's noise."""
    A = rand_mps(L, chi, d, dtype, seed)
    W = heis_lrud(L, dtype) if mpo == "heis" else rand_mpo(L, D, d, dtype, seed + 1)
    guess = None if bsz == 2 else full_mps(L, chi, d, dtype, seed + 2)
    # no cutoff: every two-site cut is made by max_bond, in a gap the margin
    # check can see (a cutoff cut may fall within noise of its threshold)
    kw = dict(max_bond=chi, bsz=bsz, max_iterations=max_iterations, seed=seed + 3, cutoff=0.0)
    spectra = []
    want = onp.fit([(W, A)], guess=guess, spectra=spectra, **kw)
    for s, mb, cut, mode in spectra:
        onp.check_svd_margin(s, mb, cut, mode)
    out = qb.mps_fit([(_dev(W), _dev(A))], guess=None if guess is None else _dev(guess), **kw)
    got = [_np(x) for x in out]
    assert [x.shape[2] for x in got] == [x.shape[2] for x in want]
    for s, r in zip(onp.schmidt_values(got), onp.schmidt_values(want)):
        np.testing.assert_allclose(s, r, rtol=0, atol=1e-10 * r[0])
    f = fidelity(got, want)
    assert abs(f - 1) < 1e-12, f


# ------------------------------------------------------------------ tests ---
def test_golden_matches_reference():
    data, meta = load_golden("fit")
    for case in meta["cases"]:
        check_golden_case(data, meta, case)


@pytest.mark.parametrize("bsz", [1, 2])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_scale_against_oracle(bsz, dtype):
    check_against_oracle(40, 128, 5, 2, dtype, bsz, seed=7,
                         mpo="heis" if dtype == np.float64 else "rand")


def test_untruncated_equals_mpo_apply():
    """max_bond >= chi D_w and cutoff = 0: the uncompressed product
    (``mpo_apply`` contracts the MPO's upper index: ``transpose=True``)."""
    L, chi, D = 7, 4, 3
    psi = _dev(rand_mps(L, chi, 2, np.complex128, 3))
    mpo = _dev(rand_mpo(L, D, 2, np.complex128, 4))
    full = qb.tebd.mpo_apply(mpo, psi)
    got = qb.mps_gate_with_mpo_fit(psi, mpo, chi * D, cutoff=0.0, bsz=2, transpose=True, seed=1)
    ff = qb.tebd.mps_overlap(full, full).real
    for x, y in ((got, full), (got, got)):
        assert abs(qb.tebd.mps_overlap(x, y) - ff) <= 1e-12 * ff


def test_untruncated_sum_equals_mps_add():
    L = 8
    psi = _dev(rand_mps(L, 5, 2, np.complex128, 5))
    phi = _dev(rand_mps(L, 4, 2, np.complex128, 6))
    full = qb.tebd.mps_add(psi, phi)
    got = qb.mps_fit([psi, phi], max_bond=9, cutoff=0.0, bsz=2, seed=2)
    ff = qb.tebd.mps_overlap(full, full).real
    for x, y in ((got, full), (got, got)):
        assert abs(qb.tebd.mps_overlap(x, y) - ff) <= 1e-12 * ff


@pytest.mark.parametrize("bsz", [1, 2])
@pytest.mark.parametrize("sweep_sequence", ["RL", "LR", "RRL"])
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_canonical_form_and_info(bsz, sweep_sequence, sweep_reverse):
    L = 8
    A = rand_mps(L, 8, 2, np.complex128, 5)
    W = rand_mpo(L, 3, 2, np.complex128, 6)
    info = {}
    out = qb.mps_fit([(_dev(W), _dev(A))], max_bond=6, bsz=bsz, max_iterations=5,
                     sweep_sequence=sweep_sequence, sweep_reverse=sweep_reverse, info=info,
                     seed=4)
    last = sweep_sequence[(5 - 1) % len(sweep_sequence)]
    c = 0 if (last == "L") != sweep_reverse else L - 1
    assert info["cur_orthog"] == (c, c)
    assert info["sweeps"] == 5 and info["max_tdiff"] == -1.0
    for i, x in enumerate(out):
        if i == c:
            continue
        x = _np(x)
        l, d, r = x.shape
        if i < c:
            m = x.reshape(l * d, r)
            g = m.conj().T @ m
        else:
            m = x.reshape(l, d * r)
            g = m @ m.conj().T
        np.testing.assert_allclose(g, np.eye(g.shape[0]), rtol=0, atol=1e-12)
    assert tuple(qb.mps_calc_current_orthog_center(list(out))) == (c, c)


@pytest.mark.parametrize("bsz", [1, 2])
def test_tol_stops_and_reports(bsz):
    L = 8
    A = rand_mps(L, 6, 2, np.complex128, 7)
    W = rand_mpo(L, 3, 2, np.complex128, 8)
    info = {}
    qb.mps_fit([(_dev(W), _dev(A))], max_bond=8, bsz=bsz, tol=1e-3, max_iterations=50,
               info=info, seed=5)
    assert 1 <= info["sweeps"] < 50
    assert 0.0 <= info["max_tdiff"] < 1e-3


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
@pytest.mark.parametrize("bsz", [1, 2])
def test_single_precision_keeps_dtype(dtype, bsz):
    L = 8
    A = rand_mps(L, 6, 2, dtype, 8)
    W = rand_mpo(L, 3, 2, dtype, 9)
    G = full_mps(L, 6, 2, dtype, 10)
    out = qb.mps_fit([(_dev(W), _dev(A))], guess=_dev(G), bsz=bsz, max_iterations=4)
    assert all(x.dtype == np.dtype(dtype) for x in out)
    wide = np.complex128 if np.dtype(dtype).kind == "c" else np.float64
    want = onp.fit([([w.astype(wide) for w in W], [a.astype(wide) for a in A])],
                   guess=[g.astype(wide) for g in G], bsz=bsz, max_iterations=4)
    got = [_np(x).astype(wide) for x in out]
    f = fidelity(got, want)
    assert abs(f - 1) < 1e-4, f


def test_mixed_dtypes_promote():
    L = 6
    A = rand_mps(L, 4, 2, np.float64, 10)
    W = rand_mpo(L, 3, 2, np.complex128, 11)
    out = qb.mps_fit([(_dev(W), _dev(A))], max_bond=8, seed=1)
    assert all(x.dtype == np.complex128 for x in out)
    psi = rand_mps(L, 4, 2, np.float32, 12)
    phi = rand_mps(L, 4, 2, np.float64, 13)
    out = qb.mps_fit([_dev(psi), _dev(phi)], max_bond=8, seed=1)
    assert all(x.dtype == np.float64 for x in out)


@pytest.mark.parametrize("bsz", [1, 2])
def test_inputs_unchanged(bsz):
    L = 8
    A = rand_mps(L, 8, 2, np.complex128, 12)
    W = rand_mpo(L, 4, 2, np.complex128, 13)
    B = rand_mps(L, 5, 2, np.complex128, 14)
    G = full_mps(L, 4, 2, np.complex128, 15)
    psi, mpo, phi, guess = _dev(A), _dev(W), _dev(B), _dev(G)
    # the guess's bonds are padded to 6 (one-site) or grow through the split
    qb.mps_fit([(mpo, psi), phi], guess=guess, max_bond=6, bsz=bsz, normalize=True,
               tol=1e-6)
    for xs, hs in ((psi, A), (mpo, W), (phi, B), (guess, G)):
        for x, a in zip(xs, hs):
            assert np.array_equal(_np(x), a)


def test_short_chains():
    """L = 2 against the reference (the fixtures' two-site cases); L = 1 is
    refused, as the reference refuses it."""
    data, meta = load_golden("fit")
    short = [c for c in meta["cases"] if meta["states"][c["targets"][0][-1]]["L"] == 2]
    assert {c.get("bsz") for c in short} >= {1, 2} and any(c["guess"] == "zipup" for c in short)
    for case in short:
        check_golden_case(data, meta, case)
    assert meta["one_site_chain_raises"]
    A = rand_mps(1, 1, 3, np.complex128, 1)
    W = rand_mpo(1, 1, 3, np.complex128, 2)
    for guess in (_dev(A), "zipup", None):
        with pytest.raises(ValueError, match="2 sites"):
            qb.mps_fit([(_dev(W), _dev(A))], max_bond=1, guess=guess)


def test_same_seed_same_bits():
    L = 10
    A = rand_mps(L, 8, 2, np.complex128, 16)
    W = rand_mpo(L, 3, 2, np.complex128, 17)
    t = [(_dev(W), _dev(A))]
    runs = [[_np(x) for x in qb.mps_fit(t, max_bond=10, cutoff=1e-10, seed=s)]
            for s in (3, 3, 4)]
    assert all(np.array_equal(x, y) for x, y in zip(runs[0], runs[1]))
    assert not all(x.shape == y.shape and np.array_equal(x, y)
                   for x, y in zip(runs[0], runs[2]))


def test_random_guess_converges_no_worse_than_dm():
    """From the random start, the two-site fit converges (``tol``) and its
    fidelity with the exact product is no worse than 'dm' at the same
    max_bond, less 1e-6."""
    L, chi = 14, 16
    A = rand_mps(L, chi, 2, np.complex128, 18)
    W = rand_mpo(L, 3, 2, np.complex128, 19)
    exact = onp.target_dense([(W, A)])
    dm = qb.mps_gate_with_mpo(_dev(A), _dev(W), method="dm", max_bond=12)
    info = {}
    out = qb.mps_gate_with_mpo_fit(_dev(A), _dev(W), 12, cutoff=1e-10, tol=1e-6,
                                   max_iterations=40, seed=6, info=info)
    assert info["sweeps"] < 40
    f_dm = onp.fidelity(onp.dense([_np(x) for x in dm]), exact)
    f_fit = onp.fidelity(onp.dense([_np(x) for x in out]), exact)
    assert f_fit >= f_dm - 1e-6, (f_fit, f_dm)


def test_argument_errors():
    L = 5
    A = rand_mps(L, 4, 2, np.float64, 16)
    psi = _dev(A)
    mpo = _dev(rand_mpo(L, 3, 2, np.float64, 17))
    t = [(mpo, psi)]
    with pytest.raises(ValueError, match="cutoff"):
        qb.mps_fit(t, max_bond=4, bsz=1, cutoff=1e-3)
    with pytest.raises(ValueError, match="max_bond"):
        qb.mps_fit(t, bsz=1)
    with pytest.raises(ValueError, match="bsz"):
        qb.mps_fit(t, max_bond=4, bsz=3)
    with pytest.raises(ValueError, match="sweep_sequence"):
        qb.mps_fit(t, max_bond=4, sweep_sequence="RX")
    with pytest.raises(ValueError, match="max_iterations"):
        qb.mps_fit(t, max_bond=4, max_iterations=0)
    with pytest.raises(ValueError, match="tol"):
        qb.mps_fit(t, max_bond=4, tol=-1.0)
    with pytest.raises(NotImplementedError, match="first"):
        qb.mps_fit([psi, (mpo, psi)], max_bond=4, guess="zipup")
    with pytest.raises(NotImplementedError, match="fit"):
        qb.mps_fit(t, max_bond=4, guess="fit")
    with pytest.raises(NotImplementedError, match="equalize_norms"):
        qb.mps_fit(t, max_bond=4, equalize_norms=True)
    with pytest.raises(ValueError, match="sites"):
        qb.mps_fit([psi, _dev(rand_mps(L - 1, 4, 2, np.float64, 3))], max_bond=4)
    with pytest.raises(ValueError, match="physical"):
        qb.mps_fit([psi, _dev(rand_mps(L, 4, 3, np.float64, 1))], max_bond=4)
    with pytest.raises(ValueError, match="guess"):
        qb.mps_fit(t, guess=_dev(rand_mps(L, 4, 3, np.float64, 2)))
    with pytest.raises(ValueError):
        qb.mps_fit([(mpo[:-1], psi)], max_bond=4)
    with pytest.raises(TypeError, match="split options"):
        qb.mps_fit(t, max_bond=4, bsz=1, renorm=True)
    with pytest.raises(TypeError):
        qb.mps_fit(t, max_bond=4, bsz=2, absorb="left")
    # the dispatcher keeps refusing the fit methods: they live behind mps_fit
    with pytest.raises(NotImplementedError):
        qb.mps_gate_with_mpo(psi, mpo, method="fit")
