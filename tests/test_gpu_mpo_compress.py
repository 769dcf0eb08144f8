"""GPU tier: MPO application with compression (``quimb_b200.mpo_compress``).

Checked against what the unmodified reference computed
(tests/golden/mpo_compress.*: bond sizes, per-bond singular values and the
dense output, all gauge-independent), against the numpy oracle
(oracle/mpo_compress_np.py) at L = 40, chi = 128, and against the
uncompressed ``tebd.mpo_apply`` product when nothing is truncated."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import mpo_compress_np as onp
from tests.conftest import load_golden
from tests.test_gpu_mps_sample import rand_mps

pytestmark = pytest.mark.gpu

METHODS = ("direct", "dm", "zipup", "zipup-first")


# ----------------------------------------------------------------- helpers ---
def _np(x):
    return np.asarray(x.to_numpy() if hasattr(x, "to_numpy") else x)


def _inputs(data, meta, case):
    L = meta["states"][case["state"]]["L"]
    A = [np.ascontiguousarray(data[f"{case['state']}__site{i}"]) for i in range(L)]
    W = [np.ascontiguousarray(data[f"{case['mpo']}__mpo{i}"]) for i in range(L)]
    return A, W


def _kwargs(case):
    return {k: v for k, v in case.items() if k not in ("state", "mpo", "bonds")}


def rand_mpo(L, D, d, dtype, seed):
    """Random (l, r, u, d) MPO host arrays, non-Hermitian when complex."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(L):
        shape = (1 if i == 0 else D, 1 if i == L - 1 else D, d, d)
        x = rng.standard_normal(shape)
        if np.dtype(dtype).kind == "c":
            x = x + 1j * rng.standard_normal(shape)
        out.append((x / (D * d) ** 0.5).astype(dtype))
    return out


def heis_lrud(L, dtype=np.float64):
    """``mps.mpo_ham_heis`` (layout 'lrdu') as (l, r, u, d) arrays."""
    return [np.ascontiguousarray(w.transpose(0, 1, 3, 2)).astype(dtype)
            for w in qb.mps.mpo_ham_heis(L)]


def overlap(bra, ket):
    """<bra|ket> of host (l, p, r) site lists."""
    E = np.ones((1, 1))
    for a, b in zip(bra, ket):
        E = np.einsum("xy,xpa,ypb->ab", E, a.conj(), b, optimize=True)
    return E.reshape(())


def check_golden_case(data, meta, case):
    """One fixture case on the device layer.  A truncating 'dm' case first
    checks, on the oracle's spectra of the same inputs, that each cut is
    decided far from the device eigh's noise (cutoff = 0 keeps everything)."""
    A, W = _inputs(data, meta, case)
    k = meta["cases"].index(case)
    if case["method"] == "dm" and case.get("cutoff", 1e-10) > 0:
        spectra = []
        onp.gate_with_mpo(A, W, spectra=spectra, **_kwargs(case))
        mb = case.get("max_bond")
        for w, nrm in spectra:
            check_dm_margin(w, nrm, w.size if mb is None else mb, case.get("cutoff", 1e-10))
    out = qb.mps_gate_with_mpo([qb.asarray(a) for a in A], [qb.asarray(w) for w in W],
                               **_kwargs(case))
    got = [_np(x) for x in out]
    assert [x.shape[2] for x in got[:-1]] == case["bonds"]
    vec = data[f"case{k}__vec"]
    np.testing.assert_allclose(onp.dense(got), vec, rtol=0, atol=1e-10 * np.max(np.abs(vec)))
    for i, s in enumerate(onp.schmidt_values(got)):
        ref = data[f"case{k}__S{i}"]
        np.testing.assert_allclose(s, ref, rtol=0, atol=1e-10 * ref[0])


def check_dm_margin(w, nrm, max_bond, cutoff):
    """The 'dm' truncation of one reduced density matrix (eigenvalues ``w``,
    descending; Frobenius norm ``nrm``) is decided far from the device
    eigh's absolute noise, eps |rho|_F: every kept eigenvalue lies above it,
    and the cut falls either in a gap wider than it (max_bond) or with the
    discarded weight ('rsum1') away from the threshold by more than the noise
    of the whole tail (cutoff)."""
    noise = 1e3 * np.finfo(np.float64).eps * nrm
    tail = np.cumsum(w[::-1])[::-1]                      # tail[n] = sum(w[n:])
    thr = cutoff * tail[0]
    n = int(np.argmax(np.append(tail, 0.0) <= thr))      # least n with sum(w[n:]) <= thr
    n = max(1, min(n, max_bond))
    assert w[n - 1] > noise, (n, w[n - 1], noise)
    if n == w.size or w[n] <= noise:
        return                                           # only noise is discarded
    if n == max_bond:
        assert w[n - 1] - w[n] > noise, (n, w[n - 1] - w[n], noise)
    else:
        margin = noise * w.size
        assert abs(tail[n] - thr) > margin and abs(tail[n - 1] - thr) > margin, (n, margin)


def check_against_oracle(L, chi, D, d, dtype, method, seed, mpo="rand"):
    """The device result against the oracle on one random MPS / MPO at
    ``max_bond = chi``: equal bonds, Schmidt values to 1e-10 of the largest,
    normalised fidelity within 1e-12 of 1.  For 'dm' every kept / discarded
    eigenvalue pair at the cut must be separated by far more than the device
    eigh's absolute accuracy, eps |rho|_F.

    The oracle takes the zip-up spanning tree from the code under test
    (``mpo_compress.ladder_tree_span``, host control logic); that tree is
    checked against the reference's ``get_tree_span`` only at the fixture
    sizes (L <= 12), so a tie-break that differs first at this length would
    not show here."""
    A = rand_mps(L, chi, d, dtype, seed)
    W = heis_lrud(L, dtype) if mpo == "heis" else rand_mpo(L, D, d, dtype, seed + 1)
    spectra = []
    want = onp.gate_with_mpo(A, W, method=method, max_bond=chi,
                             spectra=spectra if method == "dm" else None)
    for w, nrm in spectra:
        check_dm_margin(w, nrm, chi, 1e-10)
    out = qb.mps_gate_with_mpo([qb.asarray(a) for a in A], [qb.asarray(w) for w in W],
                               method=method, max_bond=chi)
    got = [_np(x) for x in out]
    assert [x.shape[2] for x in got] == [x.shape[2] for x in want]
    for s, r in zip(onp.schmidt_values(got), onp.schmidt_values(want)):
        np.testing.assert_allclose(s, r, rtol=0, atol=1e-10 * r[0])
    f = abs(overlap(got, want)) ** 2 / (overlap(got, got).real * overlap(want, want).real)
    assert abs(f - 1) < 1e-12, f


# ------------------------------------------------------------------ tests ---
def test_golden_matches_reference():
    data, meta = load_golden("mpo_compress")
    for case in meta["cases"]:
        check_golden_case(data, meta, case)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_scale_against_oracle(method, dtype):
    check_against_oracle(40, 128, 5, 2, dtype, method, seed=7,
                         mpo="heis" if dtype == np.float64 else "rand")


@pytest.mark.parametrize("method", METHODS)
def test_untruncated_equals_mpo_apply(method):
    """max_bond >= chi D_w and cutoff = 0: the uncompressed product, compared
    through mps_overlap (``mpo_apply`` contracts the MPO's upper index, i.e.
    ``transpose=True`` here)."""
    L, chi, D = 7, 4, 3
    A = rand_mps(L, chi, 2, np.complex128, 3)
    W = rand_mpo(L, D, 2, np.complex128, 4)
    psi = [qb.asarray(a) for a in A]
    mpo = [qb.asarray(w) for w in W]
    full = qb.tebd.mpo_apply(mpo, psi)
    got = qb.mps_gate_with_mpo(psi, mpo, method=method, max_bond=chi * D, cutoff=0.0,
                               transpose=True)
    ff = qb.tebd.mps_overlap(full, full).real
    for x, y in ((got, full), (got, got)):
        assert abs(qb.tebd.mps_overlap(x, y) - ff) <= 1e-12 * ff


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_canonical_form_and_info(method, sweep_reverse):
    L = 8
    A = rand_mps(L, 8, 2, np.complex128, 5)
    W = rand_mpo(L, 3, 2, np.complex128, 6)
    info = {}
    out = qb.mps_gate_with_mpo([qb.asarray(a) for a in A], [qb.asarray(w) for w in W],
                               method=method, max_bond=6, sweep_reverse=sweep_reverse,
                               info=info)
    c = L - 1 if sweep_reverse else 0
    assert info["cur_orthog"] == (c, c)
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


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
@pytest.mark.parametrize("method", METHODS)
def test_single_precision_keeps_dtype(dtype, method):
    L = 8
    A = rand_mps(L, 6, 2, dtype, 8)
    W = rand_mpo(L, 3, 2, dtype, 9)
    out = qb.mps_gate_with_mpo([qb.asarray(a) for a in A], [qb.asarray(w) for w in W],
                               method=method, max_bond=6)
    assert all(x.dtype == np.dtype(dtype) for x in out)
    wide = np.complex128 if np.dtype(dtype).kind == "c" else np.float64
    want = onp.gate_with_mpo([a.astype(wide) for a in A], [w.astype(wide) for w in W],
                             method=method, max_bond=6)
    got = [_np(x).astype(wide) for x in out]
    f = abs(overlap(got, want)) ** 2 / (overlap(got, got).real * overlap(want, want).real)
    assert abs(f - 1) < 1e-4, f


def test_mixed_dtypes_promote():
    L = 6
    A = rand_mps(L, 4, 2, np.float64, 10)
    W = rand_mpo(L, 3, 2, np.complex128, 11)
    out = qb.mps_gate_with_mpo([qb.asarray(a) for a in A], [qb.asarray(w) for w in W],
                               max_bond=8)
    assert all(x.dtype == np.complex128 for x in out)


@pytest.mark.parametrize("method", METHODS)
def test_inputs_unchanged(method):
    L = 8
    A = rand_mps(L, 8, 2, np.complex128, 12)
    W = rand_mpo(L, 4, 2, np.complex128, 13)
    psi = [qb.asarray(a) for a in A]
    mpo = [qb.asarray(w) for w in W]
    qb.mps_gate_with_mpo(psi, mpo, method=method, max_bond=5, normalize=True)
    for x, a in zip(psi, A):
        assert np.array_equal(_np(x), a)
    for x, w in zip(mpo, W):
        assert np.array_equal(_np(x), w)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("L", [1, 2])
def test_short_chains(method, L):
    A = rand_mps(L, 2, 3, np.complex128, 14)
    W = rand_mpo(L, 2, 3, np.complex128, 15)
    out = qb.mps_gate_with_mpo([qb.asarray(a) for a in A], [qb.asarray(w) for w in W],
                               method=method, max_bond=4)
    want = onp.gate_with_mpo(A, W, method=method, max_bond=4)
    got = [_np(x) for x in out]
    v, u = onp.dense(got), onp.dense(want)
    np.testing.assert_allclose(v, u, rtol=0, atol=1e-12 * np.max(np.abs(u)))


@pytest.mark.parametrize("method", METHODS)
def test_split_opts_override_defaults(method):
    """Extra split options override the methods' defaults as in the
    reference: an explicit default or ``renorm`` changes nothing, and 'direct'
    / 'zipup-first' reject options the direct sweep does not take."""
    L = 7
    A = rand_mps(L, 6, 2, np.complex128, 18)
    W = rand_mpo(L, 3, 2, np.complex128, 19)
    psi = [qb.asarray(a) for a in A]
    mpo = [qb.asarray(w) for w in W]
    extra = {"direct": dict(absorb="left", reduced="right"),
             "dm": dict(positive=1, absorb=None),
             "zipup": dict(absorb="left"),
             "zipup-first": dict(absorb="left")}[method]
    base = [_np(x) for x in qb.mps_gate_with_mpo(psi, mpo, method=method, max_bond=5)]
    for kw in (extra, dict(renorm=False)):
        got = [_np(x) for x in qb.mps_gate_with_mpo(psi, mpo, method=method, max_bond=5, **kw)]
        v, u = onp.dense(got), onp.dense(base)
        np.testing.assert_allclose(v, u, rtol=0, atol=1e-12 * np.max(np.abs(u)))
    if method in ("direct", "zipup-first"):
        with pytest.raises(TypeError, match="positive"):
            qb.mps_gate_with_mpo(psi, mpo, method=method, max_bond=5, positive=1)


def test_argument_errors():
    L = 5
    psi = [qb.asarray(a) for a in rand_mps(L, 4, 2, np.float64, 16)]
    mpo = [qb.asarray(w) for w in rand_mpo(L, 3, 2, np.float64, 17)]
    with pytest.raises(ValueError):
        qb.mps_gate_with_mpo(psi, mpo[:-1])
    with pytest.raises(ValueError):
        qb.mps_gate_with_mpo(psi, [qb.asarray(w) for w in rand_mpo(L, 3, 3, np.float64, 1)])
    with pytest.raises(ValueError):
        qb.mps_gate_with_mpo(psi, mpo, method="nope")
    with pytest.raises(ValueError):
        qb.mps_gate_with_mpo(psi, mpo, method="zipup-first", max_bond=4,
                             max_bond_oversample=0)
    with pytest.raises(ValueError):
        qb.mps_gate_with_mpo(psi, mpo, method="zipup-first", max_bond_oversample=1.5)
    for m in ("fit", "fit-zipup", "src", "src-oversample", "sdc", "srcmps", "projector",
              "autofit"):
        with pytest.raises(NotImplementedError, match=m):
            qb.mps_gate_with_mpo(psi, mpo, method=m)
    with pytest.raises(NotImplementedError):
        qb.mps_gate_with_mpo(psi, mpo, equalize_norms=True)
