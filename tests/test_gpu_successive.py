"""GPU tier: successive compression of an MPO-applied MPS
(``quimb_b200.successive``) and its sketch kernel ``qb_sketch_env``.

Checked against what the unmodified reference computed from the same noise
(tests/golden/successive.*: bond sizes, per-bond singular values and the
dense output), against the numpy oracle (oracle/successive_np.py) at
L = 40, chi = 128, and against the uncompressed ``tebd.mpo_apply`` product
when the sketch is at least the exact rank."""

import ctypes
import warnings

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from oracle import successive_np as onp
from quimb_b200 import _lib
from quimb_b200.successive import sketch_env
from tests.conftest import load_golden
from tests.test_gpu_mpo_compress import heis_lrud, overlap, rand_mpo
from tests.test_gpu_mps_sample import rand_mps

pytestmark = pytest.mark.gpu

METHODS = ("src", "src-oversample", "srcmps", "srcmps-oversample", "sdc", "sdc-oversample")


# ----------------------------------------------------------------- helpers ---
def _np(x):
    return np.asarray(x.to_numpy() if hasattr(x, "to_numpy") else x)


def _inputs(data, meta, case):
    L = meta["states"][case["state"]]["L"]
    A = [np.ascontiguousarray(data[f"{case['state']}__site{i}"]) for i in range(L)]
    W = [np.ascontiguousarray(data[f"{case['mpo']}__mpo{i}"]) for i in range(L)]
    return A, W


def _kwargs(data, meta, case):
    """The call's options: the stored sampling MPS for 'srcmps', a Generator
    where the case asked for one."""
    kw = {k: v for k, v in case.items()
          if k not in ("state", "mpo", "bonds", "fit", "seed_generator")}
    if case["method"].startswith("srcmps"):
        kw.pop("seed", None)
        n = meta["fits"][case["fit"]]["L"]
        kw["tn_fit"] = [data[f"{case['fit']}__fit{i}"] for i in range(n)]
    if case["method"].startswith("sdc"):
        kw.pop("seed", None)
    if case.get("seed_generator"):
        kw["seed"] = np.random.default_rng(case["seed"])
    return kw


def _fidelity(got, want):
    return abs(overlap(got, want)) ** 2 / (overlap(got, got).real * overlap(want, want).real)


def check_golden_case(data, meta, case, k):
    A, W = _inputs(data, meta, case)
    kw = _kwargs(data, meta, case)
    if "tn_fit" in kw:
        kw["tn_fit"] = [qb.asarray(f) for f in kw["tn_fit"]]
    out = qb.mps_gate_with_mpo_successive([qb.asarray(a) for a in A],
                                          [qb.asarray(w) for w in W], **kw)
    got = [_np(x) for x in out]
    assert [x.shape[2] for x in got[:-1]] == case["bonds"], case
    vec = data[f"case{k}__vec"]
    np.testing.assert_allclose(onp.dense(got), vec, rtol=0, atol=1e-10 * np.max(np.abs(vec)))
    for i, s in enumerate(onp.schmidt_values(got)):
        ref = data[f"case{k}__S{i}"]
        np.testing.assert_allclose(s, ref, rtol=0, atol=1e-10 * ref[0])


def check_against_oracle(L, chi, d, dtype, method, seed, mpo="heis"):
    """Device against oracle on one random MPS / MPO at max_bond = chi, the
    same noise and sampling MPS: equal bonds, Schmidt values to 1e-9 of the
    largest, normalised fidelity within 1e-10 of 1."""
    A = rand_mps(L, chi, d, dtype, seed)
    W = heis_lrud(L, dtype) if mpo == "heis" else rand_mpo(L, 3, d, dtype, seed + 1)
    F = None
    if method.startswith("srcmps"):
        k = chi if method == "srcmps" else qb.successive.oversample_bond(chi, None)
        F = qb.fit.random_guess_host([d] * L, k, dtype, seed + 2)
    want = onp.gate_with_mpo_successive(A, W, chi, method=method, seed=seed, tn_fit=F)
    out = qb.mps_gate_with_mpo_successive(
        [qb.asarray(a) for a in A], [qb.asarray(w) for w in W], chi, method=method, seed=seed,
        tn_fit=None if F is None else [qb.asarray(f) for f in F])
    got = [_np(x) for x in out]
    assert [x.shape[2] for x in got] == [x.shape[2] for x in want]
    for s, r in zip(onp.schmidt_values(got), onp.schmidt_values(want)):
        np.testing.assert_allclose(s, r, rtol=0, atol=1e-9 * r[0])
    f = _fidelity(got, want)
    assert abs(f - 1) < 1e-10, f


# ------------------------------------------------------------------ tests ---
def test_golden_matches_reference():
    data, meta = load_golden("successive")
    methods = set()
    for k, case in enumerate(meta["cases"]):
        check_golden_case(data, meta, case, k)
        methods.add(case["method"])
    assert methods == set(METHODS)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_scale_against_oracle(method, dtype):
    check_against_oracle(40, 128, 2, dtype, method, seed=7,
                         mpo="heis" if dtype == np.float64 else "rand")


@pytest.mark.parametrize("method", ["src", "sdc"])
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_exact_when_sketch_covers_the_rank(method, sweep_reverse):
    """max_bond at least the exact rank of every bond: the uncompressed
    product (``mpo_apply`` contracts the MPO's upper index)."""
    L, chi, D = 7, 4, 3
    A = rand_mps(L, chi, 2, np.complex128, 3)
    W = rand_mpo(L, D, 2, np.complex128, 4)
    psi = [qb.asarray(a) for a in A]
    mpo = [qb.asarray(w) for w in W]
    full = qb.tebd.mpo_apply(mpo, psi)
    got = qb.mps_gate_with_mpo_successive(psi, mpo, 2 * chi * D, method=method, cutoff=0.0,
                                          transpose=True, seed=1, sweep_reverse=sweep_reverse)
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
    out = qb.mps_gate_with_mpo_successive([qb.asarray(a) for a in A],
                                          [qb.asarray(w) for w in W], 6, method=method,
                                          sweep_reverse=sweep_reverse, info=info, seed=2)
    c = L - 1 if sweep_reverse else 0
    assert info["cur_orthog"] == (c, c)
    for i, x in enumerate(out):
        if i == c:
            continue
        x = _np(x)
        l, d, r = x.shape
        m = x.reshape(l * d, r) if i < c else x.reshape(l, d * r)
        g = m.conj().T @ m if i < c else m @ m.conj().T
        np.testing.assert_allclose(g, np.eye(g.shape[0]), rtol=0, atol=1e-12)


@pytest.mark.parametrize("method", ["src", "src-oversample", "srcmps"])
def test_seed_reproducible_and_inputs_unchanged(method):
    L = 8
    A = rand_mps(L, 8, 2, np.complex128, 12)
    W = rand_mpo(L, 4, 2, np.complex128, 13)
    psi = [qb.asarray(a) for a in A]
    mpo = [qb.asarray(w) for w in W]

    def run(seed):
        return [_np(x) for x in qb.mps_gate_with_mpo_successive(psi, mpo, 5, method=method,
                                                                seed=seed, normalize=True)]
    a, b = run(3), run(3)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    g1, g2 = run(np.random.default_rng(3)), run(np.random.default_rng(3))
    assert all(np.array_equal(x, y) for x, y in zip(g1, g2))
    c = run(4)
    assert not all(np.array_equal(x, y) for x, y in zip(a, c) if x.shape == y.shape)
    for x, v in zip(psi, A):
        assert np.array_equal(_np(x), v)
    for x, w in zip(mpo, W):
        assert np.array_equal(_np(x), w)


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
@pytest.mark.parametrize("method", ["src", "sdc", "srcmps-oversample"])
def test_single_precision_keeps_dtype(dtype, method):
    L = 8
    A = rand_mps(L, 6, 2, dtype, 8)
    W = rand_mpo(L, 3, 2, dtype, 9)
    wide = np.complex128 if np.dtype(dtype).kind == "c" else np.float64
    F = None
    if method.startswith("srcmps"):
        F = qb.fit.random_guess_host([2] * L, 16, wide, 1)
    out = qb.mps_gate_with_mpo_successive(
        [qb.asarray(a) for a in A], [qb.asarray(w) for w in W], 6, method=method, seed=1,
        tn_fit=None if F is None else [qb.asarray(f.astype(dtype)) for f in F])
    assert all(x.dtype == np.dtype(dtype) for x in out)
    want = onp.gate_with_mpo_successive(
        [a.astype(wide) for a in A], [w.astype(wide) for w in W], 6, method=method, seed=1,
        tn_fit=None if F is None else [f.astype(dtype).astype(wide) for f in F])
    f = _fidelity([_np(x).astype(wide) for x in out], want)
    assert abs(f - 1) < 1e-4, f


def test_mixed_dtypes_promote():
    L = 6
    A = rand_mps(L, 4, 2, np.float64, 10)
    W = rand_mpo(L, 3, 2, np.complex128, 11)
    out = qb.mps_gate_with_mpo_successive([qb.asarray(a) for a in A],
                                          [qb.asarray(w) for w in W], 8, seed=0)
    assert all(x.dtype == np.complex128 for x in out)


def test_argument_errors_and_warnings():
    L = 5
    psi = [qb.asarray(a) for a in rand_mps(L, 4, 2, np.float64, 16)]
    mpo = [qb.asarray(w) for w in rand_mpo(L, 3, 2, np.float64, 17)]
    f = qb.mps_gate_with_mpo_successive
    with pytest.raises(ValueError, match="unknown method"):
        f(psi, mpo, 4, method="src-nope")
    for m in ("src", "src-oversample", "srcmps-oversample", "sdc-oversample"):
        with pytest.raises(ValueError, match="max_bond"):
            f(psi, mpo, None, method=m)
    with pytest.raises(ValueError, match="noise mode"):
        f(psi, mpo, 4, noise_mode="nope")
    with pytest.raises(ValueError):
        f(psi, mpo, 4, noise_dist="nope", seed=0)
    with pytest.raises(ValueError):
        f(psi, mpo, 4, method="src-oversample", max_bond_oversample=0)
    with pytest.raises(ValueError):
        f(psi, mpo[:-1], 4)
    with pytest.raises(ValueError, match="tn_fit"):
        f(psi, mpo, 4, method="srcmps", tn_fit=psi[:-1])
    with pytest.raises(TypeError):
        f(psi, mpo, 4, method="src", absorb="left")
    with pytest.raises(NotImplementedError):
        f(psi, mpo, 4, equalize_norms=True)
    for kw, pat in ((dict(cutoff=1e-3), "`cutoff` is ignored"),
                    (dict(compress_opts={"absorb": "left"}), "`compress_opts` is ignored"),
                    (dict(canonize=False), "`canonize=False` is ignored")):
        with pytest.warns(UserWarning, match=pat):
            f(psi, mpo, 4, method="src", seed=0, **kw)
    for m in ("sdc", "sdc-oversample", "src-oversample", "srcmps"):
        with pytest.warns(UserWarning, match="canonize"):
            f(psi, mpo, 4, method=m, seed=0, canonize=False)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        for m in METHODS:
            f(psi, mpo, 4, method=m, seed=0)
    # the dispatcher keeps refusing these methods
    with pytest.raises(NotImplementedError):
        qb.mps_gate_with_mpo(psi, mpo, method="src")


# --------------------------------------------------------- the raw kernel ---
_DTYPES = [torch.float64, torch.complex128, torch.float32, torch.complex64]


def _rand(shape, dtype, gen):
    x = torch.randn(shape, dtype=torch.float64, generator=gen)
    if dtype.is_complex:
        x = torch.complex(x, torch.randn(shape, dtype=torch.float64, generator=gen))
    return x.to(dtype).cuda()


def _want(LE, W, Om):
    wide = torch.complex128 if LE.dtype.is_complex else torch.float64
    return torch.einsum("Bav,vuop,Bo->Baup", LE.cpu().to(wide), W.cpu().to(wide),
                        Om.cpu().to(wide))


@pytest.mark.parametrize("dtype", _DTYPES)
@pytest.mark.parametrize("shape", [(3, 5, 5, 5, 2, 2), (16, 130, 5, 5, 2, 2),
                                   (7, 33, 11, 9, 3, 4), (2, 300, 1, 70, 1, 3),
                                   (1, 1, 20, 1, 1, 1)])
def test_kernel_against_einsum(dtype, shape):
    """Contiguous operands, then permuted and strided views of larger
    buffers (including an expanded, stride-0 environment); bitwise repeats."""
    nB, na, nv, nu, no, np_ = shape
    gen = torch.Generator().manual_seed(sum(shape))
    LE = _rand((nB, na, nv), dtype, gen)
    W = _rand((nv, nu, no, np_), dtype, gen)
    Om = _rand((nB, no), dtype, gen)
    want = _want(LE, W, Om)
    tol = 1e-12 if dtype in (torch.float64, torch.complex128) else 1e-5
    scale = want.abs().max().item()
    H = sketch_env(LE, W, Om)
    assert torch.allclose(H.cpu().to(want.dtype), want, rtol=0, atol=tol * scale)
    assert torch.equal(H, sketch_env(LE, W, Om))
    LEp = _rand((nv, nB, 2, na), dtype, gen)[:, :, 1, :].permute(1, 2, 0)
    Wp = _rand((np_, no, 2 * nu, nv), dtype, gen)[:, :, ::2, :].permute(3, 2, 1, 0)
    Omp = _rand((no, nB), dtype, gen).t()
    Hp = sketch_env(LEp, Wp, Omp)
    wp = _want(LEp, Wp, Omp)
    assert torch.allclose(Hp.cpu().to(wp.dtype), wp, rtol=0,
                          atol=tol * wp.abs().max().item())
    unit = torch.ones((1, 1, 1), dtype=dtype, device="cuda").expand(nB, 1, 1)
    Wu = _rand((1, nu, no, np_), dtype, gen)
    Hu = sketch_env(unit, Wu, Om)
    wu = _want(unit, Wu, Om)
    assert torch.allclose(Hu.cpu().to(wu.dtype), wu, rtol=0, atol=tol * wu.abs().max().item())


def test_kernel_one_launch_stream_and_nonfinite():
    gen = torch.Generator().manual_seed(5)
    LE = _rand((8, 40, 5), torch.complex128, gen)
    W = _rand((5, 5, 2, 2), torch.complex128, gen)
    Om = _rand((8, 2), torch.complex128, gen)
    ref = sketch_env(LE, W, Om)
    n0 = qb.launch_count()
    sketch_env(LE, W, Om)
    assert qb.launch_count() - n0 == 1
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        other = sketch_env(LE, W, Om)
    s.synchronize()
    assert torch.equal(ref, other)
    LE2 = LE.clone()
    LE2[3, 7, 2] = float("nan")
    W2 = W.clone()
    W2[1, 4, 0, 1] = float("inf")
    H = sketch_env(LE2, W2, Om).cpu()
    assert torch.isnan(H[3, 7]).all()
    assert not torch.isfinite(H[:, :, 4, 1]).any()
    assert torch.isfinite(H[0, 0, 0, 0])


def test_kernel_error_codes():
    lib = _lib.load()
    arr3, arr4, arr2 = ctypes.c_int64 * 3, ctypes.c_int64 * 4, ctypes.c_int64 * 2
    buf = torch.zeros(64, dtype=torch.float64, device="cuda")
    p = buf.data_ptr()
    s3, s4, s2 = arr3(1, 1, 1), arr4(1, 1, 1, 1), arr2(1, 1)
    n0 = qb.launch_count()
    assert lib.qb_sketch_env(9, 1, 1, 1, 1, 1, 1, p, s3, p, s4, p, s2, p, s4, None) == -1
    assert lib.qb_sketch_env(_lib.QB_F64, 0, 1, 1, 1, 1, 1, p, s3, p, s4, p, s2, p, s4,
                             None) == -2
    assert lib.qb_sketch_env(_lib.QB_F64, 1, 1, 1, 1, 1, 1, None, s3, p, s4, p, s2, p, s4,
                             None) == -3
    assert lib.qb_sketch_env(_lib.QB_C128, 1, 1, 1, 1, 1, 1, p + 8, s3, p, s4, p, s2, p, s4,
                             None) == -3
    assert lib.qb_sketch_env(_lib.QB_F64, 1, 1, 1, 1, 1, 1, p, None, p, s4, p, s2, p, s4,
                             None) == -3
    assert lib.qb_sketch_env(_lib.QB_F64, 2 ** 31, 2 ** 20, 1, 1, 1, 1, p, s3, p, s4, p, s2, p,
                             s4, None) == -4
    assert qb.launch_count() == n0
    assert "qb_sketch_env" in _lib.last_error()
