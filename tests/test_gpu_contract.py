"""GPU tier: the CUDA contraction path (through the Python layer and the C
ABI) against the numpy oracle and the reference-generated golden vectors."""

import itertools

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from oracle import contract_np as cn
from tests import route_oracle as ro

pytestmark = pytest.mark.gpu

RTOL = 1e-12  # fp64 parity bar; BASELINE asks for 1e-10


def _rand(rng, shape, dtype):
    x = rng.standard_normal(shape)
    if dtype.startswith("complex"):
        x = x + 1j * rng.standard_normal(shape)
    return np.asarray(x, dtype=dtype)


def _close(a, b, tol=RTOL):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape
    if not b.size:
        return
    scale = max(1.0, float(np.max(np.abs(b))))
    assert np.max(np.abs(a - b)) <= tol * scale * 10


def test_golden_contractions(golden_contract):
    data, meta = golden_contract
    for name, m in meta.items():
        if name.startswith("_"):
            continue
        arrays = [qb.asarray(data[f"{name}__in{k}"]) for k in range(len(m["inds"]))]
        inds = [tuple(i) for i in m["inds"]]
        out_inds = m["output_inds"]
        if out_inds is None:
            out_inds = qb.gen_output_inds(itertools.chain.from_iterable(inds))
        assert list(out_inds) == m["result_inds"], name   # bit-exact bookkeeping
        out = qb.array_contract(arrays, inds, tuple(out_inds))
        _close(out.to_numpy(), data[f"{name}__out"])


def test_golden_strip_exponent(golden_contract):
    """strip_exponent / base exponent of tensor_contract (tensor_core.py:330-341)
    against the reference-generated mantissas; the scaled inputs (up to 1e160
    each) overflow double precision without stripping."""
    data, meta = golden_contract
    n = 0
    for name, m in meta.items():
        if name.startswith("_") or "strip" not in m:
            continue
        sc = m["strip"]["input_scales"]
        arrays = [qb.asarray(data[f"{name}__in{k}"] * 10.0 ** sc[k])
                  for k in range(len(m["inds"]))]
        keep = [a.to_numpy().copy() for a in arrays]
        (mant, e), inds_out = qb.tensor_contract(arrays, [tuple(i) for i in m["inds"]],
                                                 m["output_inds"], strip_exponent=True,
                                                 exponent=m["strip"]["base_exponent"])
        assert list(inds_out) == m["result_inds"]
        assert e == pytest.approx(m["strip"]["exponent"], abs=1e-8), name
        ref = data[f"{name}__strip_mantissa"]
        np.testing.assert_allclose(mant.to_numpy(), ref, rtol=1e-10, atol=1e-12)
        for a, k in zip(arrays, keep):                   # inputs are never scaled in place
            np.testing.assert_array_equal(a.to_numpy(), k)
        n += 1
    assert n >= 4
    # plain result scaled by a base exponent
    x = np.arange(6.0).reshape(2, 3)
    out, io = qb.tensor_contract([qb.asarray(x), qb.asarray(x.T.copy())], ["ab", "bc"], exponent=2.0)
    np.testing.assert_allclose(out.to_numpy(), 100.0 * x @ x.T)
    assert io == ("a", "c")


def test_strip_exponent_long_chain_no_overflow():
    """An unnormalised MPS-norm-like chain whose value (~1e600) is far outside
    double range: mantissa/exponent agree with the oracle."""
    rng = np.random.default_rng(3)
    mats = [rng.standard_normal((24, 24)) * 1e10 for _ in range(60)]
    inds = [(i, i + 1) for i in range(60)]
    (mant, e), _ = qb.tensor_contract([qb.asarray(x) for x in mats], inds, strip_exponent=True,
                                      optimize="greedy")
    (mo, eo), _ = cn.tensor_contract(mats, inds, strip_exponent=True, optimize="greedy")
    assert e > 600 and np.isfinite(e)
    # different trees -> compare the represented value
    shift = e - eo
    np.testing.assert_allclose(mant.to_numpy() * 10.0 ** shift, mo, rtol=1e-9, atol=1e-12)


CASES = [
    ("ab,bc->ac", dict(a=37, b=45, c=29)),
    ("ab,bc->ac", dict(a=300, b=257, c=190)),
    ("ba,bc->ac", dict(a=64, b=130, c=70)),
    ("ab,cb->ca", dict(a=33, b=65, c=17)),
    ("abcd,cdef->abef", dict(a=12, b=11, c=10, d=9, e=8, f=7)),
    ("acbd,dfce->abef", dict(a=12, b=11, c=10, d=9, e=8, f=7)),
    ("abcd,cdef->feba", dict(a=12, b=11, c=10, d=9, e=8, f=7)),
    ("gab,gbc->gac", dict(g=3, a=20, b=31, c=12)),
    ("agb,bcg->acg", dict(g=5, a=20, b=31, c=12)),
    ("ab,cd->abcd", dict(a=7, b=8, c=9, d=10)),
    ("abc,abc->", dict(a=30, b=40, c=50)),
    (",ab->ab", dict(a=5, b=6)),
    ("abe,bc->ac", dict(a=12, b=13, c=14, e=5)),
    ("ab,b->a", dict(a=1000, b=777)),
    ("a,a->", dict(a=1_000_003)),
    ("aab,bc->ac", dict(a=9, b=10, c=11)),          # diagonal of an operand
    ("abcdefg,cdexyz->abfgxyz", {c: 2 for c in "abcdefgxyz"}),
    ("xwa,asbt->xwsbt", dict(x=32, w=5, a=32, s=2, b=32, t=2)),
    ("xwsbt,wvsu->xvubt", dict(x=32, w=5, s=2, b=32, t=2, v=5, u=2)),
]


def _elementwise_bound(eq, sizes, a, b):
    """|C_kernel - C_numpy| <= 2 gamma_K (|A|.|B|) element by element (complex:
    2 sqrt(2) gamma_{2K+2}), K = number of summed terms: both results are
    inner products in some summation order (route_oracle.dmma_bound)."""
    lhs, rhs = eq.split("->")
    K = int(np.prod([sizes[c] for c in set(lhs.replace(",", "")) if c not in rhs]))
    absref = np.einsum(eq, np.abs(a), np.abs(b))
    if np.iscomplexobj(a):
        return 2 * np.sqrt(2) * ro.gamma(2 * K + 2) * absref * 1.001
    return 2 * ro.gamma(K) * absref * 1.001


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
@pytest.mark.parametrize("eq,sizes", CASES)
def test_pairwise_vs_oracle(eq, sizes, dtype):
    rng = np.random.default_rng(abs(hash(eq)) % 2**31)
    lhs, rhs = eq.split("->")
    ta, tb = lhs.split(",")
    a = _rand(rng, [sizes[c] for c in ta], dtype)
    b = _rand(rng, [sizes[c] for c in tb], dtype)
    ref = np.einsum(eq, a, b)
    out = qb.einsum(eq, qb.asarray(a), qb.asarray(b)).to_numpy()
    assert out.shape == ref.shape
    assert np.all(np.abs(out - ref) <= _elementwise_bound(eq, sizes, a, b))


def test_oracle_pair_executor_agrees():
    # the oracle's tensordot+transpose executor and the kernel on a pure pair
    rng = np.random.default_rng(5)
    a = rng.standard_normal((6, 4, 5, 3)); b = rng.standard_normal((3, 2, 4, 7))
    ref = cn.contract_pair(a, "acbd", b, "dfce", "abef")
    out = qb.array_contract([a, b], ["acbd", "dfce"], "abef")
    _close(out.to_numpy(), ref)


def test_tensordot_semantics():
    rng = np.random.default_rng(1)
    a = rng.standard_normal((5, 6, 7)); b = rng.standard_normal((7, 6, 4))
    A, B = qb.asarray(a), qb.asarray(b)
    _close(qb.tensordot(A, B, axes=1).to_numpy(), np.tensordot(a, b, axes=1))
    _close(qb.tensordot(A, B, axes=((1, 2), (1, 0))).to_numpy(),
           np.tensordot(a, b, axes=((1, 2), (1, 0))))
    _close(qb.tensordot(A, B, axes=0).to_numpy(), np.tensordot(a, b, axes=0))
    _close((A.reshape(30, 7) @ B.reshape(7, 24)).to_numpy(),
           a.reshape(30, 7) @ b.reshape(7, 24))
    with pytest.raises(ValueError):
        qb.tensordot(A, B, axes=((0,), (0,)))


def test_views_conj_transpose_are_free_and_correct():
    rng = np.random.default_rng(2)
    a = rng.standard_normal((9, 8, 7)) + 1j * rng.standard_normal((9, 8, 7))
    b = rng.standard_normal((7, 9, 5)) + 1j * rng.standard_normal((7, 9, 5))
    A, B = qb.asarray(a), qb.asarray(b)
    n0 = qb.launch_count()
    At = A.transpose(2, 0, 1).conj()       # no kernels
    Bs = B[::2, :, 1:]
    assert qb.launch_count() == n0
    out = qb.tensordot(At, Bs, axes=((1,), (1,)))
    assert qb.launch_count() == n0 + 1     # exactly one launch, no transposes
    ref = np.tensordot(a.transpose(2, 0, 1).conj(), b[::2, :, 1:], axes=((1,), (1,)))
    _close(out.to_numpy(), ref, 1e-11)
    # materialise through the permute kernel
    _close(qb.materialize(At).to_numpy(), a.transpose(2, 0, 1).conj())
    _close(At.reshape(7, 72).to_numpy(), a.transpose(2, 0, 1).conj().reshape(7, 72))


def test_alpha_beta_accumulate():
    rng = np.random.default_rng(3)
    a = rng.standard_normal((70, 40)); b = rng.standard_normal((40, 50))
    c = rng.standard_normal((70, 50))
    C = qb.asarray(c.copy())
    qb.contract_pair(qb.asarray(a).t, [0, 1], qb.asarray(b).t, [1, 2], [0, 2],
                     out=C.t, alpha=-0.5, beta=2.0)
    _close(C.to_numpy(), -0.5 * a @ b + 2.0 * c)


def test_edge_cases_empty_and_degenerate():
    A = qb.zeros((0, 4)); B = qb.ones((4, 3))
    assert qb.tensordot(A, B, axes=1).shape == (0, 3)
    A = qb.ones((3, 0)); B = qb.ones((0, 2))
    out = qb.tensordot(A, B, axes=1)
    assert out.shape == (3, 2) and float(abs(out).max().item()) == 0.0
    one = qb.ones(())
    s = qb.tensordot(one, one, axes=0)
    assert s.shape == () and s.item() == 1.0


def test_three_tensor_tree_and_expression():
    rng = np.random.default_rng(4)
    L = rng.standard_normal((7, 5, 7)); x = rng.standard_normal((7, 2, 2, 6))
    W1 = rng.standard_normal((5, 4, 2, 2)); W2 = rng.standard_normal((4, 3, 2, 2))
    R = rng.standard_normal((6, 3, 6))
    inputs = [("x", "w", "a"), ("a", "s", "t", "b"), ("w", "v", "s", "p"),
              ("v", "z", "t", "q"), ("y", "z", "b")]
    out_inds = ("x", "p", "q", "y")
    arrays = [L, x, W1, W2, R]
    ref = cn.array_contract(arrays, inputs, out_inds, "optimal")
    expr = qb.ContractExpression(inputs, out_inds, [a.shape for a in arrays],
                                 constants={0: L, 2: W1, 3: W2, 4: R})
    out = expr(qb.asarray(x))
    _close(out.to_numpy(), ref, 1e-11)
    out2 = qb.array_contract(arrays, inputs, out_inds, optimize="greedy")
    _close(out2.to_numpy(), ref, 1e-11)


def test_full_size_properties_chi1024():
    """BASELINE-size checks through size-independent properties."""
    chi, d = 1024, 2
    g = torch.Generator(device="cuda").manual_seed(0)
    A = qb.Array(torch.randn(chi, chi, d, dtype=torch.float64, device="cuda", generator=g))
    E1 = qb.Array(torch.randn(chi, chi, dtype=torch.float64, device="cuda", generator=g))
    E2 = qb.Array(torch.randn(chi, chi, dtype=torch.float64, device="cuda", generator=g))
    I = qb.eye(chi)
    # identity: I . A == A exactly (products with 0/1 are exact)
    out = qb.tensordot(I, A, axes=((1,), (0,)))
    assert float(abs(out - A).max().item()) == 0.0
    # linearity
    lhs = qb.tensordot(E1 * 0.5 + E2 * 2.0, A, axes=((1,), (0,)))
    rhs = qb.tensordot(E1, A, axes=((1,), (0,))) * 0.5 + qb.tensordot(E2, A, axes=((1,), (0,))) * 2.0
    assert float(abs(lhs - rhs).max().item()) < 1e-10
    # transpose symmetry: (E1 A)^T-contraction equals contraction of views
    a = qb.tensordot(E1, A, axes=((1,), (0,)))
    b = qb.tensordot(A.transpose(2, 1, 0), E1.T, axes=((2,), (0,))).transpose(2, 1, 0)
    assert float(abs(a - b).max().item()) < 1e-10


# ---- int8 (error-free split) engine -------------------------------------
OZ_CASES = [
    ("ab,bc->ac", dict(a=128, b=128, c=64)),
    ("ab,bc->ac", dict(a=1000, b=777, c=333)),
    ("ba,bc->ac", dict(a=300, b=200, c=150)),
    ("acbd,dfce->abef", dict(a=32, b=20, c=24, d=28, e=16, f=18)),
    ("xwa,asbt->xwsbt", dict(x=64, w=5, a=256, s=2, b=64, t=2)),
]


@pytest.mark.parametrize("eq,sizes", OZ_CASES)
def test_int8_engine_matches_oracle(eq, sizes):
    rng = np.random.default_rng(abs(hash(eq)) % 2**31)
    lhs, rhs = eq.split("->")
    ta, tb = lhs.split(",")
    a = _rand(rng, [sizes[c] for c in ta], "float64")
    b = _rand(rng, [sizes[c] for c in tb], "float64")
    sym = {c: i for i, c in enumerate(dict.fromkeys(ta + tb + rhs))}
    A, B = qb.asarray(a), qb.asarray(b)
    n0 = qb.launch_count()
    out = qb.contract_pair(A.t, [sym[c] for c in ta], B.t, [sym[c] for c in tb],
                           [sym[c] for c in rhs], engine=2)
    # rowmax + split for each operand, then the int8 GEMM: 5 launches
    assert qb.launch_count() - n0 == 5
    ref = np.einsum(eq, a, b)
    # fp64-level: error relative to max|row| max|col| sqrt(K)
    assert np.max(np.abs(out.cpu().numpy() - ref)) <= 1e-12 * np.max(np.abs(ref))


def test_int8_engine_badly_scaled_and_accumulate():
    rng = np.random.default_rng(8)
    a = rng.standard_normal((256, 384)) * np.logspace(-9, 9, 256)[:, None]
    b = rng.standard_normal((384, 192)) * np.logspace(-7, 7, 192)[None, :]
    c0 = rng.standard_normal((256, 192))
    C = qb.asarray(c0.copy())
    qb.contract_pair(qb.asarray(a).t, [0, 1], qb.asarray(b).t, [1, 2], [0, 2],
                     out=C.t, engine=2, alpha=1.0, beta=0.0)
    ref = a @ b
    scale = np.abs(a).max(1)[:, None] * np.abs(b).max(0)[None, :] * np.sqrt(384)
    assert np.max(np.abs(C.to_numpy() - ref) / scale) < 1e-14
    # small shapes silently use the exact DMMA engine
    small = qb.contract_pair(qb.asarray(a[:8, :16]).t, [0, 1], qb.asarray(b[:16, :8]).t,
                             [1, 2], [0, 2], engine=2)
    np.testing.assert_allclose(small.cpu().numpy(), a[:8, :16] @ b[:16, :8], rtol=1e-12, atol=1e-6)


def test_batched_small_contractions_one_launch():
    rng = np.random.default_rng(12)
    n = 37
    As = [rng.standard_normal((6, 5, 4)) for _ in range(n)]
    Bs = [rng.standard_normal((4, 5, 7)) for _ in range(n)]
    ta = [qb.asarray(a).t for a in As]
    tb = [qb.asarray(b).t for b in Bs]
    n0 = qb.launch_count()
    outs = qb.contract_batched(ta, [0, 1, 2], tb, [2, 1, 3], [3, 0])
    assert qb.launch_count() - n0 == 1
    for a, b, o in zip(As, Bs, outs):
        np.testing.assert_allclose(o.cpu().numpy(), np.einsum("abc,cbd->da", a, b), atol=1e-12)
    with pytest.raises(ValueError):
        qb.contract_batched(ta, [0, 1, 2], tb[:-1], [2, 1, 3], [3, 0])


def test_batched_complex_full_contracted_extent():
    """pointer-array batches of complex128 pairs sum over the whole contracted
    extent (the kernel counts k in real units: 2 per complex element)."""
    rng = np.random.default_rng(13)
    n = 9
    As = [rng.standard_normal((5, 40)) + 1j * rng.standard_normal((5, 40)) for _ in range(n)]
    Bs = [rng.standard_normal((40, 6)) + 1j * rng.standard_normal((40, 6)) for _ in range(n)]
    outs = qb.contract_batched([qb.asarray(a).t for a in As], [0, 1],
                               [qb.asarray(b).t for b in Bs], [1, 2], [0, 2])
    for a, b, o in zip(As, Bs, outs):
        np.testing.assert_allclose(o.cpu().numpy(), a @ b, atol=1e-12)


@pytest.mark.parametrize("dtype,tol", [("float32", 2e-6), ("complex64", 2e-6)])
def test_single_precision_dtype_preserved(dtype, tol):
    """f32 / c64 in -> same dtype out (reference: test_dmrg.py:290-300 dtype
    preservation), values at fp32 accuracy of the fp32 numpy result."""
    rng = np.random.default_rng(3)
    a = _rand(rng, (24, 18, 10), dtype); b = _rand(rng, (10, 18, 7), dtype)
    out = qb.einsum("abc,cbd->ad", qb.asarray(a), qb.asarray(b))
    assert out.dtype == np.dtype(dtype)
    ref = np.einsum("abc,cbd->ad", a.astype(np.result_type(dtype, np.float64)),
                    b.astype(np.result_type(dtype, np.float64)))
    assert np.max(np.abs(out.to_numpy() - ref)) <= tol * np.max(np.abs(ref))
    # views + conj
    out2 = qb.tensordot(qb.asarray(a).transpose(2, 1, 0).conj(), qb.asarray(b), axes=((0, 1), (0, 1)))
    ref2 = np.tensordot(a.transpose(2, 1, 0).conj(), b, axes=((0, 1), (0, 1)))
    assert out2.dtype == np.dtype(dtype)
    assert np.max(np.abs(out2.to_numpy() - ref2)) <= 10 * tol * np.max(np.abs(ref2))


# ---- native single precision / complex on the int8 engine ------------------
SINGLE_CASES = [
    ("ab,bc->ac", dict(a=256, b=192, c=160)),
    ("ba,bc->ca", dict(a=300, b=200, c=150)),
    ("apb,bqc->apqc", dict(a=130, p=2, b=140, q=2, c=70)),        # MPS-like
    ("xyab,abcd->xycd", dict(x=16, y=16, a=12, b=12, c=9, d=9)),  # boundary absorb-like
]


@pytest.mark.parametrize("dtype", ["float32", "complex64"])
@pytest.mark.parametrize("eq,sizes", SINGLE_CASES)
def test_native_single_precision_engine(eq, sizes, dtype):
    """float32 / complex64 contractions above the tile minimum run on the
    int8 engine directly (4 int8 slices, float epilogue): 5 launches, no
    conversion passes; result at fp32 accuracy of the exact product (the
    reference's numpy path rounds every partial sum to fp32, this rounds once)."""
    rng = np.random.default_rng(abs(hash(eq + dtype)) % 2**31)
    lhs, rhs = eq.split("->")
    ta, tb = lhs.split(",")
    a = _rand(rng, [sizes[c] for c in ta], dtype)
    b = _rand(rng, [sizes[c] for c in tb], dtype)
    sym = {c: i for i, c in enumerate(dict.fromkeys(ta + tb + rhs))}
    A, B = qb.asarray(a), qb.asarray(b)
    n0 = qb.launch_count()
    out = qb.contract_pair(A.t, [sym[c] for c in ta], B.t, [sym[c] for c in tb],
                           [sym[c] for c in rhs])
    assert qb.launch_count() - n0 == 5
    assert out.dtype == A.t.dtype
    wide = np.result_type(dtype, np.float64)
    ref = np.einsum(eq, a.astype(wide), b.astype(wide))
    assert np.max(np.abs(out.cpu().numpy() - ref)) <= 2e-6 * np.max(np.abs(ref))
    # conjugation flags are signs inside the split gather
    outc = qb.contract_pair(A.t, [sym[c] for c in ta], B.t, [sym[c] for c in tb],
                            [sym[c] for c in rhs], conj_a=True, conj_b=False)
    refc = np.einsum(eq, a.astype(wide).conj(), b.astype(wide))
    assert np.max(np.abs(outc.cpu().numpy() - refc)) <= 2e-6 * np.max(np.abs(refc))


def test_native_single_accumulate_and_strided_output():
    rng = np.random.default_rng(21)
    a = _rand(rng, (200, 150), "complex64"); b = _rand(rng, (150, 180), "complex64")
    c0 = _rand(rng, (180, 200), "complex64")
    C = qb.asarray(c0.copy())
    # out is written through its transpose (a strided view), accumulating
    qb.contract_pair(qb.asarray(a).t, [0, 1], qb.asarray(b).t, [1, 2], [0, 2],
                     out=C.t.t(), alpha=0.5, beta=2.0, conj_b=True)
    ref = 0.5 * (a.astype(np.complex128) @ b.astype(np.complex128).conj()) + 2.0 * c0.T
    assert np.max(np.abs(C.to_numpy().T - ref)) <= 3e-6 * np.max(np.abs(ref))


def test_int8_engine_complex128_embedding():
    """complex128 through the same engine (8 slices): the complex operands are
    embedded into the real GEMM inside the split gather."""
    rng = np.random.default_rng(22)
    a = _rand(rng, (160, 6, 40), "complex128"); b = _rand(rng, (40, 6, 130), "complex128")
    out = qb.contract_pair(qb.asarray(a).t, [0, 1, 2], qb.asarray(b).t, [2, 1, 3], [3, 0],
                           conj_a=True, engine=2)
    ref = np.einsum("abc,cbd->da", a.conj(), b)
    assert np.max(np.abs(out.cpu().numpy() - ref)) <= 1e-12 * np.max(np.abs(ref))


# ---- int8 engine edges: ragged tiles, the K limit, special values, range ----
_INT8_DTYPES = ["float32", "complex64", "float64", "complex128"]


def _int8_engine(dtype):
    # float32 / complex64 take it by default, float64 / complex128 on request
    return ro.ENGINE_INT8 if dtype in ("float64", "complex128") else 0


def _int8_route(M, K, N, dtype):
    return ro.route_of("ab,bc", M, K, N, dtype, _int8_engine(dtype))


def _run_int8(a, b, dtype, **kw):
    out = qb.contract_pair(torch.from_numpy(a).cuda(), [0, 1], torch.from_numpy(b).cuda(),
                           [1, 2], [0, 2], engine=_int8_engine(dtype), **kw)
    return out.cpu().numpy()


def _ragged_cases():
    for dtype in _INT8_DTYPES:
        ns = (32, 33) if dtype.startswith("complex") else (64, 65, 97)
        for M, N, K in itertools.product((128, 129, 255), ns, (128, 129, 255)):
            yield dtype, M, N, K


@pytest.mark.parametrize("dtype,M,N,K", list(_ragged_cases()))
def test_int8_engine_ragged_edges(dtype, M, N, K):
    """Extents around the 128-row tile, the output-column tile (64 float32 /
    32 float64 real columns; complex columns count twice) and the 128-byte
    k-block: exact on integer inputs, within the engine's bound on normal ones."""
    assert _int8_route(M, K, N, dtype)["kind"] == "int8"
    rng = np.random.default_rng(M * 7919 + N * 31 + K)
    a, b = ro.int_operand(rng, (M, K), dtype), ro.int_operand(rng, (K, N), dtype)
    np.testing.assert_array_equal(_run_int8(a, b, dtype), (ro.wide(a) @ ro.wide(b)).astype(dtype))
    a, b = ro.normal_operand(rng, (M, K), dtype), ro.normal_operand(rng, (K, N), dtype)
    got = ro.wide(_run_int8(a, b, dtype))
    bound = ro.int8_bound(a, b, dtype in ("float32", "complex64"))
    assert np.all(np.abs(got - ro.wide(a) @ ro.wide(b)) <= bound)


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_int8_engine_k_limit(dtype):
    """K = 65535 is the largest contracted extent whose int32 sums are proven
    exact; entries of magnitude 1 - 2^-8 (just below a power of two) make every
    first slice +-64 and the first accumulator of an all-positive row / column
    reach 65535 * 4096.  Exact oracle: the products have 17 significant bits
    and every partial sum stays below 2^16, so float64 numpy is exact.
    K = 65536 leaves the engine (float64: DMMA; float32: widened)."""
    M, N = 128, 64
    rng = np.random.default_rng(65535)
    for K, kind in ((65535, "int8"), (65536, "dmma" if dtype == "float64" else "widen")):
        assert _int8_route(M, K, N, dtype)["kind"] == kind
        v = 1.0 - 2.0 ** -8
        a = rng.choice([-v, v], size=(M, K))
        b = rng.choice([-v, v], size=(K, N))
        a[0], b[:, 0] = v, v
        ref = a @ b
        assert ref[0, 0] == K * v * v
        got = _run_int8(a.astype(dtype), b.astype(dtype), dtype)
        np.testing.assert_array_equal(got, ref.astype(dtype))


@pytest.mark.parametrize("dtype", _INT8_DTYPES)
def test_int8_engine_nonfinite_inputs(dtype):
    """NaN, +inf and -inf in A and B: the int8 slices cannot hold them, so the
    rows and columns that contain them are computed directly; every output
    element is in the IEEE class of the exact result and the finite ones keep
    the engine's bound."""
    M, K = 130, 200
    N = 40 if dtype.startswith("complex") else 70
    assert _int8_route(M, K, N, dtype)["kind"] == "int8"
    rng = np.random.default_rng(404)
    a, b = ro.plant_nonfinite(ro.normal_operand(rng, (M, K), dtype),
                              ro.normal_operand(rng, (K, N), dtype))
    got = ro.wide(_run_int8(a, b, dtype))
    ro.check_classes(a[None], b[None], got[None], int8=True)


def test_int8_engine_extreme_exponents():
    """float64 on the int8 engine across the exponent range: rows whose maximum
    is subnormal (2^-1030 ~ 1e-310) against columns near 2^1000, rows near
    2^1020 (~1e307) against columns near 2^-1020, all-zero rows and columns.
    Where the exact result is a normal number it meets the engine's bound;
    zero rows and columns give 0."""
    M, K, N = 130, 256, 70
    assert _int8_route(M, K, N, "float64")["kind"] == "int8"
    rng = np.random.default_rng(1015)
    ea = np.zeros(M, dtype=int)
    ea[:20], ea[20:40] = -1030, 1020
    eb = np.zeros(N, dtype=int)
    eb[:15], eb[15:30], eb[30:40] = -1020, 1000, -40
    a = np.ldexp(rng.standard_normal((M, K)), ea[:, None])
    b = np.ldexp(rng.standard_normal((K, N)), eb[None, :])
    a[40], b[:, 40] = 0.0, 0.0
    # the exact product of the inputs as given (subnormal rows keep fewer bits)
    a1, b1 = np.ldexp(a, -ea[:, None]), np.ldexp(b, -eb[None, :])
    with np.errstate(over="ignore"):     # results beyond the double range are not checked
        ref = np.ldexp(a1 @ b1, ea[:, None] + eb[None, :])
        bound = np.ldexp(ro.int8_bound(a1[None], b1[None], False)[0], ea[:, None] + eb[None, :])
    got = _run_int8(a, b, "float64")
    normal = np.isfinite(ref) & (np.abs(ref) >= np.finfo(np.float64).tiny)
    normal &= np.isfinite(bound)
    assert normal[:20].any() and normal[20:40, :15].all()
    assert np.all(np.abs(got[normal] - ref[normal]) <= bound[normal])
    assert np.all(got[40] == 0.0) and np.all(got[:, 40] == 0.0)
