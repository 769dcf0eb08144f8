"""GPU tier: the HBM-bound vector kernels (csrc/elementwise.cu, csrc/convert.cu)
through the C ABI on torch buffers, against exact references.

Reference arithmetic:
- integer inputs |x| <= 2^10 and n <= 2^22 + 3: every partial sum of
  products is an integer below 2^53, so float64 results are exact in any
  summation order and the kernels must match bit for bit (float32 results:
  the exact value rounded once, since the kernels accumulate in double);
- random-normal inputs: ``route_oracle.exact_dot`` (the correctly rounded
  sum), with the kernel within gamma_n sum |x_i y_i| of it.

Sizes straddle a 256-thread block, the fixed 592-block grids of the two-stage
reductions and the 8 * SMs block cap of the element-wise grids, up to the
32 MiB vector of the benchmark.  Inputs sit in NaN-padded buffers (a stray
read poisons the result) and outputs in buffers of a sentinel bit pattern
that must survive outside the written range.

The last test records the Krylov basis of one Lanczos cycle and checks it is
orthonormal and that the returned Ritz value is the one of V^T A V: Lanczos
corrects its own errors, so a wrong Gram-Schmidt kernel still converges and
only shows up there.
"""

import ctypes
import warnings

import numpy as np
import pytest
import torch

from quimb_b200 import _lib, lanczos, ops
from quimb_b200.array import Array
from tests import route_oracle as ro

pytestmark = pytest.mark.gpu

DTYPES = ["float32", "float64", "complex64", "complex128"]
REAL_OF = {"float32": "float32", "float64": "float64", "complex64": "float32",
           "complex128": "float64"}
PAD = 40            # elements of padding on either side of every buffer
LIM = 2 ** 10
EPS = 2.0 ** -52


@pytest.fixture(scope="module")
def sizes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g, e = 592 * 256, 8 * sms * 256
    return [1, 255, 256, 257, g - 1, g + 1, e - 1, e + 1, 2 ** 22 + 3]


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _st():
    return _lib.stream_ptr()


def _pair(z):
    return (ctypes.c_double * 2)(float(np.real(z)), float(np.imag(z)))


def _in(x):
    """Device copy of numpy `x` (1-d) inside a NaN-filled buffer."""
    buf = ro.nan_fill(torch.empty(x.size + 2 * PAD, dtype=ro.TORCH[str(x.dtype)],
                                  device="cuda"))
    view = buf[PAD:PAD + x.size]
    view.copy_(torch.from_numpy(np.ascontiguousarray(x).ravel()))
    return view


def _out(n, dtype, init=None):
    """(buffer, view of n elements) in a sentinel-filled buffer; `init`
    (numpy) is copied into the view."""
    buf = torch.empty(n + 2 * PAD, dtype=ro.TORCH[dtype], device="cuda")
    ro.bits(buf).fill_(ro.BITS[dtype][1])
    view = buf[PAD:PAD + n]
    if init is not None:
        view.copy_(torch.from_numpy(np.ascontiguousarray(init)))
    return buf, view


def _check_pads(buf, n, dtype):
    mask = np.zeros(buf.numel(), dtype=bool)
    mask[PAD:PAD + n] = True
    ro.assert_sentinel_kept(buf, mask, dtype)


def _ints(rng, n, dtype, lim=LIM):
    return ro.int_operand(rng, (n,), dtype, lim)


def _exact_int_dot(x, y):
    """conj(x) . y of integer-valued arrays as Python ints (per part)."""
    xr, yr = np.real(x).astype(np.int64), np.real(y).astype(np.int64)
    if not np.iscomplexobj(x):
        return int(xr @ yr), 0
    xi, yi = np.imag(x).astype(np.int64), np.imag(y).astype(np.int64)
    return int(xr @ yr + xi @ yi), int(xr @ yi - xi @ yr)


def _as(dtype, re, im=0.0):
    """Exact value (Python ints / floats, exact in float64) rounded once to `dtype`."""
    if dtype.startswith("complex"):
        r = np.dtype(REAL_OF[dtype]).type
        return np.array(complex(r(float(re)), r(float(im))), dtype=dtype)
    return np.array(float(re), dtype=dtype)


def _same_bits(got, want):
    got, want = np.atleast_1d(got), np.atleast_1d(want)
    if np.iscomplexobj(got):
        got, want = got.view(REAL_OF[str(got.dtype)]), want.view(REAL_OF[str(want.dtype)])
    return np.array_equal(got.view(f"u{got.itemsize}"), want.view(f"u{want.itemsize}"))


# ---- qb_dot -------------------------------------------------------------------
def _dot(lib, dtype, x, y, n=None):
    n = x.numel() if n is None else n
    ws = torch.empty(lib.qb_dot_workspace(n), dtype=torch.uint8, device="cuda")
    buf, out = _out(1, dtype)
    rc = lib.qb_dot(ro.QB_DTYPE[dtype], n, x.data_ptr(), y.data_ptr(), out.data_ptr(),
                    ws.data_ptr(), _st())
    _lib.check(rc, "qb_dot")
    _check_pads(buf, 1, dtype)
    return out.cpu().numpy()[0]


@pytest.mark.parametrize("dtype", DTYPES)
def test_dot_exact_bounded_and_deterministic(lib, sizes, dtype):
    rng = np.random.default_rng(DTYPES.index(dtype))
    cplx = dtype.startswith("complex")
    u_out = 2.0 ** -24 if REAL_OF[dtype] == "float32" else 0.0
    for n in sizes:
        x, y = _ints(rng, n, dtype), _ints(rng, n, dtype)
        got = _dot(lib, dtype, _in(x), _in(y))
        want = _as(dtype, *_exact_int_dot(x, y))
        assert _same_bits(got, want), (n, got, want)

        x, y = ro.normal_operand(rng, (n,), dtype), ro.normal_operand(rng, (n,), dtype)
        X, Y = _in(x), _in(y)
        got = _dot(lib, dtype, X, Y)
        exact, scale = ro.exact_vdot(x, y)
        bound = ro.gamma(2 * n if cplx else n) * scale
        bound += u_out * (abs(exact) + bound)
        for g, e in ((got.real, exact.real), (got.imag, exact.imag)):
            assert abs(float(g) - e) <= bound, (n, float(g), e, bound)
        if n == sizes[-1]:
            assert _same_bits(_dot(lib, dtype, X, Y), got), "repeated dot differs"
    # n = 0: an empty sum
    assert _dot(lib, dtype, _in(np.ones(1, dtype)), _in(np.ones(1, dtype)), n=0) == 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_dot_nonfinite_classes(lib, dtype):
    """NaN, +-inf and inf * 0 inputs: the output has the IEEE class of the
    exact sum (per part for complex)."""
    rng = np.random.default_rng(11)
    n = 5000
    cases = [{5: (np.nan, 1.0)}, {5: (np.inf, 2.0)}, {5: (np.inf, -2.0)},
             {n - 1: (-np.inf, 3.0)}, {5: (np.inf, 0.0)},
             {5: (np.inf, 1.0), 4000: (-np.inf, 1.0)}, {7: (1.0, np.inf), 8: (2.0, np.inf)}]
    for case in cases:
        x, y = ro.normal_operand(rng, (n,), dtype), ro.normal_operand(rng, (n,), dtype)
        for i, (xv, yv) in case.items():
            x[i], y[i] = xv, yv
        got = _dot(lib, dtype, _in(x), _in(y))
        a, b = ro.wide(x).conj()[None, :], ro.wide(y)[:, None]
        want = ro.nonfinite_class(a, b)
        if dtype.startswith("complex"):
            assert ro.classify(got.real) == want[0][0, 0], (case, got)
            assert ro.classify(got.imag) == want[1][0, 0], (case, got)
        else:
            assert ro.classify(got) == want[0, 0], (case, got)


# ---- qb_multi_dot / qb_multi_axpy --------------------------------------------
def _basis(rng, n, ldv, lim=LIM):
    """16 x ldv float64 host matrix: integer rows, NaN in every row's gap."""
    V = np.full((16, ldv), np.nan)
    V[:, :n] = rng.integers(-lim, lim + 1, size=(16, n))
    return V


def _dev(x):
    """Device copy of a host array (any shape) at offset PAD of a NaN buffer."""
    return _in(x.ravel())


def _ldvs(n, sizes):
    return (n + 37,) if n == sizes[-1] else (n, n + 1, n + 37)


def _ms(n):
    return range(1, 17) if n < 2 ** 20 else (1, 2, 15, 16)


def _multi_dot(lib, m, n, V, ldv, w, ws):
    buf, out = _out(16, "float64")
    rc = lib.qb_multi_dot(_lib.QB_F64, m, n, V.data_ptr(), ldv, w.data_ptr(),
                          out.data_ptr(), ws.data_ptr(), _st())
    _lib.check(rc, "qb_multi_dot")
    mask = np.zeros(buf.numel(), dtype=bool)
    mask[PAD:PAD + m] = True
    ro.assert_sentinel_kept(buf, mask, "float64")
    return out.cpu().numpy()[:m]


def test_multi_dot(lib, sizes):
    rng = np.random.default_rng(21)
    ws = torch.empty(lib.qb_multi_dot_workspace(), dtype=torch.uint8, device="cuda")
    for n in sizes:
        w = rng.integers(-LIM, LIM + 1, size=n).astype(np.float64)
        W = _in(w)
        for ldv in _ldvs(n, sizes):
            V = _basis(rng, n, ldv)
            Vd = _dev(V)
            ref = V[:, :n] @ w                  # exact: integer partial sums < 2^53
            for m in _ms(n):
                got = _multi_dot(lib, m, n, Vd, ldv, W, ws)
                np.testing.assert_array_equal(got, ref[:m], err_msg=f"n={n} ldv={ldv} m={m}")
    # a NaN in row j poisons out[j] only
    n, ldv = 257, 258
    V = _basis(rng, n, ldv)
    w = rng.integers(-LIM, LIM + 1, size=n).astype(np.float64)
    ref = V[:, :n] @ w
    for j in (0, 9, 15):
        Vj = V.copy()
        Vj[j, n // 2] = np.nan
        got = _multi_dot(lib, 16, n, _dev(Vj), ldv, _in(w), ws)
        assert np.isnan(got[j])
        np.testing.assert_array_equal(np.delete(got, j), np.delete(ref, j))
    # bit-identical on repeat (random normals, grid-wrapping length)
    n = sizes[5]
    Vd = _dev(rng.standard_normal((16, n)))
    W = _in(rng.standard_normal(n))
    first = _multi_dot(lib, 16, n, Vd, n, W, ws)
    assert _same_bits(_multi_dot(lib, 16, n, Vd, n, W, ws), first)
    for m in (0, 17):
        rc = lib.qb_multi_dot(_lib.QB_F64, m, n, Vd.data_ptr(), n, W.data_ptr(),
                              W.data_ptr(), ws.data_ptr(), _st())
        assert rc == -2


def test_multi_axpy(lib, sizes):
    """w += alpha * sum_{j<m} h[j] V[j], h read at a nonzero device offset
    (as ``lanczos._combine`` passes coeffs[j0:]); exact on integers, nothing
    outside w[:n] written."""
    rng = np.random.default_rng(31)
    h = rng.integers(1, 9, size=16) * rng.choice([-1.0, 1.0], size=16)   # all nonzero
    hbuf = ro.nan_fill(torch.empty(16 + 5, dtype=torch.float64, device="cuda"))
    hbuf[5:].copy_(torch.from_numpy(h))
    hdev = hbuf[5:]
    for n in sizes:
        w0 = rng.integers(-LIM, LIM + 1, size=n).astype(np.float64)
        for ldv in _ldvs(n, sizes):
            V = _basis(rng, n, ldv)
            Vd = _dev(V)
            for alpha in (1.0, -1.0, 0.5):
                for m in _ms(n):
                    buf, w = _out(n, "float64", w0)
                    rc = lib.qb_multi_axpy(_lib.QB_F64, m, n, Vd.data_ptr(), ldv,
                                           hdev.data_ptr(), alpha, w.data_ptr(), _st())
                    _lib.check(rc, "qb_multi_axpy")
                    want = w0 + (alpha * h[:m]) @ V[:m, :n]
                    np.testing.assert_array_equal(w.cpu().numpy(), want,
                                                  err_msg=f"n={n} ldv={ldv} m={m} a={alpha}")
                    _check_pads(buf, n, "float64")
    for m in (0, 17):
        assert lib.qb_multi_axpy(_lib.QB_F64, m, 4, Vd.data_ptr(), 4, hdev.data_ptr(), 1.0,
                                 w.data_ptr(), _st()) == -2


# ---- axpby / scale / scale_into / scale_diag -----------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_axpby(lib, sizes, dtype):
    rng = np.random.default_rng(41 + DTYPES.index(dtype))
    cplx = dtype.startswith("complex")
    alpha, beta = (3 - 2j, -1 + 2j) if cplx else (3.0, -1.0)
    for n in sizes:
        x, y = _ints(rng, n, dtype), _ints(rng, n, dtype)
        buf, Y = _out(n, dtype, y)
        rc = lib.qb_axpby(ro.QB_DTYPE[dtype], n, _pair(alpha), _in(x).data_ptr(),
                          _pair(beta), Y.data_ptr(), _st())
        _lib.check(rc, "qb_axpby")
        want = (alpha * ro.wide(x) + beta * ro.wide(y)).astype(dtype)
        np.testing.assert_array_equal(Y.cpu().numpy(), want, err_msg=f"n={n}")
        _check_pads(buf, n, dtype)
        # beta = 0: y is not read (NaN-filled y gives a finite result)
        Yn = _in(np.full(n, np.nan, dtype=dtype))
        rc = lib.qb_axpby(ro.QB_DTYPE[dtype], n, _pair(alpha), _in(x).data_ptr(),
                          _pair(0.0), Yn.data_ptr(), _st())
        _lib.check(rc, "qb_axpby")
        np.testing.assert_array_equal(Yn.cpu().numpy(), (alpha * ro.wide(x)).astype(dtype))


def _scalar(v, dtype):
    """Device divisor in the real type of `dtype`."""
    return torch.tensor([v], dtype=ro.TORCH[REAL_OF[dtype]], device="cuda")


@pytest.mark.parametrize("dtype", DTYPES)
def test_scale_and_scale_into(lib, sizes, dtype):
    rng = np.random.default_rng(51 + DTYPES.index(dtype))
    cplx = dtype.startswith("complex")
    code = ro.QB_DTYPE[dtype]
    for n in sizes:
        x = _ints(rng, n, dtype)
        xw = ro.wide(x)
        # (alpha, divisor or None, exact factor)
        cases = [(3.0, 4.0, 0.75), (2.0, None, 2.0), (3.0, 0.0, 0.0)]
        if cplx:
            cases += [(3 - 2j, 2.0, 1.5 - 1j), (1 + 1j, 0.0, 0.0)]
        for alpha, div, f in cases:
            buf, X = _out(n, dtype, x)
            d = _scalar(div, dtype) if div is not None else None
            rc = lib.qb_scale(code, n, _pair(alpha), d.data_ptr() if d is not None else None,
                              X.data_ptr(), _st())
            _lib.check(rc, "qb_scale")
            np.testing.assert_array_equal(X.cpu().numpy(), (xw * f).astype(dtype),
                                          err_msg=f"n={n} alpha={alpha} div={div}")
            _check_pads(buf, n, dtype)
        for alpha, div, f in ((3.0, 8.0, 0.375), (-1.0, None, -1.0), (5.0, 0.0, 0.0)):
            buf, Y = _out(n, dtype)
            d = _scalar(div, dtype) if div is not None else None
            rc = lib.qb_scale_into(code, n, alpha, d.data_ptr() if d is not None else None,
                                   _in(x).data_ptr(), Y.data_ptr(), _st())
            _lib.check(rc, "qb_scale_into")
            np.testing.assert_array_equal(Y.cpu().numpy(), (xw * f).astype(dtype),
                                          err_msg=f"n={n} alpha={alpha} div={div}")
            _check_pads(buf, n, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_scale_diag(lib, sizes, dtype):
    """x *= d[col]^p (side 1) or d[row]^p (side 0), p in {1, 1/2}; d is a
    power of 4, so its square root is exact."""
    rng = np.random.default_rng(61 + DTYPES.index(dtype))
    shapes = [(1, n) for n in sizes] + [(n, 1) for n in sizes] + [(37, 41)]
    for rows, cols in shapes:
        x = ro.int_operand(rng, (rows, cols), dtype, LIM)
        for side in (0, 1):
            k = rng.integers(-3, 4, size=cols if side else rows)
            d = np.ldexp(1.0, 2 * k).astype(REAL_OF[dtype])
            for sq in (0, 1):
                buf, X = _out(rows * cols, dtype, x.ravel())
                rc = lib.qb_scale_diag(ro.QB_DTYPE[dtype], rows, cols, X.data_ptr(),
                                       _in(d).data_ptr(), side, sq, _st())
                _lib.check(rc, "qb_scale_diag")
                f = np.ldexp(1.0, k) if sq else np.ldexp(1.0, 2 * k)
                want = ro.wide(x) * (f[None, :] if side else f[:, None])
                np.testing.assert_array_equal(X.cpu().numpy().reshape(rows, cols),
                                              want.astype(dtype),
                                              err_msg=f"{rows}x{cols} side={side} sqrt={sq}")
                _check_pads(buf, rows * cols, dtype)


# ---- qb_permute ---------------------------------------------------------------------
def _permute(lib, src, dst, conj=0):
    return lib.qb_permute(_lib.desc(src), _lib.desc(dst), conj, _st())


def _random_bits(rng, shape, dtype):
    """Arbitrary bit patterns (NaN payloads, subnormals, infinities) with
    -0.0 planted, as a device tensor of `dtype`."""
    it, _ = ro.BITS[dtype]
    nreal = int(np.prod(shape)) * (2 if dtype.startswith("complex") else 1)
    npdt = np.int32 if it == torch.int32 else np.int64
    b = rng.integers(np.iinfo(npdt).min, np.iinfo(npdt).max, size=nreal, dtype=npdt)
    b[::7] = np.array(-0.0, dtype=REAL_OF[dtype]).view(npdt)
    t = torch.from_numpy(b).cuda().view(ro.TORCH[REAL_OF[dtype]])
    if dtype.startswith("complex"):
        t = torch.view_as_complex(t.view(-1, 2))
    return t.view(shape)


def _host_bits(t):
    return ro.bits(t.contiguous()).cpu().numpy()


@pytest.mark.parametrize("dtype", DTYPES)
def test_permute_bitwise_edges(lib, dtype):
    """A bitwise copy through both kernels (tiled transpose, row copy): NaN
    payloads and -0.0 survive; extents 31/32/33 around the 32-wide tile, a
    stride-0 source, an output view with gaps, a base one element off, and
    conjugation on both kernels."""
    rng = np.random.default_rng(71 + DTYPES.index(dtype))
    sent = ro.BITS[dtype][1]
    cplx = dtype.startswith("complex")
    for p in (31, 32, 33):
        for q in (31, 32, 33):
            base = _random_bits(rng, (3 * p * q + 1,), dtype)
            s3 = base[1:].view(3, p, q)                       # one element off
            for src, what in ((s3.permute(0, 2, 1), "tiled"), (s3.permute(1, 0, 2), "rows"),
                              (s3[0].t(), "tiled 2-d"),
                              (base[1:q + 1].view(1, q).expand(p, q), "stride-0 rows of a row"),
                              (base[1:q + 1].view(q, 1).expand(q, p), "stride-0 copies of a column")):
                # output view with gaps: every other row, columns 1.. of a wider buffer
                shp = tuple(src.shape)
                obuf = torch.empty(shp[:-2] + (2 * shp[-2], shp[-1] + 3),
                                   dtype=ro.TORCH[dtype], device="cuda")
                ro.bits(obuf).fill_(sent)
                dst = obuf[..., ::2, 1:1 + shp[-1]]
                for conj in ((0, 1) if cplx else (0,)):
                    assert _permute(lib, src, dst, conj) == 0, _lib.last_error()
                    want = _host_bits(src)
                    if conj:                 # IEEE negate of the imaginary part: sign bit only
                        want[..., 1] ^= np.array(1, want.dtype) << (8 * want.itemsize - 1)
                    assert np.array_equal(_host_bits(dst), want), (what, p, q, conj)
                    mask = np.zeros(obuf.shape, dtype=bool)
                    mask[..., ::2, 1:1 + shp[-1]] = True
                    ro.assert_sentinel_kept(obuf, mask, dtype)


def test_permute_mode_limit_and_empty(lib):
    """16 jointly non-mergeable rest modes are taken, 17 are refused with -100
    (the message the host layer keys its regrouping on); a zero-size copy
    launches nothing."""
    rng = np.random.default_rng(81)
    for tiled in (False, True):
        for rest, ok in ((16, True), (17, False)):
            # reversed axes never merge; the row kernel keeps the last axis in place
            nax = rest + (2 if tiled else 1)
            x = _random_bits(rng, (2,) * (nax - 1) + (3,), "float64")
            perm = list(range(nax))[::-1] if tiled else list(range(nax - 1))[::-1] + [nax - 1]
            src = x.permute(perm)
            dst = torch.empty(src.shape, dtype=torch.float64, device="cuda")
            rc = _permute(lib, src, dst)
            if ok:
                assert rc == 0, _lib.last_error()
                assert np.array_equal(_host_bits(dst), _host_bits(src))
            else:
                assert rc == -100 and "non-mergeable" in _lib.last_error()
    e = torch.empty((0, 5), dtype=torch.float64, device="cuda")
    n0 = _lib.launch_count()
    assert _permute(lib, e.t(), torch.empty((5, 0), dtype=torch.float64, device="cuda")) == 0
    assert _lib.launch_count() == n0


# ---- qb_convert ---------------------------------------------------------------------
def _convert(lib, x, dst_dtype):
    n = x.size
    buf, out = _out(n, dst_dtype)
    rc = lib.qb_convert(ro.QB_DTYPE[str(x.dtype)], ro.QB_DTYPE[dst_dtype], n,
                        _in(x).data_ptr(), out.data_ptr(), _st())
    _lib.check(rc, "qb_convert")
    _check_pads(buf, n, dst_dtype)
    return out.cpu().numpy()


def _same_or_both_nan(got, want):
    got, want = np.asarray(got), np.asarray(want)
    if np.iscomplexobj(got):
        return (_same_or_both_nan(got.real, want.real)
                and _same_or_both_nan(got.imag, want.imag))
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and _same_bits(got[~nan], want[~nan])


def _narrowing_edges():
    fmax = float(np.finfo(np.float32).max)
    tiny = 2.0 ** -149                      # smallest float32 subnormal
    half_up = fmax + 2.0 ** 103             # FLT_MAX + 1/2 ulp: a tie, rounds to inf
    v = [1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24, -(1 + 2.0 ** -24), 2.0 ** 20 + 0.5 ** 4,
         np.nextafter(1 + 2.0 ** -24, 2), np.nextafter(1 + 2.0 ** -24, 0),
         fmax, np.nextafter(half_up, 0), half_up, np.nextafter(half_up, np.inf), -half_up,
         tiny, tiny / 2, np.nextafter(tiny / 2, 1), np.nextafter(tiny / 2, 0), 3 * tiny / 2,
         5 * tiny / 2, -tiny / 2, 2.0 ** -126, np.nextafter(2.0 ** -126, 0), 2.0 ** -140 / 3,
         1e-300, -1e-300, 0.0, -0.0, np.nan, np.inf, -np.inf, 1e300, -1e300]
    return np.array(v, dtype=np.float64)


def test_convert_rounding_and_subnormals(lib, sizes):
    """f64 -> f32 rounds to nearest-even exactly as numpy's astype: ties,
    the two sides of FLT_MAX + 1/2 ulp, the float32 subnormal range including
    the halfway case at the smallest subnormal, +-0.0, NaN; f32 -> f64 is exact
    on subnormals; complex on both parts; odd and grid-wrapping lengths."""
    rng = np.random.default_rng(91)
    edges = _narrowing_edges()
    sub32 = rng.integers(1, 2 ** 23, size=1001, dtype=np.int32).view(np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for n in [edges.size] + sizes:
            if n == edges.size:
                x = edges
            else:
                e = rng.integers(-160, 140, size=n)
                x = np.ldexp(rng.standard_normal(n), e)
                x[: min(n, edges.size)] = edges[: min(n, edges.size)]
            assert _same_or_both_nan(_convert(lib, x, "float32"), x.astype(np.float32)), n
            z = np.empty(x.size, dtype=np.complex128)
            z.real, z.imag = x, x[::-1]
            assert _same_or_both_nan(_convert(lib, z, "complex64"), z.astype(np.complex64)), n
        for y in (sub32, sub32[:257], edges.astype(np.float32)):
            assert _same_or_both_nan(_convert(lib, y, "float64"), y.astype(np.float64))
            zc = np.empty(y.size, dtype=np.complex64)
            zc.real, zc.imag = y, y[::-1]
            assert _same_or_both_nan(_convert(lib, zc, "complex128"), zc.astype(np.complex128))


# ---- Lanczos basis --------------------------------------------------------------------
@pytest.mark.parametrize("ncv", [8, 16, 17, 20, 33])
def test_lanczos_basis_is_orthonormal(ncv):
    """One full cycle of ``eigh_lanczos`` on a diagonal operator with distinct
    dyadic eigenvalues: the recorded basis is orthonormal to 10 m sqrt(n) eps
    and the returned Ritz value is the lowest eigenvalue of V^T A V to
    10 m eps |A|.  ncv = 17 and 33 cross the 16-row chunks of the fused
    Gram-Schmidt kernels."""
    n = 20000
    rng = np.random.default_rng(ncv)
    d = (rng.permutation(n) - n // 3) / 2.0 ** 14         # distinct, dyadic
    D = torch.from_numpy(d).cuda()
    basis = []

    def matvec(v):
        basis.append(v.t.clone())
        return Array(D * v.t)

    v0 = ops.asarray(rng.standard_normal(n))
    theta, _ = lanczos.eigh_lanczos(matvec, v0, ncv=ncv, tol=1e-15, min_steps=ncv, maxiter=1)
    V = torch.stack(basis).cpu().numpy()
    m = V.shape[0]
    assert m == ncv
    gram = V.astype(np.longdouble) @ V.T.astype(np.longdouble)
    assert np.max(np.abs(gram - np.eye(m))) <= 10 * m * np.sqrt(n) * EPS
    H = (V.astype(np.longdouble) * d) @ V.T.astype(np.longdouble)
    low = np.linalg.eigvalsh(np.asarray(H, dtype=np.float64))[0]
    assert abs(theta - low) <= 10 * m * EPS * np.max(np.abs(d)), (theta, low)
