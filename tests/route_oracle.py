"""Helpers of the contraction route tests: the route search over a fixed
shape grid (host-only: it asks the library's planner), padded operand views,
and the reference results the kernels are held to.

Reference arithmetic is plain numpy in float64.  ``nonfinite_class`` gives the
IEEE class (NaN / +inf / -inf / finite) of every element of A @ B from the
positions of the special values alone, so it does not depend on how a BLAS
treats them.  ``exact_dot`` is the correctly rounded inner product (products
split exactly, summed by ``math.fsum``) the vector-kernel tests compare with."""

import math

import numpy as np
import torch

from quimb_b200 import _lib
from quimb_b200.contract import route_pair

# 16384: a complex matrix-vector product takes the tall tile without split-K
# only from about 16k rows
SIZES = (64, 130, 256, 384, 512, 768, 1024, 1536, 2048, 4096, 16384)
MAX_MACS = 3e9      # host reference work per chosen shape (complex: 4 real MACs)
GROUPS = 2          # batch extent of the batched form

# form -> (A storage axes, A labels, B storage axes, B labels, C axes, C labels)
FORMS = {
    "ab,bc": ("MK", (0, 1), "KN", (1, 2), "MN", (0, 2)),
    "ba,bc": ("KM", (1, 0), "KN", (1, 2), "MN", (0, 2)),
    "ab,cb": ("MK", (0, 1), "NK", (2, 1), "MN", (0, 2)),
    "ba,cb": ("KM", (1, 0), "NK", (2, 1), "MN", (0, 2)),
    "gab,gbc": ("GMK", (3, 0, 1), "GKN", (3, 1, 2), "GMN", (3, 0, 2)),
    # matrix-vector (N = 1): the only way complex operands reach the tall tile
    "ab,b": ("MK", (0, 1), "K", (1,), "M", (0,)),
}
QB_DTYPE = {"float32": _lib.QB_F32, "float64": _lib.QB_F64,
            "complex64": _lib.QB_C64, "complex128": _lib.QB_C128}
ENGINE_INT8 = 2
ENGINE_STREAM = 3

# the streaming engine's compiled (KMAX, NMAX) variants (contract_stream.cu):
# real operators up to 32 x 32, complex ones up to 16 x 16
STREAM_VARIANTS = {"float64": ((4, 4), (16, 4), (4, 16), (16, 16), (32, 32)),
                   "complex128": ((4, 4), (16, 4), (4, 16), (16, 16))}
# its search grid: every variant at its largest (K, N) and just past the
# previous variant's limit; M = 3 full 256-row blocks and a ragged one
STREAM_KN = (1, 4, 5, 16, 17, 32)
STREAM_M = 3 * 256 + 7
# zero-fill shapes: contracted extent 0, a 3-element output is the cheapest
ZERO_FILL_M, ZERO_FILL_N = 3, 5


def strides(shape):
    st, acc = [], 1
    for e in reversed(shape):
        st.append(acc)
        acc *= e
    return list(reversed(st))


def shapes(form, M, K, N):
    ext = dict(M=M, K=K, N=N, G=GROUPS)
    fa, la, fb, lb, fc, lc = FORMS[form]
    return [ext[c] for c in fa], la, [ext[c] for c in fb], lb, [ext[c] for c in fc], lc


def route_of(form, M, K, N, dtype, engine=0):
    sa, la, sb, lb, sc, lc = shapes(form, M, K, N)
    return route_pair(sa, strides(sa), la, sb, strides(sb), lb, sc, strides(sc), lc,
                      QB_DTYPE[dtype], engine)


def route_key(dtype, r):
    """Identity of a compiled kernel variant: dtype x engine x tile config x
    {plain, split-K, stream-K} x cfg-0 layout of real operands; the streaming
    engine's (KMAX, NMAX) variant; the zero fill and the widening path."""
    if r["kind"] == "int8":
        return (dtype, "int8")
    if r["kind"] == "stream":
        return (dtype, "stream", r["stream_k"], r["stream_n"])
    if r["kind"] in ("zero_fill", "widen"):
        return (dtype, r["kind"])
    if r["kind"] == "dmma_streamk":
        return (dtype, "streamk", 0, r["layout"])
    if r["kind"] == "dmma":
        if r["splitk"] > 1:
            return (dtype, "splitk", r["cfg"], -1)
        return (dtype, "plain", r["cfg"], r["layout"])
    return None


def required_keys():
    """Every route qb_contract_pair can dispatch a float64 / complex128
    contraction to (DMMA, int8 on request, every streaming variant on
    request), the int8 engine and the widening path of float32 / complex64,
    and the zero fill of all four dtypes."""
    keys = set()
    for dt, variants in STREAM_VARIANTS.items():
        for k, n in variants:
            keys.add((dt, "stream", k, n))
    for dt in QB_DTYPE:
        keys.add((dt, "zero_fill"))
    keys.add(("float32", "widen"))
    keys.add(("complex64", "widen"))
    for dt in ("float64", "complex128"):
        for c in range(1, 5):
            keys.add((dt, "plain", c, -1))
        for c in range(5):
            keys.add((dt, "splitk", c, -1))
        keys.add((dt, "int8"))
    for lay in range(4):
        keys.add(("float64", "plain", 0, lay))
        keys.add(("float64", "streamk", 0, lay))
    keys.add(("complex128", "plain", 0, -1))
    keys.add(("complex128", "streamk", 0, -1))
    keys.add(("float32", "int8"))
    keys.add(("complex64", "int8"))
    return keys


def einsum_spec(la, lb, lc):
    """numpy einsum subscripts of integer mode labels."""
    sym = {}
    for l in list(la) + list(lb) + list(lc):
        sym.setdefault(l, chr(ord("a") + len(sym)))
    word = lambda ls: "".join(sym[l] for l in ls)  # noqa: E731
    return f"{word(la)},{word(lb)}->{word(lc)}"


def macs(form, M, K, N, dtype):
    g = GROUPS if form.startswith("g") else 1
    return g * M * K * N * (4 if dtype.startswith("complex") else 1)


def search_routes():
    """Cheapest grid shape for every route key: {key: (form, M, K, N, engine, route)}."""
    best = {}
    for dtype in QB_DTYPE:
        # float64 / complex128 take the int8 engine only on request
        engines = (0, ENGINE_INT8) if dtype in ("float64", "complex128") else (0,)
        for form, M, K, N in ((f, M, K, N) for f in FORMS for M in SIZES
                              for K in SIZES for N in ((1,) if f == "ab,b" else SIZES)):
            cost = macs(form, M, K, N, dtype)
            if cost > MAX_MACS:
                continue
            for eng in engines:
                r = route_of(form, M, K, N, dtype, eng)
                key = route_key(dtype, r)
                if key is None or (eng == ENGINE_INT8 and key[1] != "int8"):
                    continue
                if key not in best or cost < best[key][0]:
                    best[key] = (cost, (form, M, K, N, eng, r))
        for form in FORMS:
            # contracted extent 0: the cheapest shape has the fewest outputs
            M, N = ZERO_FILL_M, 1 if form == "ab,b" else ZERO_FILL_N
            r = route_of(form, M, 0, N, dtype)
            key = route_key(dtype, r)
            cost = (GROUPS if form.startswith("g") else 1) * M * N
            if key is not None and (key not in best or cost < best[key][0]):
                best[key] = (cost, (form, M, 0, N, 0, r))
    # streaming variants at their largest operator (then the cheapest form)
    for key, shapes in stream_shapes().items():
        best[key] = (None, max(shapes, key=lambda s: (s[2] * s[3], -macs(*s[:4], key[0]))))
    return {k: v[1] for k, v in best.items()}


def stream_shapes():
    """{streaming route key: [(form, M, K, N, engine, route), ...]} over the
    streaming grid (K, N in STREAM_KN, M = STREAM_M) with the engine
    requested."""
    out = {}
    for dtype in STREAM_VARIANTS:
        for form in FORMS:
            for K in STREAM_KN:
                for N in ((1,) if form == "ab,b" else STREAM_KN):
                    r = route_of(form, STREAM_M, K, N, dtype, ENGINE_STREAM)
                    key = route_key(dtype, r)
                    if key is not None and key[1] == "stream":
                        out.setdefault(key, []).append((form, STREAM_M, K, N, ENGINE_STREAM, r))
    return out


def stream_lower_edges():
    """Cheapest shape of every streaming variant: for each variant past the
    first one, a shape just past the previous variant's limit."""
    return {key: min(shapes, key=lambda s: macs(*s[:4], key[0]))
            for key, shapes in stream_shapes().items()}


# ---- operand layouts ---------------------------------------------------------
def to_storage(form, a, b):
    """Canonical a [G, M, K], b [G, K, N] -> the operands as the form stores them."""
    if form == "gab,gbc":
        return a, b
    a2, b2 = a[0], b[0]
    if form.startswith("ba"):
        a2 = a2.T
    if form == "ab,b":
        b2 = b2[:, 0]
    elif form.endswith("cb"):
        b2 = b2.T
    return np.ascontiguousarray(a2), np.ascontiguousarray(b2)


def from_storage(form, c):
    """The output as the form stores it -> canonical [G, M, N]."""
    if form == "gab,gbc":
        return c
    if form == "ab,b":
        return c[None, :, None]
    return c[None]


def out_storage(form, c):
    """Canonical [G, M, N] -> the output as the form stores it."""
    if form == "gab,gbc":
        return c
    if form == "ab,b":
        return c[0, :, 0]
    return c[0]


def canonical_shapes(form, M, K, N):
    g = GROUPS if form == "gab,gbc" else 1
    return (g, M, K), (g, K, N)


def pad_spec(shape):
    """Buffer shape and view offset of a padded view of `shape`: every axis
    padded, the innermost pitch and offset even so that 16-byte alignment
    (and with it the planner's vector loads) is the same as for a
    contiguous tensor."""
    pad = [3] * (len(shape) - 1) + [4 + shape[-1] % 2]
    off = [1] * (len(shape) - 1) + [2]
    return [s + p for s, p in zip(shape, pad)], off


# ---- device buffers with NaN padding / sentinel bits -----------------------
TORCH = {"float32": torch.float32, "float64": torch.float64,
         "complex64": torch.complex64, "complex128": torch.complex128}
# integer view and sentinel bit pattern (a quiet NaN with a payload) per dtype
BITS = {"float32": (torch.int32, 0x7FC0BEEF), "complex64": (torch.int32, 0x7FC0BEEF),
        "float64": (torch.int64, 0x7FF8DEADBEEF0001),
        "complex128": (torch.int64, 0x7FF8DEADBEEF0001)}


def dtype_name(t):
    return {v: k for k, v in TORCH.items()}[t.dtype]


def bits(t):
    """Integer view of the real parts of `t` (bitwise comparisons)."""
    r = torch.view_as_real(t) if t.is_complex() else t
    return r.view(BITS[dtype_name(t)][0])


def nan_fill(buf):
    buf.fill_(float("nan") if not buf.is_complex() else complex(float("nan"), float("nan")))
    return buf


def padded(x, fill_bits=None, transpose=False):
    """Device view holding numpy `x` inside a larger buffer whose other
    elements are NaN (inputs) or the sentinel bit pattern (outputs).
    transpose: the buffer stores the last two axes swapped and the view
    permutes them back.  Returns (buffer, view, mask of the view's elements)."""
    dt = str(x.dtype)
    shape = list(x.shape)
    if transpose:
        shape[-2:] = shape[-2:][::-1]
    bshape, off = pad_spec(shape)
    buf = torch.empty(bshape, dtype=TORCH[dt], device="cuda")
    if fill_bits is None:
        nan_fill(buf)
    else:
        bits(buf).fill_(fill_bits)
    sl = tuple(slice(o, o + s) for o, s in zip(off, shape))
    view = buf[sl]
    if transpose:
        view = view.transpose(-1, -2)
    view.copy_(torch.from_numpy(np.ascontiguousarray(x)))
    mask = np.zeros(bshape, dtype=bool)
    mask[sl] = True
    return buf, view, mask


def assert_sentinel_kept(buf, mask, dtype):
    """Every element of `buf` outside `mask` still holds the sentinel bits."""
    b = bits(buf).cpu().numpy()
    if b.ndim > mask.ndim:
        mask = np.broadcast_to(mask[..., None], b.shape)
    outside = b[~mask]
    assert np.all(outside == BITS[dtype][1]), "a store landed outside the output view"


# ---- numbers ---------------------------------------------------------------
def int_operand(rng, shape, dtype, lim=8):
    """Integer-valued entries in [-lim, lim] (complex: both parts)."""
    x = rng.integers(-lim, lim + 1, size=shape).astype(np.float64)
    if dtype.startswith("complex"):
        x = x + 1j * rng.integers(-lim, lim + 1, size=shape)
    return x.astype(dtype)


def normal_operand(rng, shape, dtype):
    x = rng.standard_normal(shape)
    if dtype.startswith("complex"):
        x = x + 1j * rng.standard_normal(shape)
    return x.astype(dtype)


def wide(x):
    return x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)


def gamma(n, u=2.0 ** -53):
    return n * u / (1 - n * u)


def _veltkamp(x):
    """x = hi + lo exactly, each part with at most 26 significant bits, so
    every product of two parts is exact in float64 (x finite, |x| < 2^995)."""
    c = x * 134217729.0                     # 2^27 + 1
    hi = c - (c - x)
    return hi, x - hi


def exact_dot(x, y):
    """sum_i x_i y_i correctly rounded to float64 (real float64 arrays): the
    products are split into exact sums of two-part products, which
    ``math.fsum`` adds without intermediate rounding."""
    x = np.asarray(x, dtype=np.float64).ravel()
    y = np.asarray(y, dtype=np.float64).ravel()
    xh, xl = _veltkamp(x)
    yh, yl = _veltkamp(y)
    terms = np.concatenate([xh * yh, xh * yl, xl * yh, xl * yl])
    return math.fsum(terms[terms != 0])


def exact_vdot(x, y):
    """conj(x) . y correctly rounded (per part for complex) and the bound
    scale sum |terms| of its real products; x, y of any dtype."""
    x, y = wide(np.asarray(x)).ravel(), wide(np.asarray(y)).ravel()
    if not np.iscomplexobj(x):
        return exact_dot(x, y), float(np.sum(np.abs(x * y)))
    xs, ys = np.concatenate([x.real, x.imag]), np.concatenate([y.real, y.imag])
    xt, yt = np.concatenate([x.real, -x.imag]), np.concatenate([y.imag, y.real])
    re, im = exact_dot(xs, ys), exact_dot(xt, yt)
    return complex(re, im), float(max(np.sum(np.abs(xs * ys)), np.sum(np.abs(xt * yt))))


def widen_bound(a, b):
    """The widening path: the float64 product within ``dmma_bound``, then
    rounded once to float32 (complex: each part, sqrt(2) u32 |C| in all)."""
    ref = np.abs(wide(a) @ wide(b))
    dm = dmma_bound(a, b)
    u32 = 2.0 ** -24 * (np.sqrt(2) if np.iscomplexobj(a) else 1.0)
    return dm + u32 * (ref + dm) * 1.001


def route_bound(kind, a, b):
    """Per-element bound of route kind `kind` ("int8", "widen", DMMA and
    streaming kinds) on C = a @ b against numpy's float64 product."""
    if kind == "int8":
        return int8_bound(a, b, a.dtype in (np.float32, np.complex64))
    if kind == "widen":
        return widen_bound(a, b)
    return dmma_bound(a, b)


def dmma_bound(a, b):
    """Per-element bound on |C_kernel - C_numpy| for C = a @ b computed in
    fp64 (a: [..., M, K], b: [..., K, N]).  Kernel and numpy both form inner
    products of K terms in some order, each within gamma_K |A|.|B| of the
    exact value (complex: the kernel sums 2K real products, within
    sqrt(2) gamma_2K |A|.|B|; numpy within sqrt(2) gamma_{K+2}), so their
    difference is within twice the larger bound."""
    K = a.shape[-1]
    absref = np.abs(wide(a)) @ np.abs(wide(b))
    if np.iscomplexobj(a):
        return 2 * np.sqrt(2) * gamma(2 * K + 2) * absref * 1.001
    return 2 * gamma(K) * absref * 1.001


def int8_bound(a, b, single):
    """Per-element bound for the int8 engine (csrc/ozaki_tc.cu) on C = a @ b,
    in its real-GEMM view: Ke contracted real units (complex: 2K), row maxima
    ra of A_e and column maxima cb of B_e (max of |re|, |im|).

    The split of a row with maximum mx < 2^e keeps x 2^(6-e) in (-64, 64) as S
    int8 digits of weight 128^-p, each rounded to nearest; the remainder after
    S digits is at most 0.5 * 128^-(S-1) in those units, i.e.
        |x - x~| <= 2^(e-7) 2^(-7(S-1)) <= mx 2^-(7S-1)       (2^e <= 2 mx).
    So |A_e B_e - A~ B~| <= Ke ra cb (2 * 2^-(7S-1) + 2^-(14S-2)).  The GEMM
    keeps the digit products with p + q < S; the dropped ones (p, q < S,
    p + q = d >= S, 2S-1-d pairs each, |digits| <= 64) add at most
        Ke 2^(eA+eB) sum_{d=S}^{2S-2} (2S-1-d) 2^-7d <= 4 Ke ra cb (S-1) 2^-7S 1.01.
    The int32 sums are exact; combining the S accumulators in fp64 rounds at
    most S times relative to sum_d |w_d acc_d| <= 4.07 Ke ra cb, adding
    S u 4.07 Ke ra cb (u = 2^-53); the final scaling is exact and the result
    is rounded once to the output type (u_out |C|).  numpy's own fp64 error is
    added as in ``dmma_bound``."""
    S = 4 if single else 8
    u = 2.0 ** -53
    u_out = 2.0 ** -24 if single else u
    aw, bw = wide(a), wide(b)
    K = a.shape[-1]
    Ke = 2 * K if np.iscomplexobj(a) else K
    mag = lambda x: np.maximum(np.abs(x.real), np.abs(x.imag))  # noqa: E731
    ra = mag(aw).max(axis=-1)
    cb = mag(bw).max(axis=-2)
    scale = ra[..., :, None] * cb[..., None, :]
    c_s = (2 * 2.0 ** -(7 * S - 1) + 2.0 ** -(14 * S - 2)
           + 4 * (S - 1) * 2.0 ** (-7 * S) * 1.01 + S * u * 4.07)
    ref = aw @ bw
    return (Ke * scale * c_s + 2 * u_out * np.abs(ref)) * 1.01 + dmma_bound(aw, bw)


def nonfinite_class(a, b):
    """IEEE class of every element of a @ b (2-d): 0 finite, 1 NaN, 2 +inf,
    3 -inf (finite sums assumed not to overflow).  Complex operands go
    through the real embedding A_e[m, 2k+c], B_e[2k+c, 2n+d] the kernels
    compute; the result has the classes of the real and imaginary parts."""
    if np.iscomplexobj(a):
        M, K = a.shape
        N = b.shape[1]
        ae = np.empty((M, 2 * K))
        ae[:, 0::2], ae[:, 1::2] = a.real, a.imag
        be = np.empty((2 * K, 2 * N))
        be[0::2, 0::2], be[0::2, 1::2] = b.real, b.imag
        be[1::2, 0::2], be[1::2, 1::2] = -b.imag, b.real
        ce = nonfinite_class(ae, be)
        return ce[:, 0::2], ce[:, 1::2]
    f = lambda m: m.astype(np.float64)  # noqa: E731
    fin_a, fin_b = np.isfinite(a), np.isfinite(b)
    pa, na = f(fin_a & (a > 0)), f(fin_a & (a < 0))
    pb, nb = f(fin_b & (b > 0)), f(fin_b & (b < 0))
    ia_p, ia_n = f(a == np.inf), f(a == -np.inf)
    ib_p, ib_n = f(b == np.inf), f(b == -np.inf)
    nan = (f(np.isnan(a)) @ np.ones(b.shape) + np.ones(a.shape) @ f(np.isnan(b))
           + (ia_p + ia_n) @ f(b == 0) + f(a == 0) @ (ib_p + ib_n))
    pinf = ia_p @ (pb + ib_p) + ia_n @ (nb + ib_n) + pa @ ib_p + na @ ib_n
    ninf = ia_p @ (nb + ib_n) + ia_n @ (pb + ib_p) + pa @ ib_n + na @ ib_p
    cls = np.zeros(nan.shape, dtype=np.int8)
    cls[ninf > 0] = 3
    cls[pinf > 0] = 2
    cls[(nan > 0) | ((pinf > 0) & (ninf > 0))] = 1
    return cls


def classify(x):
    x = np.asarray(x)
    cls = np.zeros(x.shape, dtype=np.int8)
    cls[x == np.inf] = 2
    cls[x == -np.inf] = 3
    cls[np.isnan(x)] = 1
    return cls


def check_classes(a, b, got, int8=False, kind=None):
    """got (float64 / complex128, [G, M, N]) against a @ b with special values
    in a, b ([G, M, K], [G, K, N]): the IEEE class of every element, and the
    finite elements -- outputs of rows and columns without special values --
    within the bound of route kind `kind` (see ``route_bound``; without it,
    the int8 engine's bound when `int8`, else the DMMA bound)."""
    if kind is None:
        kind = "int8" if int8 else "dmma"
    for g in range(a.shape[0]):
        want = nonfinite_class(wide(a[g]), wide(b[g]))
        if np.iscomplexobj(got):
            for part, w in zip((got[g].real, got[g].imag), want):
                np.testing.assert_array_equal(classify(part), w)
        else:
            np.testing.assert_array_equal(classify(got[g]), want)
    a0 = np.where(np.isfinite(a), a, 0)
    b0 = np.where(np.isfinite(b), b, 0)
    fin = np.isfinite(got)
    ref = wide(a0) @ wide(b0)
    bound = route_bound(kind, a0, b0)
    assert np.all(np.abs(got[fin] - ref[fin]) <= bound[fin])


def plant_nonfinite(a, b):
    """NaN, +inf and -inf at fixed positions of 2-d a (M x K) and b (K x N),
    including the last row / column (ragged tile edges), plus an exact zero
    in b that meets a's +inf (inf * 0 = NaN)."""
    a, b = a.copy(), b.copy()
    M, K = a.shape
    N = b.shape[1]
    a[0, 1] = np.nan
    a[3, 2] = np.inf
    a[M - 1, K - 1] = -np.inf
    b[2, 3 % N] = 0.0
    b[K // 2, N // 2] = np.nan
    b[5 % K, 7 % N] = np.inf
    b[K - 1, N - 1] = -np.inf
    return a, b
