"""GPU tier: every kernel route of the pairwise contraction against exact and
bounded oracles.

The library reports which route a contraction takes (``route_pair``: engine,
tile configuration, split-K, stream-K, cfg-0 shared-memory layout).  The route
search (``tests/route_oracle.py``) asks it, at this device's SM count, for the
cheapest shape of a fixed grid that reaches each route, and every route is run
through:

(a) an exact oracle: integer inputs |x| <= 8, so every partial sum is an
    integer below 2^24 and the float64 numpy result is exact in any order; the
    kernel must reproduce it exactly (with alpha / beta accumulation, either
    operand conjugated, and an output written through a permuted view);
(b) a bounded oracle: random-normal inputs, each element within the rigorous
    per-element bound of the engine, and a repeated call bit-identical;
(c) sentinel padding: operands are views into NaN-filled buffers (a stray read
    poisons the result), the output is a view into a buffer of a sentinel bit
    pattern that must survive outside the view, and beta = 0 into a NaN-filled
    output must not read it;
(d) stream-K routes three times in a row through the Python layer, which keeps
    the workspace flag words zero between launches;
(e) non-finite inputs: every output element in the IEEE class (NaN / +inf /
    -inf / finite) of the exact result.

A dependent chain of contractions over alternating routes without host
synchronisation checks the programmatic-dependent-launch ordering.
"""

import zlib

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from tests import route_oracle as ro

pytestmark = pytest.mark.gpu

_TORCH = {"float32": torch.float32, "float64": torch.float64,
          "complex64": torch.complex64, "complex128": torch.complex128}
_BITS = {"float32": (torch.int32, 0x7FC0BEEF), "complex64": (torch.int32, 0x7FC0BEEF),
         "float64": (torch.int64, 0x7FF8DEADBEEF0001),
         "complex128": (torch.int64, 0x7FF8DEADBEEF0001)}
KEYS = sorted(ro.required_keys(), key=str)


@pytest.fixture(scope="module")
def routes():
    return ro.search_routes()


def _id(key):
    return "-".join(str(k) for k in key)


def _chosen(routes, key):
    assert key in routes, f"no grid shape reaches route {key}"
    return routes[key]


def _bits(t):
    r = torch.view_as_real(t) if t.is_complex() else t
    return r.view(_BITS[_dtype_name(t)][0])


def _dtype_name(t):
    return {v: k for k, v in _TORCH.items()}[t.dtype]


def _padded(x, fill_bits=None, transpose=False):
    """Device view holding numpy `x` inside a larger buffer whose other
    elements are NaN (inputs) or the sentinel bit pattern (outputs).
    transpose: the buffer stores the last two axes swapped and the view
    permutes them back.  Returns (buffer, view, mask of the view's elements)."""
    dt = str(x.dtype)
    shape = list(x.shape)
    if transpose:
        shape[-2:] = shape[-2:][::-1]
    bshape, off = ro.pad_spec(shape)
    buf = torch.empty(bshape, dtype=_TORCH[dt], device="cuda")
    if fill_bits is None:
        buf.fill_(float("nan") if not buf.is_complex() else complex(float("nan"), float("nan")))
    else:
        _bits(buf).fill_(fill_bits)
    sl = tuple(slice(o, o + s) for o, s in zip(off, shape))
    view = buf[sl]
    if transpose:
        view = view.transpose(-1, -2)
    view.copy_(torch.from_numpy(np.ascontiguousarray(x)))
    mask = np.zeros(bshape, dtype=bool)
    mask[sl] = True
    return buf, view, mask


def _route_of_views(form, a, b, c, dtype, eng):
    _, la, _, lb, _, lc = ro.FORMS[form]
    return qb.route_pair(list(a.shape), list(a.stride()), la, list(b.shape), list(b.stride()),
                         lb, list(c.shape), list(c.stride()), lc, ro.QB_DTYPE[dtype], eng,
                         ptrs=(a.data_ptr(), b.data_ptr(), c.data_ptr()))


def _contract(form, A, B, out, eng, **kw):
    _, la, _, lb, _, lc = ro.FORMS[form]
    return qb.contract_pair(A, la, B, lb, lc, out=out, engine=eng, **kw)


def _canon_out(form, view):
    return ro.from_storage(form, view.cpu().numpy())


def _assert_sentinel_kept(buf, mask, dtype):
    bits = _bits(buf).cpu().numpy()
    if bits.ndim > mask.ndim:
        mask = np.broadcast_to(mask[..., None], bits.shape)
    outside = bits[~mask]
    assert np.all(outside == _BITS[dtype][1]), "a store landed outside the output view"


def _rng(key, salt):
    return np.random.default_rng(zlib.crc32(f"{key}{salt}".encode()))


def test_route_search_covers_every_route(routes):
    """Every route the library dispatches float64 / complex128 to (cfg 0-4 x
    plain / split-K, stream-K, the four cfg-0 real layouts in both launch
    modes) and the int8 engine for all four dtypes is reached by the grid."""
    lines = []
    for key in KEYS:
        if key in routes:
            form, M, K, N, eng, r = routes[key]
            lines.append(f"{_id(key):32s} {form:8s} M={M} K={K} N={N} engine={eng} "
                         f"splitk={r['splitk']} streamk={r['streamk']} sms={r['sms']}")
    print("\n" + "\n".join(lines))
    missing = [k for k in KEYS if k not in routes]
    assert not missing, f"routes no grid shape reaches: {missing}"
    assert {r["sms"] for *_, r in routes.values()} == {torch.cuda.get_device_properties(0)
                                                      .multi_processor_count}


@pytest.mark.parametrize("key", KEYS, ids=_id)
def test_route_exact_oracle(routes, key):
    dtype = key[0]
    form, M, K, N, eng, r = _chosen(routes, key)
    rng = _rng(key, "exact")
    sa, sb = ro.canonical_shapes(form, M, K, N)
    a, b = ro.int_operand(rng, sa, dtype), ro.int_operand(rng, sb, dtype)
    ref = (ro.wide(a) @ ro.wide(b)).astype(dtype)
    xa, xb = ro.to_storage(form, a, b)
    _, A, _ = _padded(xa)
    _, B, _ = _padded(xb)
    xc = ro.out_storage(form, ref)
    # beta = 0 into a NaN-pattern output: C is not read, nothing outside it written
    sent = _BITS[dtype][1]
    cbuf, C, cmask = _padded(np.zeros_like(xc), fill_bits=sent)
    _bits(cbuf).fill_(sent)
    got = _route_of_views(form, A, B, C, dtype, eng)
    assert ro.route_key(dtype, got) == key, (got, r)
    _contract(form, A, B, C, eng)
    np.testing.assert_array_equal(_canon_out(form, C), ref)
    _assert_sentinel_kept(cbuf, cmask, dtype)

    if form != "ab,b":   # output through a permuted (transposed) view
        tbuf, T, tmask = _padded(np.zeros_like(xc), fill_bits=sent, transpose=True)
        _bits(tbuf).fill_(sent)
        assert ro.route_key(dtype, _route_of_views(form, A, B, T, dtype, eng)) == key
        _contract(form, A, B, T, eng)
        np.testing.assert_array_equal(_canon_out(form, T), ref)
        _assert_sentinel_kept(tbuf, tmask, dtype)

    if not (key[1] == "int8" and dtype in ("float64", "complex128")):
        # alpha / beta accumulation (qb_contract_pair_ab has no engine argument:
        # float64 / complex128 accumulate on DMMA, so the int8 routes of those
        # dtypes are not reached this way)
        c0 = ro.int_operand(rng, xc.shape, dtype)
        _, C2, _ = _padded(c0)
        _contract(form, A, B, C2, eng, alpha=-2.0, beta=3.0)
        want = (-2.0 * ro.wide(ref) + 3.0 * ro.from_storage(form, ro.wide(c0))).astype(dtype)
        np.testing.assert_array_equal(_canon_out(form, C2), want)

    if dtype.startswith("complex"):
        for ca, cb in ((True, False), (False, True)):
            out = _contract(form, A, B, None, eng, conj_a=ca, conj_b=cb)
            want = ((ro.wide(a).conj() if ca else ro.wide(a))
                    @ (ro.wide(b).conj() if cb else ro.wide(b))).astype(dtype)
            np.testing.assert_array_equal(_canon_out(form, out), want)

    if key[1] == "streamk":
        # back-to-back launches through the Python layer, which keeps the
        # flag words zero between launches instead of clearing them: a flag
        # left set would hand the next launch's owner a stale partial tile
        for i in range(3):
            a_i = ro.int_operand(rng, sa, dtype)
            xa_i, _ = ro.to_storage(form, a_i, b)
            out = _contract(form, torch.from_numpy(xa_i).cuda(), B, None, eng)
            np.testing.assert_array_equal(_canon_out(form, out),
                                          (ro.wide(a_i) @ ro.wide(b)).astype(dtype))


@pytest.mark.parametrize("key", KEYS, ids=_id)
def test_route_bounded_and_deterministic(routes, key):
    dtype = key[0]
    form, M, K, N, eng, _ = _chosen(routes, key)
    rng = _rng(key, "normal")
    sa, sb = ro.canonical_shapes(form, M, K, N)
    a, b = ro.normal_operand(rng, sa, dtype), ro.normal_operand(rng, sb, dtype)
    xa, xb = ro.to_storage(form, a, b)
    A, B = torch.from_numpy(xa).cuda(), torch.from_numpy(xb).cuda()
    out1 = _contract(form, A, B, None, eng)
    out2 = _contract(form, A, B, None, eng)
    assert torch.equal(_bits(out1), _bits(out2)), "repeated call is not bit-identical"
    got = _canon_out(form, out1)
    ref = ro.wide(a) @ ro.wide(b)
    if key[1] == "int8":
        bound = ro.int8_bound(a, b, dtype in ("float32", "complex64"))
    else:
        bound = ro.dmma_bound(a, b)
    err = np.abs(ro.wide(got) - ref)
    assert np.all(err <= bound), f"max err / bound = {np.max(err / bound):.3g}"


@pytest.mark.parametrize("key", KEYS, ids=_id)
def test_route_nonfinite_inputs(routes, key):
    """NaN, +inf and -inf in A and B (including the last row / column and an
    inf meeting an exact zero): every output element in the class IEEE
    arithmetic gives the exact result, the finite ones within the bound."""
    dtype = key[0]
    form, M, K, N, eng, _ = _chosen(routes, key)
    rng = _rng(key, "nonfinite")
    sa, sb = ro.canonical_shapes(form, M, K, N)
    a, b = ro.normal_operand(rng, sa, dtype), ro.normal_operand(rng, sb, dtype)
    a[0], b[0] = ro.plant_nonfinite(a[0], b[0])
    xa, xb = ro.to_storage(form, a, b)
    out = _contract(form, torch.from_numpy(xa).cuda(), torch.from_numpy(xb).cuda(), None, eng)
    got = ro.wide(_canon_out(form, out))
    ro.check_classes(a, b, got, key[1] == "int8")


def _chain_steps():
    """Right multiplications X <- X @ W (X: M x C) whose routes alternate
    classic cfg 0 -> stream-K -> split-K -> int8 -> small tile, found by
    asking the planner over the size grid."""
    want = [lambda r: r["kind"] == "dmma" and r["cfg"] == 0 and r["splitk"] == 1,
            lambda r: r["kind"] == "dmma_streamk",
            lambda r: r["kind"] == "dmma" and r["splitk"] > 1,
            lambda r: r["kind"] == "int8",
            lambda r: r["kind"] == "dmma" and r["cfg"] == 4]
    engines = [0, 0, 0, ro.ENGINE_INT8, 0]

    def dfs(M, C, i, path):
        if i == len(want):
            return path
        for n in ro.SIZES:
            if ro.macs("ab,bc", M, C, n, "float64") > ro.MAX_MACS:
                continue
            r = ro.route_of("ab,bc", M, C, n, "float64", engines[i])
            if want[i](r):
                res = dfs(M, n, i + 1, path + [(C, n, engines[i])])
                if res:
                    return res
        return None

    for M in ro.SIZES:
        for C in ro.SIZES:
            res = dfs(M, C, 0, [])
            if res:
                return M, res
    return None, None


def test_dependent_chain_alternating_routes():
    """X_{i+1} = X_i @ W_i on one stream with no host synchronisation between
    the launches; every W column holds two entries +-1, so all values stay
    small integers and the float64 chain is exact."""
    M, steps = _chain_steps()
    assert steps, "no chain of shapes reaches the five routes"
    rng = np.random.default_rng(17)
    x0 = ro.int_operand(rng, (M, steps[0][0]), "float64")
    ws = []
    for c, n, _ in steps:
        w = np.zeros((c, n))
        for j in range(n):
            rows = rng.choice(c, size=2, replace=False)
            w[rows, j] = rng.choice([-1.0, 1.0], size=2)
        ws.append(w)
    X = torch.from_numpy(x0).cuda()
    W = [torch.from_numpy(w).cuda() for w in ws]
    torch.cuda.synchronize()
    outs = []
    for (c, n, eng), w in zip(steps, W):
        X = qb.contract_pair(X, [0, 1], w, [1, 2], [0, 2], engine=eng)
        outs.append(X)
    ref = x0
    for w, o in zip(ws, outs):
        ref = ref @ w
        np.testing.assert_array_equal(o.cpu().numpy(), ref)
