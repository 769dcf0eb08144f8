"""GPU tier: every kernel route of the pairwise contraction against exact and
bounded oracles.

The library reports which route a contraction takes (``route_pair``: engine,
tile configuration, split-K, stream-K, cfg-0 shared-memory layout, the
streaming engine's (KMAX, NMAX) variant, the zero fill and the widening path
of single precision).  The route
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

Streaming variants also run at a shape just past the previous variant's limit.
A dependent chain of contractions over alternating routes without host
synchronisation checks the programmatic-dependent-launch ordering.  Explicit
tests cover what a route key cannot: the zero fill's byte tail, 8-byte aligned
and strided outputs; the streaming engine past 65535 batch entries and past
its capped row grid; pointer-array batches on every tile configuration with a
misaligned item, and across the 65535-entry chunk boundary.
"""

import zlib

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from tests import route_oracle as ro

pytestmark = pytest.mark.gpu

KEYS = sorted(ro.required_keys(), key=str)


@pytest.fixture(scope="module")
def routes():
    return ro.search_routes()


def _id(key):
    return "-".join(str(k) for k in key)


def _chosen(routes, key):
    assert key in routes, f"no grid shape reaches route {key}"
    return routes[key]


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


def _rng(key, salt):
    return np.random.default_rng(zlib.crc32(f"{key}{salt}".encode()))


def test_route_search_covers_every_route(routes):
    """Every route the library dispatches float64 / complex128 to (cfg 0-4 x
    plain / split-K, stream-K, the four cfg-0 real layouts in both launch
    modes, the 9 streaming variants), the int8 engine for all four dtypes,
    the widening path of float32 / complex64 and the zero fill of all four
    dtypes is reached by the grid."""
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
    shapes = [_chosen(routes, key)]
    if key[1] == "stream":
        # the variant's largest operator, then a shape just past the previous
        # variant's limit (the first k / n of the register arrays used)
        shapes.append(ro.stream_lower_edges()[key])
    for form, M, K, N, eng, r in shapes:
        _exact_oracle(key, form, M, K, N, eng, r)


def _exact_oracle(key, form, M, K, N, eng, r):
    dtype = key[0]
    rng = _rng(key, f"exact{K}{N}")
    sa, sb = ro.canonical_shapes(form, M, K, N)
    a, b = ro.int_operand(rng, sa, dtype), ro.int_operand(rng, sb, dtype)
    ref = (ro.wide(a) @ ro.wide(b)).astype(dtype)
    xa, xb = ro.to_storage(form, a, b)
    _, A, _ = ro.padded(xa)
    _, B, _ = ro.padded(xb)
    xc = ro.out_storage(form, ref)
    # beta = 0 into a NaN-pattern output: C is not read, nothing outside it written
    sent = ro.BITS[dtype][1]
    cbuf, C, cmask = ro.padded(np.zeros_like(xc), fill_bits=sent)
    ro.bits(cbuf).fill_(sent)
    got = _route_of_views(form, A, B, C, dtype, eng)
    assert ro.route_key(dtype, got) == key, (got, r)
    _contract(form, A, B, C, eng)
    np.testing.assert_array_equal(_canon_out(form, C), ref)
    ro.assert_sentinel_kept(cbuf, cmask, dtype)

    if form != "ab,b":   # output through a permuted (transposed) view
        tbuf, T, tmask = ro.padded(np.zeros_like(xc), fill_bits=sent, transpose=True)
        ro.bits(tbuf).fill_(sent)
        assert ro.route_key(dtype, _route_of_views(form, A, B, T, dtype, eng)) == key
        _contract(form, A, B, T, eng)
        np.testing.assert_array_equal(_canon_out(form, T), ref)
        ro.assert_sentinel_kept(tbuf, tmask, dtype)

    c0 = ro.int_operand(rng, xc.shape, dtype)
    if key[1] == "zero_fill":
        # an empty sum: beta = 1 leaves C as it is, any other beta but 0 is refused
        _, C2, _ = ro.padded(c0)
        _contract(form, A, B, C2, eng, alpha=-2.0, beta=1.0)
        np.testing.assert_array_equal(C2.cpu().numpy(), c0)
        with pytest.raises(ValueError, match=r"code -10"):
            _contract(form, A, B, C2, eng, alpha=1.0, beta=0.5)
    elif key[1] not in ("int8", "stream") or dtype in ("float32", "complex64"):
        # alpha / beta accumulation (qb_contract_pair_ab has no engine argument:
        # float64 / complex128 accumulate on DMMA, so the int8 and streaming
        # routes of those dtypes are not reached this way)
        _, C2, _ = ro.padded(c0)
        _contract(form, A, B, C2, eng, alpha=-2.0, beta=3.0)
        want = (-2.0 * ro.wide(ref) + 3.0 * ro.from_storage(form, ro.wide(c0))).astype(dtype)
        np.testing.assert_array_equal(_canon_out(form, C2), want)

    if dtype.startswith("complex"):
        for ca, cb in ((True, False), (False, True), (True, True)):
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
    assert torch.equal(ro.bits(out1), ro.bits(out2)), "repeated call is not bit-identical"
    got = _canon_out(form, out1)
    ref = ro.wide(a) @ ro.wide(b)
    bound = ro.route_bound(key[1], a, b)
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
    if key[1] == "zero_fill":
        # no input element exists to hold a special value: the empty sum is
        # +0 everywhere, whatever NaN the output held before
        xa, xb = ro.to_storage(form, a, b)
        xc = ro.out_storage(form, np.zeros((a.shape[0], M, N)))
        out = ro.nan_fill(torch.empty(xc.shape, dtype=ro.TORCH[dtype], device="cuda"))
        _contract(form, torch.from_numpy(xa).cuda(), torch.from_numpy(xb).cuda(), out, eng)
        assert not ro.bits(out).any(), "zero fill left a nonzero bit"
        return
    a[0], b[0] = ro.plant_nonfinite(a[0], b[0])
    xa, xb = ro.to_storage(form, a, b)
    out = _contract(form, torch.from_numpy(xa).cuda(), torch.from_numpy(xb).cuda(), None, eng)
    got = ro.wide(_canon_out(form, out))
    ro.check_classes(a, b, got, kind=key[1])


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


# ---- what a route key cannot express --------------------------------------
@pytest.mark.parametrize("dtype", list(ro.TORCH))
def test_zero_fill_tail_alignment_and_strides(dtype):
    """A contracted extent of 0 zeroes the output: the 16-byte vector fill
    with a byte tail (3 float32 = 12 bytes), an output whose base is only
    8-byte aligned and a strided view take the element-wise fill.  Every
    other element of the buffer keeps its sentinel bits."""
    tdt, sent = ro.TORCH[dtype], ro.BITS[dtype][1]
    a = torch.ones((3, 0), dtype=tdt, device="cuda")
    b = torch.ones((0, 5), dtype=tdt, device="cuda")
    b1 = torch.ones((0,), dtype=tdt, device="cuda")
    cases = [("contiguous, 16-byte aligned", lambda buf: buf[:3], b1)]
    if dtype != "complex128":           # complex128 elements are 16 bytes
        off = 8 // ro.TORCH[dtype].itemsize
        cases.append(("8-byte aligned base", lambda buf: buf[off:off + 3], b1))
    cases.append(("strided", lambda buf: buf.view(8, 8)[1:4, 2:7], b))
    for what, view_of, bop in cases:
        buf = torch.empty(64, dtype=tdt, device="cuda")
        ro.bits(buf).fill_(sent)
        out = view_of(buf)
        probe = torch.zeros(64, dtype=torch.int64)
        view_of(probe).fill_(1)
        mask = probe.numpy() == 1
        lb, lc = ([1], [0]) if bop.dim() == 1 else ([1, 2], [0, 2])
        r = qb.route_pair([3, 0], [0, 1], [0, 1], list(bop.shape), list(bop.stride()), lb,
                          list(out.shape), list(out.stride()), lc, ro.QB_DTYPE[dtype],
                          ptrs=(a.data_ptr(), bop.data_ptr(), out.data_ptr()))
        assert r["kind"] == "zero_fill" and r["launches"] == 1, (what, r)
        qb.contract_pair(a, [0, 1], bop, lb, lc, out=out)
        assert not ro.bits(out).any(), f"{what}: output not zeroed"
        ro.assert_sentinel_kept(buf, mask, dtype)


def _stream_case(dtype, shape_a, la, shape_b, lb, lc, out_shape):
    """Integer operands, a sentinel-filled output, the streaming engine; the
    output must equal the exact product everywhere."""
    rng = np.random.default_rng(len(shape_a) * 1000 + shape_a[0])
    a, b = ro.int_operand(rng, shape_a, dtype), ro.int_operand(rng, shape_b, dtype)
    A, B = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    out = torch.empty(out_shape, dtype=ro.TORCH[dtype], device="cuda")
    ro.bits(out).fill_(ro.BITS[dtype][1])
    r = qb.route_pair(list(A.shape), list(A.stride()), la, list(B.shape), list(B.stride()), lb,
                      list(out.shape), list(out.stride()), lc, ro.QB_DTYPE[dtype],
                      ro.ENGINE_STREAM)
    assert r["kind"] == "stream", r
    qb.contract_pair(A, la, B, lb, lc, out=out, engine=ro.ENGINE_STREAM)
    want = np.einsum(ro.einsum_spec(la, lb, lc), ro.wide(a), ro.wide(b)).astype(dtype)
    np.testing.assert_array_equal(out.cpu().numpy(), want)


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_stream_engine_batch_past_grid_y_limit(dtype):
    """More than 65535 batch entries: the kernel's grid-y loop wraps."""
    G = 65535 + 77
    _stream_case(dtype, (G, 3, 2), [3, 0, 1], (G, 2, 2), [3, 1, 2], [3, 0, 2], (G, 3, 2))


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_stream_engine_rows_past_grid_x_cap(dtype):
    """More than 8 * SMs * 256 rows: the grid-x loop of the capped grid wraps."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = 8 * sms * 256 + 300
    _stream_case(dtype, (M, 2), [0, 1], (2, 3), [1, 2], [0, 2], (M, 3))


def _batched_items(routes):
    """(dtype, cfg) -> (form, M, K, N) for every DMMA tile configuration the
    plain route keys reach: the key's own shape when its per-item signature
    (no batch label) plans the same configuration, else the cheapest
    non-batched grid shape that does."""
    items = {}
    for key in sorted(routes, key=str):
        if key[1] != "plain":
            continue
        dtype, cfg = key[0], key[2]
        form, M, K, N, _, _ = routes[key]
        if (dtype, cfg) in items:
            continue
        if not form.startswith("g") and ro.route_of(form, M, K, N, dtype)["cfg"] == cfg:
            items[(dtype, cfg)] = (form, M, K, N)
            continue
        best = None
        for f in (f for f in ro.FORMS if not f.startswith("g")):
            for M2 in ro.SIZES:
                for K2 in ro.SIZES:
                    for N2 in ((1,) if f == "ab,b" else ro.SIZES):
                        c = ro.macs(f, M2, K2, N2, dtype)
                        if c <= ro.MAX_MACS and (best is None or c < best[0]) and \
                                ro.route_of(f, M2, K2, N2, dtype)["cfg"] == cfg:
                            best = (c, (f, M2, K2, N2))
        assert best, f"no item shape plans tile configuration {cfg} for {dtype}"
        items[(dtype, cfg)] = best[1]
    return items


def test_contract_batched_every_tile_config(routes):
    """Pointer-array batches of 3 items on every tile configuration the plain
    routes reach; item 1's operands sit one element past an aligned address,
    so the descriptor carries the weakest alignment and the vector loads are
    dropped for all items.  Complex operands are both conjugated."""
    items = _batched_items(routes)
    assert {c for (dt, c) in items if dt == "float64"} == set(range(5))
    assert {c for (dt, c) in items if dt == "complex128"} == set(range(5))
    for (dtype, cfg), (form, M, K, N) in sorted(items.items()):
        rng = np.random.default_rng(cfg * 7 + len(dtype))
        sa, sb = ro.canonical_shapes(form, M, K, N)
        _, la, _, lb, _, lc = ro.FORMS[form]
        conj = dtype.startswith("complex")
        A, B, want = [], [], []
        for i in range(3):
            a, b = ro.int_operand(rng, sa, dtype), ro.int_operand(rng, sb, dtype)
            xa, xb = ro.to_storage(form, a, b)
            if i == 1:
                ta, tb = (torch.empty(x.size + 1, dtype=ro.TORCH[dtype], device="cuda")
                          for x in (xa, xb))
                ta, tb = ta[1:].view(xa.shape), tb[1:].view(xb.shape)
                ta.copy_(torch.from_numpy(xa))
                tb.copy_(torch.from_numpy(xb))
            else:
                ta, tb = torch.from_numpy(xa).cuda(), torch.from_numpy(xb).cuda()
            A.append(ta)
            B.append(tb)
            aw, bw = ro.wide(a), ro.wide(b)
            want.append(((aw.conj() if conj else aw) @ (bw.conj() if conj else bw)).astype(dtype))
        outs = qb.contract_batched(A, la, B, lb, lc, conj_a=conj, conj_b=conj)
        for i, (o, w) in enumerate(zip(outs, want)):
            np.testing.assert_array_equal(_canon_out(form, o), w,
                                          err_msg=f"{dtype} cfg {cfg} item {i}")


def test_contract_batched_two_chunks():
    """65536 items: two launches of at most 65535 entries; every output exact."""
    n = 65536
    rng = np.random.default_rng(5)
    a = ro.int_operand(rng, (n, 2, 3), "float64")
    b = ro.int_operand(rng, (n, 3, 2), "float64")
    A, B = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    outs = qb.contract_batched(list(A.unbind(0)), [0, 1], list(B.unbind(0)), [1, 2], [0, 2])
    np.testing.assert_array_equal(torch.stack(outs).cpu().numpy(), a @ b)
