"""GPU tier: every contraction route on non-canonical label structures.

The structures of ``tests/label_oracle.py`` -- repeated (diagonal) labels,
labels summed out of one operand only, broadcast (stride-0) operands,
overlapping input views, batch modes interleaved with free modes, groups of
several non-mergeable modes, size-1 modes -- each run on every route key the
host route search finds for them, at the cheapest grid shape that reaches it
(pinned in ``tests/golden/label_routes.json`` for the H100 SXM's 132 SMs,
searched at this device's SM count otherwise):

(a) exact oracle: integer operands |x| <= 8 and K (every summed term) small
    enough that every sum is an exact integer, also in float32; the output
    must equal the reference exactly, also through a transposed output,
    with alpha = -2, beta = 3 where ``qb_contract_pair_ab`` reaches the
    route, and with either operand conjugated (complex);
(b) sentinels: operands are views into NaN-filled buffers, the output a view
    into a buffer of a NaN sentinel pattern that must survive outside the
    view, and beta = 0 must not read the output;
(c) bounded oracle: random-normal operands within the route's per-element
    bound (K over every summed term), a repeated call bit-identical;
(d) the route ``route_pair`` reports for the device views (real pointers)
    is the key the search chose;
(e) broadcast and diagonal structures also run on contiguous copies (the
    broadcast expanded, the diagonal taken), within the (c) bound, bitwise
    equal when both runs take the same route and feed with one K mode (not
    stream-K: it splits a tile's k range at a point that depends on the
    tile, and the copy may order the rows differently);
(f) pointer-array batches of every structure without batch labels on every
    tile configuration its routes reach.

The group of 13 non-mergeable modes takes the regrouping fallback; with a
repeated label it is refused.
"""

import zlib

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from tests import label_oracle as lo
from tests import route_oracle as ro

pytestmark = pytest.mark.gpu

NAMES = [s.name for s in lo.STRUCTURES]
DTYPES = list(ro.QB_DTYPE)


def _rng(*salt):
    return np.random.default_rng(zlib.crc32("/".join(map(str, salt)).encode()))


def _contract(case, A, B, out=None, eng=0, **kw):
    return qb.contract_pair(A, case.la, B, case.lb, case.lc, out=out, engine=eng, **kw)


def _ints(rng, dtype):
    return lambda n: ro.int_operand(rng, n, dtype)


def _normals(rng, dtype):
    return lambda n: ro.normal_operand(rng, n, dtype)


def _ptrs(A, B, C):
    return A.data_ptr(), B.data_ptr(), C.data_ptr()


def _exact(case, key, eng):
    dtype, sent = key[0], ro.BITS[key[0]][1]
    rng = _rng(case.name, key, "exact")
    A, xa = lo.device_operand(case.A, _ints(rng, dtype), dtype)
    B, xb = lo.device_operand(case.B, _ints(rng, dtype), dtype)
    ref = lo.reference(case, xa, xb)
    for transpose in (False, True):
        Cop = lo.out_operand(case, transpose)
        cbuf, C = lo.device_output(Cop, dtype, sent)
        got = lo.route_of(case, dtype, eng, C=Cop, ptrs=_ptrs(A, B, C))
        assert ro.route_key(dtype, got) == key, got
        _contract(case, A, B, C, eng)
        np.testing.assert_array_equal(C.cpu().numpy(), ref.astype(dtype),
                                      err_msg=f"transposed output: {transpose}")
        lo.assert_outside_kept(cbuf, Cop, dtype)

    Cop = lo.out_operand(case)
    C2, c0 = lo.device_operand(Cop, _ints(rng, dtype), dtype)
    if key[1] == "zero_fill":
        # an empty sum: beta = 1 leaves C as it is, any other beta but 0 is refused
        _contract(case, A, B, C2, eng, alpha=-2.0, beta=1.0)
        np.testing.assert_array_equal(C2.cpu().numpy(), c0)
        with pytest.raises(ValueError, match=r"code -10"):
            _contract(case, A, B, C2, eng, alpha=1.0, beta=0.5)
    elif key[1] not in ("int8", "stream") or dtype in ("float32", "complex64"):
        # qb_contract_pair_ab has no engine argument: float64 / complex128
        # accumulate on DMMA, so their int8 and streaming routes are not
        # reached this way
        _contract(case, A, B, C2, eng, alpha=-2.0, beta=3.0)
        want = (-2.0 * ref + 3.0 * ro.wide(c0)).astype(dtype)
        np.testing.assert_array_equal(C2.cpu().numpy(), want, err_msg="alpha, beta")

    if dtype.startswith("complex"):
        for ca, cb in ((True, False), (False, True)):
            out = _contract(case, A, B, None, eng, conj_a=ca, conj_b=cb)
            want = lo.reference(case, xa, xb, ca, cb).astype(dtype)
            np.testing.assert_array_equal(out.cpu().numpy(), want, err_msg=f"conj {ca, cb}")


def _materialized(case):
    """The same logical contraction on contiguous operands: the diagonal of
    every repeated label taken, every broadcast expanded."""
    ua, ub = list(dict.fromkeys(case.la)), list(dict.fromkeys(case.lb))
    A = lo.dense([case.sizes[l] for l in ua])
    B = lo.dense([case.sizes[l] for l in ub])
    return lo.Case(case.name + "/contiguous", ua, ub, case.lc, case.sizes, A, B)


def _bounded(case, key, eng):
    dtype = key[0]
    rng = _rng(case.name, key, "normal")
    A, xa = lo.device_operand(case.A, _normals(rng, dtype), dtype)
    B, xb = lo.device_operand(case.B, _normals(rng, dtype), dtype)
    out1 = _contract(case, A, B, None, eng)
    out2 = _contract(case, A, B, None, eng)
    assert torch.equal(ro.bits(out1), ro.bits(out2)), "repeated call is not bit-identical"
    ref = lo.reference(case, xa, xb)
    bound = lo.bound(case, key[1], xa, xb)
    got = ro.wide(out1.cpu().numpy())
    err = np.abs(got - ref)
    assert np.all(err <= bound), f"max err / bound = {np.max(err / np.maximum(bound, 1e-300)):.3g}"

    st = lo.BY_NAME[case.name]
    if not (st.name.startswith("broadcast") or st.name.startswith("diag")) or key[1] == "zero_fill":
        return
    mc = _materialized(case)
    xa_m = np.ascontiguousarray(np.einsum(xa, case.la, mc.la))
    xb_m = np.ascontiguousarray(np.einsum(xb, case.lb, mc.lb))
    Am, Bm = torch.from_numpy(xa_m).cuda(), torch.from_numpy(xb_m).cuda()
    outm = _contract(mc, Am, Bm, None, eng)
    gotm = ro.wide(outm.cpu().numpy())
    assert np.all(np.abs(gotm - ref) <= bound), "contiguous copy outside the bound"
    rm = lo.route_of(mc, dtype, eng, ptrs=_ptrs(Am, Bm, outm))
    same_order = (ro.route_key(dtype, rm) == key and key[1] != "streamk"
                  and lo.feed_of(mc, dtype, ptrs=_ptrs(Am, Bm, outm))
                  == lo.feed_of(case, dtype, ptrs=_ptrs(A, B, out1))
                  and lo.plan_of(case, dtype)["n_k"] == 1 == lo.plan_of(mc, dtype)["n_k"])
    if same_order:
        assert torch.equal(ro.bits(outm), ro.bits(out1)), "contiguous copy not bitwise equal"


def _shapes(name, dtype):
    """{key: (M, K, N, engine)}: the pinned table on a device with its SM
    count (so a planner change that moves a shape off its key fails here
    too), else the search at this device's SM count."""
    if torch.cuda.get_device_properties(0).multi_processor_count == lo.PINNED_SMS:
        return lo.pinned_shapes(name, dtype)
    return {k: v[:4] for k, v in lo.search(name, dtype).items()}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", NAMES)
def test_structure_on_every_route(name, dtype):
    st = lo.BY_NAME[name]
    found = _shapes(name, dtype)
    assert found, f"{name} reaches no route in {dtype}"
    for key, (M, K, N, eng) in sorted(found.items(), key=str):
        case = st.make(M, K, N)
        try:
            _exact(case, key, eng)
            _bounded(case, key, eng)
        except AssertionError as e:
            raise AssertionError(f"{name} {key} M, K, N = {M, K, N}: {e}") from None


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
@pytest.mark.parametrize("name", [s.name for s in lo.STRUCTURES if not s.batch])
def test_batched_on_every_tile_config(name, dtype):
    """Pointer-array batches of 3 items, both operands conjugated for
    complex, at the shape of every tile configuration the structure's routes
    reach (the batched path runs the planner's configuration without
    split-K)."""
    st = lo.BY_NAME[name]
    shapes = {}
    for key, (M, K, N, eng) in sorted(_shapes(name, dtype).items(), key=str):
        if key[1] in ("plain", "splitk", "streamk"):
            shapes.setdefault(key[2], (M, K, N))
    # without N modes the planner never picks the 64- and 128-column tiles
    assert set(shapes) == set(range(5)) or not st.has_n, sorted(shapes)
    conj = dtype.startswith("complex")
    for cfg, (M, K, N) in sorted(shapes.items()):
        case = st.make(M, K, N)
        rng = _rng(name, dtype, cfg, "batched")
        items = [(lo.device_operand(case.A, _ints(rng, dtype), dtype),
                  lo.device_operand(case.B, _ints(rng, dtype), dtype)) for _ in range(3)]
        outs = qb.contract_batched([a for (a, _), _ in items], case.la,
                                   [b for _, (b, _) in items], case.lb, case.lc,
                                   conj_a=conj, conj_b=conj)
        for i, (((_, xa), (_, xb)), o) in enumerate(zip(items, outs)):
            want = lo.reference(case, xa, xb, conj, conj).astype(dtype)
            np.testing.assert_array_equal(o.cpu().numpy(), want,
                                          err_msg=f"{name} cfg {cfg} item {i}")


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_many_modes_take_the_regrouping_fallback(dtype):
    """13 non-mergeable modes in M (8192 rows, past the small tile): the
    operands are regrouped by the permute kernel and contracted exactly,
    into a fresh output and into a strided one; with a repeated label the
    signature is refused."""
    case = lo.many_modes()
    rng = _rng("many", dtype)
    A, xa = lo.device_operand(case.A, _ints(rng, dtype), dtype)
    B, xb = lo.device_operand(case.B, _ints(rng, dtype), dtype)
    ref = lo.reference(case, xa, xb).astype(dtype)
    np.testing.assert_array_equal(_contract(case, A, B).cpu().numpy(), ref)
    Cop = lo.out_operand(case, transpose=True)
    cbuf, C = lo.device_output(Cop, dtype, ro.BITS[dtype][1])
    _contract(case, A, B, C)
    np.testing.assert_array_equal(C.cpu().numpy(), ref)
    lo.assert_outside_kept(cbuf, Cop, dtype)
    rep = lo.many_modes(repeat=True)
    Ar, _ = lo.device_operand(rep.A, _ints(rng, dtype), dtype)
    Br, _ = lo.device_operand(rep.B, _ints(rng, dtype), dtype)
    with pytest.raises(ValueError, match="repeated label"):
        _contract(rep, Ar, Br)
