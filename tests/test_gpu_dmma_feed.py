"""GPU tier: the affine operand feed of the 128x128 fp64 DMMA tile gives
bitwise the results of the offset-table feed.

The same logical operands run twice or more: stored so that the planner proves
the affine feed, and as views into padded buffers (a gap every 64 rows of the
row group) that force the offset tables for A, B or both, with the same row
and k order.  Over classic and stream-K launches and the four shared-memory
layouts, every variant must be bitwise equal, reproduce the exact product of
integer operands, and stay within the DMMA error bound for normal operands.
"""

import zlib

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from tests import route_oracle as ro

pytestmark = pytest.mark.gpu

# (M, N, K): 128 tiles run the classic grid, 64 tiles with K = 2048 stream-K
SHAPES = {"classic": (1024, 2048, 1024), "streamk": (1024, 1024, 2048)}
# A stored (m, k) or (k, m), B stored (k, n) or (n, k): the four layouts
FORMS = ("mk,kn", "km,kn", "mk,nk", "km,nk")
M1, M2, K_, N1, N2 = 0, 1, 2, 3, 4


def _operand(x, rows_first, pad):
    """x: [R, K] on the device -> (tensor, labels-order) with the row mode
    split as (R / 64, 64); pad puts a 2-element gap behind every 64 rows."""
    R, K = x.shape
    e = 66 if pad else 64
    if rows_first:   # (r1, r2, k)
        buf = torch.full((R // 64, e, K), float("nan"), dtype=x.dtype, device=x.device)
        v = buf[:, :64, :]
        v.copy_(x.reshape(R // 64, 64, K))
        return v, "rrk"
    buf = torch.full((K, R // 64, e), float("nan"), dtype=x.dtype, device=x.device)
    v = buf[:, :, :64]
    v.copy_(x.t().reshape(K, R // 64, 64))
    return v, "krr"


def _labels(order, r1, r2):
    return [r1, r2, K_] if order == "rrk" else [K_, r1, r2]


def _run(form, a, b, pad_a, pad_b):
    fa, fb = form.split(",")
    A, oa = _operand(a, fa == "mk", pad_a)
    B, ob = _operand(b.t(), fb == "nk", pad_b)
    la, lb, lc = _labels(oa, M1, M2), _labels(ob, N1, N2), [M1, M2, N1, N2]
    M, N = a.shape[0], b.shape[1]
    C = torch.empty((M // 64, 64, N // 64, 64), dtype=a.dtype, device=a.device)
    feed = qb.feed_pair(list(A.shape), list(A.stride()), la, list(B.shape), list(B.stride()),
                        lb, list(C.shape), list(C.stride()), lc,
                        ptrs=(A.data_ptr(), B.data_ptr(), C.data_ptr()))
    route = qb.route_pair(list(A.shape), list(A.stride()), la, list(B.shape), list(B.stride()),
                          lb, list(C.shape), list(C.stride()), lc,
                          ptrs=(A.data_ptr(), B.data_ptr(), C.data_ptr()))
    qb.contract_pair(A, la, B, lb, lc, out=C)
    return C.reshape(M, N), feed, route


@pytest.mark.parametrize("launch", sorted(SHAPES))
@pytest.mark.parametrize("form", FORMS)
def test_affine_feed_bitwise_equals_table_feed(launch, form):
    M, N, K = SHAPES[launch]
    rng = np.random.default_rng(zlib.crc32(f"{launch}/{form}".encode()))
    dev = torch.device("cuda:0")
    for kind in ("normal", "int"):
        if kind == "int":
            a_h, b_h = ro.int_operand(rng, (M, K), "float64"), ro.int_operand(rng, (K, N), "float64")
        else:
            a_h, b_h = ro.normal_operand(rng, (M, K), "float64"), ro.normal_operand(rng, (K, N), "float64")
        a, b = torch.from_numpy(a_h).to(dev), torch.from_numpy(b_h).to(dev)
        outs, routes = {}, set()
        for pad_a in (False, True):
            for pad_b in (False, True):
                c, feed, route = _run(form, a, b, pad_a, pad_b)
                want = {"A": "table" if pad_a else "affine", "B": "table" if pad_b else "affine"}
                assert feed == want, (pad_a, pad_b, feed)
                assert route["cfg"] == 0
                assert route["kind"] == ("dmma" if launch == "classic" else "dmma_streamk")
                routes.add((route["kind"], route["layout"]))
                outs[(pad_a, pad_b)] = c.cpu().numpy()
        assert len(routes) == 1, routes
        ref = outs[(True, True)]   # offset tables for both operands
        for key, c in outs.items():
            assert np.array_equal(c.view(np.int64), ref.view(np.int64)), key
        exact = a_h @ b_h
        if kind == "int":
            np.testing.assert_array_equal(ref, exact)
        else:
            assert np.all(np.abs(ref - exact) <= ro.dmma_bound(a_h, b_h))


def test_every_layout_is_reached():
    dev = torch.device("cuda:0")
    layouts = set()
    for form in FORMS:
        for launch, (M, N, K) in SHAPES.items():
            a = torch.zeros((M, K), dtype=torch.float64, device=dev)
            b = torch.zeros((K, N), dtype=torch.float64, device=dev)
            _, _, route = _run(form, a, b, False, False)
            layouts.add((route["kind"], route["layout"]))
    assert layouts == {(k, l) for k in ("dmma", "dmma_streamk") for l in range(4)}, layouts
