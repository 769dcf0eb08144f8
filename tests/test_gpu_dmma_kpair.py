"""GPU tier: the k-pair A tile of the 128x128 fp64 DMMA tile.

The MPS-norm bra step contracts conj(A)[a', p, b'] T[a', p, b] -> E'[b', b]
with the site stored "lrp": A's rows b' sit 2 doubles apart and its k pairs
are (p = 0, 1), so its tile is staged in k-pair layout.  With integer
operands every product is exact, so each launch mode (classic grid for 128
tiles, stream-K pair schedule for 64) and both layouts of the B tile must
reproduce the exact result bitwise, on every call and under graph replay,
and the stream-K flag words stay zero.
"""

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from quimb_b200.contract import _WS, capture_graph, contract_pair

pytestmark = pytest.mark.gpu

CHI, D = 1024, 2
LB, P, RB, R = 0, 1, 2, 3


def _ints(shape, seed):
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return torch.randint(-4, 5, shape, generator=g, device="cuda").to(torch.float64)


@pytest.mark.parametrize("n", [CHI, 2 * CHI], ids=["pair", "classic"])
@pytest.mark.parametrize("tform", ["apb", "bap"])
def test_kpair_bra_exact(n, tform):
    site = _ints((CHI, CHI, D), 1).permute(0, 2, 1)          # (l, p, r), lrp storage
    if tform == "apb":
        T = _ints((CHI, D, n), 2)                                # [k][n] B tile
        lt = [LB, P, R]
    else:
        T = _ints((n, CHI, D), 2)                                # [n][k] B tile
        lt = [R, LB, P]
    la, lc = [LB, P, RB], [RB, R]
    E = torch.empty((CHI, n), dtype=torch.float64, device="cuda")
    args = (list(site.shape), list(site.stride()), la, list(T.shape), list(T.stride()), lt,
            list(E.shape), list(E.stride()), lc)
    ptrs = (site.data_ptr(), T.data_ptr(), E.data_ptr())
    assert qb.feed_pair(*args, ptrs=ptrs) == {"A": "affine", "B": "affine"}
    route = qb.route_pair(*args, ptrs=ptrs)
    assert route["layout"] == (2 if tform == "apb" else 3)
    if n == CHI:
        assert qb.schedule_pair(*args, ptrs=ptrs) == "pair"
    else:
        assert route["streamk"] == 0

    a = site.cpu().numpy().astype(np.int64)
    t = T.cpu().numpy().astype(np.int64)
    if tform == "bap":
        t = t.transpose(1, 2, 0)
    ref = np.einsum("apx,apy->xy", a, t).astype(np.float64)

    contract_pair(site, la, T, lt, lc, out=E)
    first = E.cpu().numpy()
    assert np.array_equal(first, ref)
    for _ in range(2):
        E.fill_(float("nan"))
        contract_pair(site, la, T, lt, lc, out=E)
        assert np.array_equal(E.cpu().numpy(), first)

    # another stream, then graph capture and replay
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        E.fill_(float("nan"))
        contract_pair(site, la, T, lt, lc, out=E)
    torch.cuda.current_stream().wait_stream(s)
    assert np.array_equal(E.cpu().numpy(), first)
    graph, _, _scratch = capture_graph(lambda: contract_pair(site, la, T, lt, lc, out=E))
    for _ in range(2):
        E.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(E.cpu().numpy(), first)
    ws = _WS.get((0, torch.cuda.current_stream().cuda_stream))
    assert ws is None or not ws[:1024].any()
