"""GPU tier: the stream-K pair schedule of the 128x128 fp64 DMMA tile.

Both stream-K schedules -- 2-CTA clusters summing two k-halves in distributed
shared memory, and the equal-cost segment loop -- must reproduce the exact
product of integer-valued operands (every partial sum is an integer far below
2^53, so the float64 result is exact in any order) bitwise, for real and
complex operands, with conjugation and with beta != 0.  The pair schedule's
output must not depend on the call, on CUDA-graph replay or on the stream, and
it must leave the stream-K flag words of the workspace zero.
"""

import pytest
import torch

import quimb_b200 as qb
from quimb_b200 import _lib
from quimb_b200.contract import _WS, capture_graph, contract_pair

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")

# (M, N, K, dtype, schedule); real K 2080 = 65 k-blocks, complex K counts
# complex elements (the tile sees 2K reals and 2N real columns)
CASES = {
    "32_tiles": (1024, 512, 2048, torch.float64, "pair"),
    "64_tiles": (1024, 1024, 2048, torch.float64, "pair"),
    "66_tiles": (768, 1408, 2048, torch.float64, "pair"),
    "odd_kblocks": (1024, 1024, 2080, torch.float64, "pair"),
    "ragged": (1000, 1000, 2048, torch.float64, "pair"),
    "ragged_odd": (1000, 1000, 2080, torch.float64, "pair"),
    "100_tiles": (1280, 1280, 2048, torch.float64, "segments"),
    "ragged_110_tiles": (1200, 1300, 2048, torch.float64, "segments"),
    "c128_32_tiles": (512, 512, 1024, torch.complex128, "pair"),
    "c128_ragged_50_tiles": (600, 620, 1040, torch.complex128, "pair"),
    "c128_72_tiles": (768, 768, 1024, torch.complex128, "segments"),
}
CODES = {torch.float64: _lib.QB_F64, torch.complex128: _lib.QB_C128}


def _ints(shape, dtype, seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    x = torch.randint(-8, 9, shape, generator=g, device=DEV).to(torch.float64)
    if dtype == torch.complex128:
        y = torch.randint(-8, 9, shape, generator=g, device=DEV).to(torch.float64)
        x = torch.complex(x, y)
    return x


def _schedule(a, b, c):
    args = []
    for t, l in ((a, [0, 1]), (b, [1, 2]), (c, [0, 2])):
        args += [list(t.shape), list(t.stride()), l]
    return qb.schedule_pair(*args, dtype_code=CODES[a.dtype],
                            ptrs=(a.data_ptr(), b.data_ptr(), c.data_ptr()))


def _operands(key, seed=0):
    M, N, K, dt, sched = CASES[key]
    A, B = _ints((M, K), dt, seed), _ints((K, N), dt, seed + 1)
    C = torch.empty((M, N), dtype=dt, device=DEV)
    assert _schedule(A, B, C) == sched
    return A, B, C


@pytest.mark.parametrize("key", sorted(CASES))
def test_exact_product(key):
    A, B, C = _operands(key)
    contract_pair(A, [0, 1], B, [1, 2], [0, 2], out=C)
    assert torch.equal(C, A @ B)


@pytest.mark.parametrize("key", ["c128_32_tiles", "c128_ragged_50_tiles", "c128_72_tiles"])
@pytest.mark.parametrize("conj", [(True, False), (False, True), (True, True)])
def test_complex_conjugation(key, conj):
    A, B, C = _operands(key, seed=3)
    contract_pair(A, [0, 1], B, [1, 2], [0, 2], conj_a=conj[0], conj_b=conj[1], out=C)
    ref = (A.conj() if conj[0] else A) @ (B.conj() if conj[1] else B)
    assert torch.equal(C, ref)


@pytest.mark.parametrize("key", ["64_tiles", "ragged_odd", "100_tiles", "c128_ragged_50_tiles"])
def test_alpha_beta(key):
    A, B, C = _operands(key, seed=5)
    C0 = _ints(tuple(C.shape), C.dtype, 7)
    C.copy_(C0)
    contract_pair(A, [0, 1], B, [1, 2], [0, 2], out=C, alpha=2.0, beta=-3.0)
    assert torch.equal(C, 2.0 * (A @ B) - 3.0 * C0)


def _normal(key):
    M, N, K, dt, _ = CASES[key]
    g = torch.Generator(device=DEV)
    g.manual_seed(11)
    A = torch.randn((M, K), dtype=dt, device=DEV, generator=g)
    B = torch.randn((K, N), dtype=dt, device=DEV, generator=g)
    return A, B


@pytest.mark.parametrize("key", ["64_tiles", "odd_kblocks", "c128_32_tiles"])
def test_pair_output_is_reproducible(key):
    # normal operands: the sum of the two k-halves is rounded, so the order of
    # every addition shows in the bits
    A, B = _normal(key)
    run = lambda: contract_pair(A, [0, 1], B, [1, 2], [0, 2])  # noqa: E731
    first = run()
    assert _schedule(A, B, first) == "pair"
    for _ in range(3):
        assert torch.equal(run(), first)
    graph, out, _scratch = capture_graph(run)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first)
    # two streams at once, each with its own workspace
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    outs = []
    for s in (s1, s2):
        with torch.cuda.stream(s):
            outs.append([run() for _ in range(3)])
    torch.cuda.synchronize()
    for o in outs:
        for x in o:
            assert torch.equal(x, first)


def test_pair_schedule_leaves_flag_words_zero():
    A, B = _normal("64_tiles")
    C = torch.empty((A.shape[0], B.shape[1]), dtype=A.dtype, device=DEV)
    assert _schedule(A, B, C) == "pair"
    for _ in range(3):
        contract_pair(A, [0, 1], B, [1, 2], [0, 2], out=C)
    torch.cuda.synchronize()
    ws = _WS[(DEV.index, torch.cuda.current_stream(DEV).cuda_stream)]
    assert not ws[:1024].any()
