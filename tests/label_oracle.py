"""Label structures of the pairwise contraction beyond the canonical forms of
``route_oracle.FORMS``: repeated (diagonal) labels, labels summed out of one
operand only, broadcast (stride-0) operands, overlapping input views, batch
modes interleaved with free modes, groups of several non-mergeable modes, and
size-1 modes sprinkled into every group.

A structure turns target logical extents (M, K, N and G for batch) into
labels, per-mode extents whose products are those targets, and the storage of
each operand.  An operand is a view ``buf.as_strided(shape, strides, offset)``
of a flat buffer of ``size`` elements, so the host planner (route search, no
device) and the device tests see the same strides.  Every element of the
buffer the view does not reach is NaN (inputs) or a sentinel (outputs).

The reference gathers each operand into a dense GEMM operand with
``np.einsum`` (diagonals taken, no sums), broadcasts it over the labels summed
out of the other operand only, and multiplies in float64 / complex128:

    a[G, M, K] @ b[G, K, N],   K = contracted x summed-out-of-A x summed-out-of-B

so K counts every summed term -- contracted, one-sided and diagonal -- and the
bounds of ``route_oracle`` (``dmma_bound``, ``int8_bound``, ``widen_bound``)
apply unchanged to these operands.
"""

import functools
import json
import math
import os
from collections import namedtuple

import numpy as np
import torch

from quimb_b200.contract import feed_pair, plan_pair, route_pair
from tests import route_oracle as ro

OFF = 4      # view offset in elements: 16-byte aligned for every dtype
GUARD = 5    # buffer elements behind the last one a view reaches

Operand = namedtuple("Operand", "shape strides offset size")
Case = namedtuple("Case", "name la lb lc sizes A B")


def dense(shape, order=None, bcast=()):
    """Contiguous storage of the axes not in `bcast` (those get stride 0),
    `order` the storage order of the axes, slowest first (default: axis
    order)."""
    shape = list(shape)
    order = list(range(len(shape))) if order is None else list(order)
    strides = [0] * len(shape)
    acc, reach = 1, 0
    stored = [ax for ax in order if ax not in bcast]
    for ax in reversed(stored):
        strides[ax] = acc
        reach += (shape[ax] - 1) * acc
        acc *= shape[ax]
    if any(e == 0 for e in shape):
        reach = 0
    return Operand(shape, strides, OFF, OFF + reach + 1 + GUARD)


def hankel(shape):
    """x[i + j] for a 2-d (M, K) view: both strides 1, rows overlap."""
    return Operand(list(shape), [1, 1], OFF, OFF + sum(shape) - 1 + GUARD)


def split(n):
    """n = d * (n / d) with d a divisor in [2, min(40, sqrt n)] nearest 6
    (1 when there is none); n = 0 gives (0, 3), an empty mode beside a
    nonempty one."""
    if n == 0:
        return 0, 3
    ds = [d for d in range(2, min(40, math.isqrt(n)) + 1) if n % d == 0]
    d = min(ds, key=lambda d: (abs(d - 6), d)) if ds else 1
    return d, n // d


def _labels(word):
    return [ord(c) - ord("a") for c in word]


# ---- the catalogue -------------------------------------------------------
class Structure:
    """One label structure: `spec` "A,B->C" in single letters, `extents(M,
    K, N, G)` -> {letter: extent}, `store(shape_a, shape_b)` -> (A, B)
    operands (default: both dense in label order); has_n: the output has N
    modes; batch: it has batch modes."""

    def __init__(self, name, spec, extents, store=None, has_n=True, batch=False):
        self.name, self.spec, self._ext, self._store = name, spec, extents, store
        self.has_n, self.batch = has_n, batch
        ins, self.wc = spec.split("->")
        self.wa, self.wb = ins.split(",")

    def make(self, M, K, N, G=ro.GROUPS):
        sz = self._ext(M, K, N, G)
        sizes = {ord(c) - ord("a"): e for c, e in sz.items()}
        sa = [sz[c] for c in self.wa]
        sb = [sz[c] for c in self.wb]
        A, B = self._store(sa, sb) if self._store else (dense(sa), dense(sb))
        return Case(self.name, _labels(self.wa), _labels(self.wb), _labels(self.wc), sizes, A, B)


def _mkn(M, K, N):
    (a, b), (k, l), (c, d) = split(M), split(K), split(N)
    return dict(a=a, b=b, k=k, l=l, c=c, d=d)


STRUCTURES = [
    # M = (a, b), K = (k, l), N = (c, d), every group interleaved
    Structure("interleaved", "akbl,lckd->cadb", lambda M, K, N, G: _mkn(M, K, N)),
    # the same with A stored mode-fastest and B stored k-fastest
    Structure("interleaved_t", "akbl,lckd->cadb", lambda M, K, N, G: _mkn(M, K, N),
              store=lambda sa, sb: (dense(sa, order=(1, 3, 0, 2)), dense(sb, order=(1, 3, 0, 2)))),
    # diagonal of a contracted label (b): K = (b, k)
    Structure("diag_contracted", "abbck,bkd->acd",
              lambda M, K, N, G: dict(zip("ac", split(M)), **dict(zip("bk", split(K))), d=N)),
    # diagonal of a free label (a): M = (a, m)
    Structure("diag_free", "aamk,kn->amn",
              lambda M, K, N, G: dict(zip("am", split(M)), k=K, n=N)),
    # diagonal of a batch label (g)
    Structure("diag_batch", "ggmk,gkn->gmn", lambda M, K, N, G: dict(g=G, m=M, k=K, n=N),
              batch=True),
    # e summed out of A only: K = (e, k), e of stride 0 in B
    Structure("summed_a", "mke,kn->mn", lambda M, K, N, G: dict(zip("ek", split(K)), m=M, n=N)),
    # f summed out of B only, B stored k-fastest
    Structure("summed_b", "mk,kfn->mn", lambda M, K, N, G: dict(zip("fk", split(K)), m=M, n=N),
              store=lambda sa, sb: (dense(sa), dense(sb, order=(2, 1, 0)))),
    # both at once, A stored m-fastest: K = (e, f, k)
    Structure("summed_both", "mke,kfn->mn",
              lambda M, K, N, G: dict(e=split(K)[0], **dict(zip("fk", split(split(K)[1]))),
                                      m=M, n=N),
              store=lambda sa, sb: (dense(sa, order=(1, 2, 0)), dense(sb))),
    # A expanded along a free mode (b, stride 0)
    Structure("broadcast_free", "mbk,kn->bmn",
              lambda M, K, N, G: dict(zip("bm", split(M)), k=K, n=N),
              store=lambda sa, sb: (dense(sa, bcast=(1,)), dense(sb))),
    # A expanded along a contracted mode (l, stride 0)
    Structure("broadcast_contracted", "mkl,kln->mn",
              lambda M, K, N, G: dict(zip("lk", split(K)), m=M, n=N),
              store=lambda sa, sb: (dense(sa, bcast=(2,)), dense(sb))),
    # A expanded along the batch mode
    Structure("broadcast_batch", "gmk,gkn->gmn", lambda M, K, N, G: dict(g=G, m=M, k=K, n=N),
              store=lambda sa, sb: (dense(sa, bcast=(0,)), dense(sb)), batch=True),
    # overlapping rows: A[m, k] = x[m + k] (input only), B stored k-fastest
    Structure("hankel", "mk,kn->mn", lambda M, K, N, G: dict(m=M, k=K, n=N),
              store=lambda sa, sb: (hankel(sa), dense(sb, order=(1, 0)))),
    # two batch modes (g, h) interleaved with the free modes in every tensor
    Structure("batch_interleaved", "agbh,bhcg->cgah",
              lambda M, K, N, G: dict(a=M, b=K, c=N, g=G, h=3), batch=True),
    # extent-1 labels in every group: free (u, w), contracted (v), batch (x),
    # summed out of A (y)
    Structure("size_one", "akuxbvly,lcvxkdw->cuaxdwb",
              lambda M, K, N, G: dict(_mkn(M, K, N), u=1, v=1, w=1, x=1, y=1)),
    # no N modes: a multi-mode matrix-vector product
    Structure("matvec", "akbl,lk->ba",
              lambda M, K, N, G: dict(zip("ab", split(M)), **dict(zip("kl", split(K)))),
              has_n=False),
]
BY_NAME = {s.name: s for s in STRUCTURES}

MANY = 13   # non-mergeable modes of one group: one more than the planner takes


def many_modes(repeat=False, ext=2, K=40, N=72):
    """A [m0 .. m12, k], B [k, n] -> C [n, m12 .. m0]: the 13 modes of M
    (2^13 rows) are contiguous in A and in C but in opposite orders, so no two
    merge.  repeat: A also holds a diagonal label r, contracted with B."""
    m = list(range(MANY))
    k, n, r = MANY, MANY + 1, MANY + 2
    la, lb, lc = m + [k], [k, n], [n] + m[::-1]
    sizes = {**{l: ext for l in m}, k: K, n: N, r: 3}
    if repeat:
        la, lb = la + [r, r], [r] + lb
    A = dense([sizes[l] for l in la])
    B = dense([sizes[l] for l in lb])
    return Case("many_modes", la, lb, lc, sizes, A, B)


# ---- label groups and the reference --------------------------------------
def groups(la, lb, lc):
    ua, ub = list(dict.fromkeys(la)), list(dict.fromkeys(lb))
    batch = [l for l in lc if l in ua and l in ub]
    free_a = [l for l in lc if l in ua and l not in ub]
    free_b = [l for l in lc if l in ub and l not in ua]
    con = [l for l in ua if l in ub and l not in lc]
    sum_a = [l for l in ua if l not in ub and l not in lc]
    sum_b = [l for l in ub if l not in ua and l not in lc]
    return batch, free_a, free_b, con, sum_a, sum_b


def logical(case):
    """(G, M, K, N) with K over every summed term."""
    batch, free_a, free_b, con, sum_a, sum_b = groups(case.la, case.lb, case.lc)
    p = lambda ls: math.prod(case.sizes[l] for l in ls)  # noqa: E731
    return p(batch), p(free_a), p(con + sum_a + sum_b), p(free_b)


def macs(case, dtype):
    G, M, K, N = logical(case)
    return G * M * K * N * (4 if dtype.startswith("complex") else 1)


def gemm_operands(case, xa, xb):
    """Logical operands (numpy, axes as labelled) -> a [G, M, K], b [G, K, N]
    in their own dtype: diagonals taken, each broadcast over the labels
    summed out of the other operand only."""
    batch, free_a, free_b, con, sum_a, sum_b = groups(case.la, case.lb, case.lc)
    ext = lambda ls: [case.sizes[l] for l in ls]  # noqa: E731
    G, M, K, N = logical(case)
    ta = np.einsum(xa, case.la, batch + free_a + con + sum_a)
    ta = np.broadcast_to(ta.reshape(ext(batch + free_a + con + sum_a) + [1] * len(sum_b)),
                         ext(batch + free_a + con + sum_a + sum_b))
    tb = np.einsum(xb, case.lb, batch + con + sum_b + free_b)
    tb = np.broadcast_to(tb.reshape(ext(batch + con) + [1] * len(sum_a) + ext(sum_b + free_b)),
                         ext(batch + con + sum_a + sum_b + free_b))
    return (np.ascontiguousarray(ta).reshape(G, M, K),
            np.ascontiguousarray(tb).reshape(G, K, N))


def to_out(case, c):
    """[G, M, N] -> the output's axes in lc order."""
    batch, free_a, free_b, *_ = groups(case.la, case.lb, case.lc)
    order = batch + free_a + free_b
    c = c.reshape([case.sizes[l] for l in order])
    return c.transpose([order.index(l) for l in case.lc])


def reference(case, xa, xb, conj_a=False, conj_b=False):
    """The contraction in float64 / complex128, axes in lc order."""
    a, b = gemm_operands(case, xa, xb)
    a, b = ro.wide(a), ro.wide(b)
    return to_out(case, (a.conj() if conj_a else a) @ (b.conj() if conj_b else b))


def bound(case, kind, xa, xb):
    """Per-element bound of route kind `kind` against ``reference``."""
    a, b = gemm_operands(case, xa, xb)
    return to_out(case, ro.route_bound(kind, a, b))


def out_operand(case, transpose=False):
    """Dense output in lc order; transpose: stored with the axis order
    reversed (every output stride permuted)."""
    shape = [case.sizes[l] for l in case.lc]
    order = list(reversed(range(len(shape)))) if transpose else None
    return dense(shape, order=order)


# ---- host-side planner queries ---------------------------------------------
BASE = 0x10000000   # 256-byte aligned fake base address of host-only queries


def ptr(op, dtype, base=BASE):
    return base + op.offset * ro.TORCH[dtype].itemsize


def _args(case, C):
    return (case.A.shape, case.A.strides, case.la, case.B.shape, case.B.strides, case.lb,
            C.shape, C.strides, case.lc)


def route_of(case, dtype, engine=0, C=None, ptrs=None):
    C = out_operand(case) if C is None else C
    if ptrs is None:
        ptrs = (ptr(case.A, dtype), ptr(case.B, dtype), ptr(C, dtype))
    return route_pair(*_args(case, C), ro.QB_DTYPE[dtype], engine, ptrs=ptrs)


def feed_of(case, dtype, C=None, ptrs=None):
    C = out_operand(case) if C is None else C
    if ptrs is None:
        ptrs = (ptr(case.A, dtype), ptr(case.B, dtype), ptr(C, dtype))
    return feed_pair(*_args(case, C), ro.QB_DTYPE[dtype], ptrs=ptrs)


def plan_of(case, dtype="float64"):
    return plan_pair(*_args(case, out_operand(case)), ro.QB_DTYPE[dtype])


# ---- route search over structures ------------------------------------------
# 259 = 7 x 37 and 1036 = 28 x 37: groups whose modes do not divide the tiles
SIZES = (64, 130, 259, 384, 512, 768, 1024, 1036, 1536, 2048, 4096, 16384)
MAX_MACS = 1.2e9    # host reference work per chosen shape (complex: 4 real MACs)


def _engines(dtype):
    return (0, ro.ENGINE_INT8) if dtype in ("float64", "complex128") else (0,)


def _grid(st):
    for M in SIZES:
        for K in SIZES:
            for N in (SIZES if st.has_n else (1,)):
                yield M, K, N


@functools.lru_cache(maxsize=None)
def search(name, dtype):
    """Cheapest grid shape of structure `name` for every route key it reaches
    in `dtype`: {key: (M, K, N, engine, route)}; the streaming variants at
    their largest operator on the streaming grid (then the cheapest)."""
    st = BY_NAME[name]
    best = {}
    for M, K, N in _grid(st):
        case = st.make(M, K, N)
        cost = macs(case, dtype)
        if cost > MAX_MACS:
            continue
        for eng in _engines(dtype):
            r = route_of(case, dtype, eng)
            key = ro.route_key(dtype, r)
            if key is None or (eng == ro.ENGINE_INT8 and key[1] != "int8"):
                continue
            if key not in best or cost < best[key][0]:
                best[key] = (cost, (M, K, N, eng, r))
    # zero fill: an empty mode in the K group
    M, N = ro.ZERO_FILL_M, ro.ZERO_FILL_N if st.has_n else 1
    r = route_of(st.make(M, 0, N), dtype)
    key = ro.route_key(dtype, r)
    if key is not None:
        best[key] = (0, (M, 0, N, 0, r))
    if dtype in ro.STREAM_VARIANTS:
        shapes = {}
        for K in ro.STREAM_KN:
            for N in (ro.STREAM_KN if st.has_n else (1,)):
                case = st.make(ro.STREAM_M, K, N)
                r = route_of(case, dtype, ro.ENGINE_STREAM)
                key = ro.route_key(dtype, r)
                if key is not None and key[1] == "stream":
                    _, Mc, Kc, Nc = logical(case)
                    shapes.setdefault(key, []).append(
                        ((Kc * Nc, -macs(case, dtype)), (ro.STREAM_M, K, N, ro.ENGINE_STREAM, r)))
        for key, s in shapes.items():
            best[key] = (None, max(s, key=lambda x: x[0])[1])
    return {k: v[1] for k, v in best.items()}


# Route keys a structure cannot reach by design, with the reason in the code.
def unreachable(st, key):
    dtype, kind = key[0], key[1]
    if st.batch and kind in ("streamk", "int8") and dtype in ("float64", "complex128"):
        return "stream-K and the int8 engine need nbatch == 1 (plan_pair, ozaki_eligible)"
    if st.batch and dtype in ("float32", "complex64") and kind == "int8":
        return "single precision with batch modes takes the widen path (ozaki_eligible)"
    return None


PINNED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "label_routes.json")
PINNED_SMS = 132    # the table is the search at the H100 SXM's SM count


def pinned_table():
    """{structure: [[key, [M, K, N, engine]], ...]} as pinned in the golden
    file."""
    with open(PINNED) as f:
        return json.load(f)


def pinned_shapes(name, dtype):
    """{key: (M, K, N, engine)} of structure `name` in `dtype` from the
    pinned table."""
    return {tuple(k): tuple(v) for k, v in pinned_table()[name] if k[0] == dtype}


def coverage():
    """{structure: {key: (M, K, N, engine, route)}} over every dtype."""
    return {st.name: {k: v for dt in ro.QB_DTYPE for k, v in search(st.name, dt).items()}
            for st in STRUCTURES}


# ---- device operands ---------------------------------------------------------
def index_map(op):
    """Buffer index of every element of the view (numpy, the view's shape)."""
    flat = torch.arange(op.size, dtype=torch.int64)
    return flat.as_strided(op.shape, op.strides, op.offset).numpy()


def device_operand(op, values_of, dtype):
    """Flat NaN buffer on the device holding the view `op`; the elements the
    view reaches come from values_of(count).  Returns (view, logical numpy
    operand with the view's shape)."""
    idx = index_map(op)
    reach = np.unique(idx)
    host = np.full(op.size, np.nan, dtype=dtype)
    if np.iscomplexobj(host):
        host += 1j * np.nan
    host[reach] = values_of(reach.size)
    buf = torch.from_numpy(host).cuda()
    return buf.as_strided(op.shape, op.strides, op.offset), host[idx]


def device_output(op, dtype, fill_bits):
    """Flat buffer of the sentinel bit pattern and the view `op` into it."""
    buf = torch.empty(op.size, dtype=ro.TORCH[dtype], device="cuda")
    ro.bits(buf).fill_(fill_bits)
    return buf, buf.as_strided(op.shape, op.strides, op.offset)


def assert_outside_kept(buf, op, dtype):
    """Every buffer element the output view does not reach keeps the
    sentinel bits."""
    mask = np.zeros(op.size, dtype=bool)
    mask[np.unique(index_map(op))] = True
    ro.assert_sentinel_kept(buf, mask, dtype)
