"""Results must not depend on the caller's stream, on other streams running at
the same time, or on CUDA-graph capture.

Every other GPU module runs one call at a time on the legacy default stream,
which hides three classes of error: work enqueued on a stream other than the
caller's, scratch memory shared by two streams, and scratch that a captured
graph references but whose initialisation never ran.  The cases here:

* A. each entry-point family runs on a fresh stream whose inputs are copied in
  behind a ``torch.cuda._sleep``; anything not ordered on that stream reads
  NaN sentinels.  Results are compared bitwise with the same call made on the
  default stream (the kernels are deterministic).
* B. four streams run dot products, Krylov orthogonalisation, contractions and
  convert / permute at once; every result equals its serial one bitwise.  A
  recorder on the library's scratch-taking entry points asserts that no
  scratch range is handed to two streams.
* C. ``GraphedContraction`` and ``ChainPlan`` at shapes that plan a stream-K
  step: two plans replayed in either order equal eager execution bitwise, no
  scratch is allocated while a capture is open, and two plans replay on two
  streams at once.
* D. ``mps_norm2`` over host sites (staged through a ring of device buffers
  on a copy stream) equals the same call over device copies bitwise.

Stream-K launches are persistent grids whose CTAs wait on one another, so two
of them must never run at the same time (DESIGN.md §3): every concurrent case
checks its routes before it launches, and the recorder refuses a stream-K
launch while concurrency is on.
"""

import ctypes

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from oracle import dmrg_np as dm
from quimb_b200 import _lib, contract, lanczos, linalg, ops
from quimb_b200 import mps as qmps
from quimb_b200 import tree as qtree
from quimb_b200.array import Array
from quimb_b200.contract import ROUTE_KINDS, contract_pair, route_pair

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 100_000_000          # ~50 ms at the H100's boost clock
TORCH = {"float32": torch.float32, "float64": torch.float64,
         "complex64": torch.complex64, "complex128": torch.complex128}


# ---------------------------------------------------------------- helpers ---
def _strides(shape):
    st, acc = [], 1
    for e in reversed(shape):
        st.append(acc)
        acc *= max(e, 1)
    return list(reversed(st))


def route_of(a, la, b, lb, out, lc, engine=0):
    """The route ``contract_pair`` takes for these very tensors."""
    return route_pair(list(a.shape), list(a.stride()), la, list(b.shape), list(b.stride()), lb,
                      list(out.shape), list(out.stride()), lc, _lib.qb_dtype(a.dtype), engine,
                      ptrs=(a.data_ptr(), b.data_ptr(), out.data_ptr()))


def to_host(x):
    """Host copy of a (nested) result, for bitwise comparison."""
    if x is None:
        return None
    if isinstance(x, (tuple, list)):
        return [to_host(v) for v in x]
    if isinstance(x, dict):
        return {k: to_host(v) for k, v in x.items()}
    if isinstance(x, Array):
        return x.to_numpy()
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy()
    return np.asarray(x)


def assert_bits(got, ref, where="result"):
    if ref is None:
        assert got is None, where
        return
    if isinstance(ref, list):
        assert isinstance(got, list) and len(got) == len(ref), where
        for i, (g, r) in enumerate(zip(got, ref)):
            assert_bits(g, r, f"{where}[{i}]")
        return
    if isinstance(ref, dict):
        assert sorted(got) == sorted(ref), where
        for k in ref:
            assert_bits(got[k], ref[k], f"{where}[{k!r}]")
        return
    assert got.dtype == ref.dtype and got.shape == ref.shape, (where, got.dtype, ref.dtype,
                                                               got.shape, ref.shape)
    g = np.ascontiguousarray(got).view(np.uint8)
    r = np.ascontiguousarray(ref).view(np.uint8)
    assert np.array_equal(g, r), f"{where} differs from the serial result"


def sentinel_like(t):
    out = torch.empty_like(t)
    if t.is_floating_point() or t.is_complex():
        return ops_nan(out)
    return out.fill_(-7)


def ops_nan(buf):
    buf.fill_(complex(float("nan"), float("nan")) if buf.is_complex() else float("nan"))
    return buf


def check_on_fresh_stream(fn, *srcs):
    """``fn(*tensors)`` on a fresh stream whose inputs hold NaN sentinels until
    a copy queued behind a ~50 ms sleep, against ``fn`` on the default stream."""
    ref = to_host(fn(*[t.clone() for t in srcs]))
    torch.cuda.synchronize()
    dst = [sentinel_like(t) for t in srcs]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for d, t in zip(dst, srcs):
            d.copy_(t)
        got = to_host(fn(*dst))
    torch.cuda.synchronize()
    assert_bits(got, ref)
    return got


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def randn(rng, shape, dtype="float64"):
    x = rng.standard_normal(shape)
    if "complex" in dtype:
        x = x + 1j * rng.standard_normal(shape)
    return dev(x.astype(dtype))


# --------------------------------------------------- scratch bookkeeping ---
# entry point -> (index of the scratch pointer, index of its size, or a
# function of the library giving the fixed size); the stream is the last arg
_SCRATCH_ARGS = {
    "qb_dot": (5, lambda lib: lib.qb_dot_workspace(0)),
    "qb_multi_dot": (7, lambda lib: lib.qb_multi_dot_workspace()),
    "qb_contract_pair": (9, 10),
    "qb_contract_pair_ab": (10, 11),
    "qb_qr_stab": (7, 8),
    "qb_svd": (7, 8),
    "qb_svd_trunc": (15, 16),
}


def _value(a):
    v = getattr(a, "value", a)
    return 0 if v is None else int(v)


class ScratchRecorder:
    """Wraps the scratch-taking entry points of the loaded library: records
    ``(entry, first byte, end, stream, capturing)`` of every call and the route kind of
    every contraction; with ``forbid_streamk`` set it refuses a stream-K
    contraction before it is launched."""

    def __init__(self, monkeypatch):
        self.lib = lib = _lib.load()
        self.calls, self.routes = [], []
        self.forbid_streamk = False
        for name, (pi, si) in _SCRATCH_ARGS.items():
            monkeypatch.setattr(lib, name, self._wrap(name, getattr(lib, name), pi, si))

    def _wrap(self, name, orig, pi, si):
        lib = self.lib

        def call(*args):
            if name.startswith("qb_contract_pair"):
                out = (ctypes.c_int64 * 16)()
                eng = (args[8] & 0xFF) if name == "qb_contract_pair" else 0
                if lib.qb_contract_pair_route(*args[:6], eng, out) == 0:
                    kind = ROUTE_KINDS[out[0]]
                    self.routes.append(kind)
                    if self.forbid_streamk and kind == "dmma_streamk":
                        raise AssertionError("a stream-K contraction while streams run concurrently")
            ptr = _value(args[pi])
            size = si(lib) if callable(si) else _value(args[si])
            if ptr and size:
                self.calls.append((name, ptr, ptr + size, _value(args[-1]),
                                   torch.cuda.is_current_stream_capturing()))
            return orig(*args)
        return call

    def shared_ranges(self):
        """Pairs of scratch ranges that overlap but were given to two streams."""
        seen = sorted(set(c[1:4] for c in self.calls))
        bad = []
        for i, (lo, hi, st) in enumerate(seen):
            for lo2, hi2, st2 in seen[i + 1:]:
                if lo2 >= hi:
                    break
                if st2 != st:
                    bad.append(((lo, hi, st), (lo2, hi2, st2)))
        return bad


@pytest.fixture
def scratch(monkeypatch):
    return ScratchRecorder(monkeypatch)


@pytest.fixture
def scratch_allocs(monkeypatch):
    """Wraps the package's scratch helpers; records (helper, capturing) for
    every buffer they allocate."""
    allocs = []
    for mod, fname, cache in ((contract, "_workspace", contract._WS),
                              (linalg, "_workspace", linalg._WS),
                              (ops, "_dot_ws", ops._DOT_WS),
                              (lanczos, "_md_ws", lanczos._MD_WS)):
        def wrapped(*a, _orig=getattr(mod, fname), _cache=cache, _name=fname, **k):
            before = {id(v) for v in _cache.values()}
            buf = _orig(*a, **k)
            if id(buf) not in before:
                allocs.append((_name, torch.cuda.is_current_stream_capturing()))
            return buf
        monkeypatch.setattr(mod, fname, wrapped)
    return allocs


# ------------------------------------------ A. ordering on the caller's stream
# one shape per route kind (float64 unless noted): (dtype, M, K, N, engine)
ROUTE_CASES = {
    "empty": ("float64", 0, 8, 8, 0),
    "zero_fill": ("float64", 3, 0, 5, 0),
    "widen": ("float32", 64, 64, 64, 0),
    "int8": ("float32", 512, 512, 512, 0),
    "stream": ("float64", 785, 16, 16, _lib.QB_ENGINE_STREAM),
    "dmma": ("complex128", 130, 130, 130, 0),
    "dmma_streamk": ("float64", 384, 384, 4096, 0),
}


def test_route_cases_cover_every_route_kind():
    assert sorted(ROUTE_CASES) == sorted(ROUTE_KINDS)


@pytest.mark.parametrize("kind", sorted(ROUTE_CASES))
def test_contract_pair_is_ordered_on_the_callers_stream(kind):
    dt, M, K, N, eng = ROUTE_CASES[kind]
    rng = np.random.default_rng(hash(kind) % 2 ** 32)
    a, b = randn(rng, (K, M), dt), randn(rng, (K, N), dt)       # a read transposed
    la, lb, lc = [1, 0], [1, 2], [0, 2]
    probe = torch.empty((M, N), dtype=TORCH[dt], device="cuda")
    assert route_of(a, la, b, lb, probe, lc, eng)["kind"] == kind

    def fn(a, b):
        out = torch.empty((M, N), dtype=a.dtype, device=a.device)
        assert route_of(a, la, b, lb, out, lc, eng)["kind"] == kind
        return contract_pair(a, la, b, lb, lc, out=out, engine=eng)
    check_on_fresh_stream(fn, a, b)


def test_contract_pair_accumulate_into_strided_out_is_ordered():
    rng = np.random.default_rng(1)
    a, b = randn(rng, (256, 192)), randn(rng, (192, 320))
    base = randn(rng, (320, 2 * 256 + 3))          # out = base[:, 1:513:2].T, strided

    def fn(a, b, base):
        out = base[:, 1:513:2].t()
        r = route_of(a, [0, 1], b, [1, 2], out, [0, 2])
        assert r["kind"] == "dmma"
        contract_pair(a, [0, 1], b, [1, 2], [0, 2], out=out, alpha=0.75, beta=-1.25)
        return base
    check_on_fresh_stream(fn, a, b, base)


def test_batched_convert_and_permute_are_ordered():
    rng = np.random.default_rng(2)
    A, B = randn(rng, (6, 24, 32), "complex128"), randn(rng, (6, 32, 16), "complex128")
    X = randn(rng, (5, 6, 7, 8, 3, 4, 2, 3, 2, 2, 3, 2))     # rank 12: several passes

    def fn(A, B, X):
        outs = contract.contract_batched(list(A), [0, 1], list(B), [1, 2], [0, 2], conj_b=True)
        order = [11, 3, 7, 0, 9, 1, 5, 10, 2, 8, 4, 6]
        return (outs, contract.convert(X[:, ::2].transpose(0, 3), torch.float32),
                contract.convert(A, torch.complex64), contract.permute_contiguous(X, order),
                contract.permute_contiguous(A, [2, 0, 1], conj=True))
    check_on_fresh_stream(fn, A, B, X)


@pytest.mark.parametrize("dtype", ["float64", "complex128", "float32"])
def test_vector_kernels_are_ordered(dtype):
    rng = np.random.default_rng(3)
    n = (1 << 20) + 37
    x, y, d = randn(rng, (n,), dtype), randn(rng, (n,), dtype), dev(np.array(3.5))

    def fn(x, y, d):
        dot = ops.vdot(Array(x), Array(y))
        nrm = linalg.norm(Array(x))
        ops.axpby(0.5 - 0.25j if x.is_complex() else 0.5, Array(x), -2.0, Array(y))
        ops.scale_(Array(x), 1.5, div_by=Array(d))
        z = torch.empty_like(y)
        ops.scale_into(Array(z), Array(y), -0.75, div_by=Array(d))
        return dot, nrm, x, y, z
    check_on_fresh_stream(fn, x, y, d)


def test_eigh_lanczos_with_a_dense_matvec_is_ordered():
    rng = np.random.default_rng(4)
    n = 300
    h = rng.standard_normal((n, n))
    H, v0 = dev(h + h.T), randn(rng, (n,))

    def fn(H, v0):
        mv = lambda v: Array(contract_pair(H, [0, 1], v.t, [1], [0]))  # noqa: E731
        return qb.eigh_lanczos(mv, Array(v0), ncv=16, tol=1e-10)
    check_on_fresh_stream(fn, H, v0)


def test_qr_svd_eigh_cholesky_are_ordered():
    rng = np.random.default_rng(5)
    X, Y = randn(rng, (200, 150)), randn(rng, (300, 200), "complex128")
    h = rng.standard_normal((96, 96))
    S = dev(h @ h.T + 96 * np.eye(96))        # n > 64: the device eigensolver

    def fn(X, Y, S):
        res = [linalg.qr(Array(X)), linalg.qr(Array(Y), stabilized=True), linalg.svd(Array(X)),
               linalg.eigh(Array(S)), linalg.cholesky(Array(S))]
        for code in (0, -1, 1, 2):            # accumulate, left, right, values-only
            info = {"error": None}
            res.append(linalg.svd_trunc(Array(X), cutoff=1e-3, absorb=code, info=info))
            res.append([info["error"], info["n_keep"]])
        return res
    assert [linalg.route_svd((200, 150), absorb=c)["epilogue"] for c in (0, -1, 1, 2)] == \
        ["accumulate", "left", "right", "values"]
    check_on_fresh_stream(fn, X, Y, S)


def test_array_split_is_ordered():
    rng = np.random.default_rng(6)
    X = randn(rng, (120, 90))

    def fn(X):
        return [qb.array_split(Array(X), method=m, max_bond=40, cutoff=1e-6)
                for m in ("svd", "svd:eig", "qr")]
    check_on_fresh_stream(fn, X)


def test_mps_sample_and_stripped_tree_are_ordered():
    sites = [dev(a) for a in dm.mps_rand(8, 16, seed=7, dtype="complex128")]
    rng = np.random.default_rng(8)
    arrays = [randn(rng, (6, 7, 5)), randn(rng, (5, 7, 9)), randn(rng, (9, 6, 4))]
    for i, t in enumerate(arrays):
        t.mul_(10.0 ** (40 * (i + 1)))        # the exponent is what strip_exponent keeps
    inputs, output = [("a", "b", "c"), ("c", "b", "d"), ("d", "a", "e")], ("e",)

    def fn(*ts):
        configs, omegas = qb.mps_sample([Array(t) for t in ts[:8]], 64, seed=9)
        tr = qtree.find_tree(inputs, output, qtree._sizes(inputs, ts[8:]), "greedy")
        mant, expo = qtree.execute(tr, [Array(t) for t in ts[8:]], strip_exponent=True)
        return configs, omegas, mant, expo
    check_on_fresh_stream(fn, *sites, *arrays)


def test_dmrg2_sweep_is_ordered():
    mpo = dm.mpo_heis(6)

    def run():
        d = qb.DMRG2(mpo, [8, 16], cutoffs=1e-10, mpo_shape="lrdu", seed=2)
        d.solve(tol=1e-12, max_sweeps=1)
        return [np.array(d.energies), d.state]
    ref = to_host(run())
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)       # everything, the MPO upload included, waits
        got = to_host(run())
    torch.cuda.synchronize()
    assert_bits(got, ref)


# ------------------------------------------------------ B. concurrent streams
def _stream_data(seed):
    rng = np.random.default_rng(seed)
    n = 1 << 21
    return {"x": randn(rng, (n,)), "y": randn(rng, (n,)), "z": randn(rng, (n,), "complex128"),
            "V": randn(rng, (20, n // 8)), "w": randn(rng, (n // 8,)),
            "a": randn(rng, (256, 1024)), "b": randn(rng, (1024, 256)),
            "c": randn(rng, (256, 256), "complex128"), "T": randn(rng, (12, 34, 56, 3))}


def _stream_work(D):
    """Everything one stream enqueues; no host synchronisation."""
    V, w = D["V"], D["w"].clone()
    h = torch.zeros(32, dtype=torch.float64, device="cuda")
    keep = torch.zeros(32, dtype=torch.float64, device="cuda")
    lanczos._orthogonalise(V, 19, w, h, keep=keep)
    out = torch.empty((256, 256), dtype=torch.float64, device="cuda")
    return [ops.vdot(Array(D["x"]), Array(D["y"])).t, linalg.norm(Array(D["z"])).t,
            ops.vdot(Array(D["z"]), Array(D["z"])).t, w, h, keep,
            contract_pair(D["a"], [0, 1], D["b"], [1, 2], [0, 2], out=out),
            contract_pair(D["c"], [0, 1], D["c"], [2, 1], [0, 2], conj_b=True),
            contract.convert(D["T"][:, 1::2].transpose(1, 2), torch.float32),
            contract.permute_contiguous(D["T"], [3, 1, 0, 2])]


def test_four_streams_at_once_equal_serial_and_never_share_scratch(scratch):
    data = [_stream_data(10 + k) for k in range(4)]
    D = data[0]
    # the contractions must not plan stream-K (they run concurrently below)
    out = torch.empty((256, 256), dtype=torch.float64, device="cuda")
    r = route_of(D["a"], [0, 1], D["b"], [1, 2], out, [0, 2])
    assert r["kind"] == "dmma" and r["splitk"] > 1         # split-K partials in the scratch
    assert route_of(D["c"], [0, 1], D["c"], [2, 1], D["c"], [0, 2])["kind"] == "dmma"
    serial = [to_host(_stream_work(Dk)) for Dk in data]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(4)]
    scratch.forbid_streamk = True
    rounds = 3
    results = [[None] * 4 for _ in range(rounds)]
    for rd in range(rounds):
        for k, s in enumerate(streams):       # operation by operation across the streams
            with torch.cuda.stream(s):
                results[rd][k] = _stream_work(data[k])
    torch.cuda.synchronize()
    scratch.forbid_streamk = False
    assert "dmma_streamk" not in scratch.routes
    for rd in range(rounds):
        for k in range(4):
            assert_bits(to_host(results[rd][k]), serial[k], f"round {rd} stream {k}")
    bad = scratch.shared_ranges()
    assert not bad, f"scratch handed to two streams: {bad[:4]}"


def test_scratch_recorder_sees_every_scratch_family(scratch):
    """The ownership check above is only as good as its coverage: every
    scratch-taking entry point reports its range and stream."""
    rng = np.random.default_rng(11)
    X = randn(rng, (200, 150))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        linalg.qr(Array(X))
        linalg.svd(Array(X))
        linalg.svd_trunc(Array(X), cutoff=1e-3, absorb=0)
        D = _stream_data(12)
        contract_pair(D["a"], [0, 1], D["b"], [1, 2], [0, 2], alpha=2.0)    # split-K
        _stream_work(D)
    torch.cuda.synchronize()
    names = {c[0] for c in scratch.calls}
    assert names == set(_SCRATCH_ARGS), names
    assert {c[3] for c in scratch.calls} == {s.cuda_stream}
    assert not any(c[4] for c in scratch.calls)
    assert not scratch.shared_ranges()


# ----------------------------------------------------------- C. graph capture
def _sites(rng, L, chi, d, dtype="float64"):
    bonds = [1] + [chi] * (L - 1) + [1]
    return [randn(rng, (bonds[i], d, bonds[i + 1]), dtype) for i in range(L)]


def _mpo(rng, L, w, d):
    bonds = [1] + [w] * (L - 1) + [1]
    return [randn(rng, (bonds[i], bonds[i + 1], d, d)) for i in range(L)]


def _eager_chain(kind, sites, mpo):
    if kind == "norm":
        return qb.mps_norm2(sites, "lpr")
    if kind == "expec":
        return qb.mps_expec(sites, mpo, "lpr", "lrud")
    return qb.compute_left_environments(sites, None, "lpr")


def _overlap(r1, r2):
    return [(a, b) for a in r1 for b in r2 if a[0] < b[1] and b[0] < a[1]]


def _captured_ranges(calls):
    return {(c[1], c[2]) for c in calls if c[4]}


def _cached_ranges():
    """Scratch any later eager call or capture can be handed."""
    return {(b.data_ptr(), b.data_ptr() + b.numel())
            for cache in (contract._WS, linalg._WS, ops._DOT_WS, lanczos._MD_WS)
            for b in cache.values()}


def _build_two(scratch, make):
    """Two plans built in a row, and the scratch each one's graph captured."""
    n0 = len(scratch.calls)
    p1 = make()
    n1 = len(scratch.calls)
    p2 = make()
    return p1, p2, _captured_ranges(scratch.calls[n0:n1]), _captured_ranges(scratch.calls[n1:])


def _assert_plans_own_scratch(r1, r2, scratch_allocs):
    assert r1 and r2
    assert not _overlap(r1, r2), "two captured plans share scratch"
    assert not _overlap(r1 | r2, _cached_ranges()), "captured scratch is reachable by later calls"
    assert not [a for a in scratch_allocs if a[1]], f"scratch allocated during capture: {scratch_allocs}"


CHAIN = dict(L=3, chi=320, d=16, w=2)   # the smallest chains whose site-1 step is stream-K


@pytest.mark.parametrize("kind", ["norm", "expec", "left_envs"])
def test_chain_plans_own_their_scratch(kind, scratch, scratch_allocs):
    rng = np.random.default_rng(20)
    L, chi, d, w = CHAIN["L"], CHAIN["chi"], CHAIN["d"], CHAIN["w"]
    sites, mpo = _sites(rng, L, chi, d), _mpo(rng, L, w, d)
    m = mpo if kind == "expec" else None
    p1, p2, r1, r2 = _build_two(scratch, lambda: qb.ChainPlan(sites, m, shape="lpr", kind=kind))
    assert "dmma_streamk" in scratch.routes
    for p in (p2, p1, p2, p1, p1, p2):        # the later plan replays first
        fresh = _sites(rng, L, chi, d)
        n0 = qb.launch_count()
        got = to_host(p(fresh))
        assert qb.launch_count() == n0
        assert_bits(got, to_host(_eager_chain(kind, fresh, m)), kind)
    _assert_plans_own_scratch(r1, r2, scratch_allocs)


def test_graphed_contractions_own_their_scratch(scratch, scratch_allocs):
    rng = np.random.default_rng(21)
    inputs, output = [("a", "b"), ("b", "c")], ("a", "c")
    A, B = randn(rng, (384, 384)), randn(rng, (384, 4096))
    probe = torch.empty((384, 4096), dtype=torch.float64, device="cuda")
    assert route_of(A, [0, 1], B, [1, 2], probe, [0, 2])["kind"] == "dmma_streamk"
    g1, g2, r1, r2 = _build_two(scratch, lambda: qb.GraphedContraction(
        inputs, output, [A, B], optimize="greedy"))
    assert "dmma_streamk" in scratch.routes
    for g in (g2, g1, g2, g1, g1, g2):
        A2, B2 = randn(rng, (384, 384)), randn(rng, (384, 4096))
        got = to_host(g(A2, B2))
        assert_bits(got, to_host(qtree.execute(g.tree, [A2, B2])))
    _assert_plans_own_scratch(r1, r2, scratch_allocs)


def test_two_plans_replay_at_once_on_two_streams(scratch):
    """Split-K partials live in the scratch: two graphs that shared it would
    mix their partials."""
    rng = np.random.default_rng(22)
    inputs, output = [("a", "b"), ("b", "c")], ("a", "c")
    A, B = randn(rng, (256, 1024)), randn(rng, (1024, 256))
    r = route_of(A, [0, 1], B, [1, 2], torch.empty((256, 256), dtype=torch.float64,
                                                   device="cuda"), [0, 2])
    assert r["kind"] == "dmma" and r["splitk"] > 1
    g = [qb.GraphedContraction(inputs, output, [A, B], optimize="greedy") for _ in range(2)]
    L, chi, d = 6, 96, 4
    sites = _sites(rng, L, chi, d)
    p = [qb.ChainPlan(sites, kind="norm", shape="lpr") for _ in range(2)]
    assert "dmma_streamk" not in scratch.routes
    ins = [[(randn(rng, (256, 1024)), randn(rng, (1024, 256))) for _ in range(2)] for _ in range(4)]
    sts = [[_sites(rng, L, chi, d) for _ in range(2)] for _ in range(4)]
    ref = [[to_host(qtree.execute(g[0].tree, list(ins[r][k]))) for k in range(2)]
           for r in range(4)]
    ref_n = [[to_host(qb.mps_norm2(sts[r][k], "lpr")) for k in range(2)] for r in range(4)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(2)]
    outs = [[None] * 2 for _ in range(4)]
    for rd in range(4):
        for k, s in enumerate(streams):
            with torch.cuda.stream(s):
                outs[rd][k] = (g[k](*ins[rd][k]).t.clone(), p[k](sts[rd][k]).t.clone())
    torch.cuda.synchronize()
    for rd in range(4):
        for k in range(2):
            assert_bits(to_host(outs[rd][k][0]), ref[rd][k], f"tree round {rd} stream {k}")
            assert_bits(to_host(outs[rd][k][1]), ref_n[rd][k], f"norm round {rd} stream {k}")


# ----------------------------------------------------- D. host-staged MPS norm
def _host_views(sites, layout, view):
    """Host arrays of (l, p, r) ``sites`` in ``layout``: C-ordered ('c'),
    Fortran-ordered ('f') or a transposed view of reversed storage ('t')."""
    out = []
    for a in sites:
        x = np.transpose(a, ["lpr".index(c) for c in layout])
        if view == "c":
            x = np.ascontiguousarray(x)
        elif view == "f":
            x = np.asfortranarray(x)
        else:
            x = np.ascontiguousarray(x.transpose(2, 1, 0)).transpose(2, 1, 0)
        out.append(x)
    return out


def _as_kind(host, kind):
    if kind == "numpy":
        return list(host)
    if kind == "pageable":
        return [torch.from_numpy(x) for x in host]
    if kind == "pinned":
        # pinned storage, same strides as the numpy view
        out = []
        for x in host:
            base = torch.from_numpy(np.ravel(x, order="K")).pin_memory()
            order = np.argsort([-s for s in x.strides], kind="stable")
            shp = [x.shape[i] for i in order]
            t = base.view(shp).permute(*np.argsort(order).tolist())
            assert t.is_pinned() and np.array_equal(t.numpy(), x)
            out.append(t)
        return out
    # mixed: even sites on the device, odd sites on the host
    return [dev(x) if i % 2 == 0 else x for i, x in enumerate(host)]


def _device_copies(host):
    """What the staging ring holds: contiguous device copies."""
    return [dev(np.asarray(x)) if not isinstance(x, torch.Tensor) or x.device.type == "cpu"
            else x for x in host]


def _oracle_tol(dtype):
    # single precision rounds every intermediate environment to float32
    return 1e-12 if dtype in ("float64", "complex128") else 2e-5


@pytest.mark.parametrize("L", [1, 2, 3, 4, 5, 9])
@pytest.mark.parametrize("dtype", ["float64", "complex128", "float32", "complex64"])
def test_host_staged_norm_equals_device_norm(dtype, L):
    sites = dm.mps_rand(L, 6, phys_dim=3, seed=30 + L, dtype=dtype)
    exact = dm.mps_norm2([a.astype(np.complex128 if "complex" in dtype else np.float64)
                          for a in sites])
    side = torch.cuda.Stream()
    for layout in ("lrp", "lpr"):
        for view in ("c", "f", "t"):
            host = _host_views(sites, layout, view)
            ref = to_host(qb.mps_norm2(_device_copies(host), layout))
            assert abs(ref - exact) <= _oracle_tol(dtype) * abs(exact), (layout, view)
            for kind in ("numpy", "pageable", "pinned", "mixed"):
                for cs in (side, None):
                    got = to_host(qb.mps_norm2(_as_kind(host, kind), layout, copy_stream=cs))
                    assert_bits(got, ref, f"{layout}/{view}/{kind}/{cs is None}")


def test_staging_ring_reuse_across_sizes_and_dtypes():
    side = torch.cuda.Stream()
    for i, (chi, dt) in enumerate([(4, "float64"), (24, "complex128"), (8, "float64"),
                                   (32, "float32"), (2, "complex128"), (16, "float64"),
                                   (32, "complex64"), (6, "float64")]):
        host = [torch.from_numpy(a).pin_memory()
                for a in dm.mps_rand(7, chi, seed=40 + i, dtype=dt)]
        ref = to_host(qb.mps_norm2(_device_copies(host), "lpr"))
        for cs in (side, None):
            assert_bits(to_host(qb.mps_norm2(host, "lpr", copy_stream=cs)), ref, (chi, dt))


def test_staging_waits_for_a_delayed_consumer():
    """The main stream sleeps before every site, so the copy stream runs ahead
    and must wait until a ring slot's consumer has passed it."""
    host = [torch.from_numpy(a).pin_memory() for a in dm.mps_rand(12, 64, seed=41)]
    ref = to_host(qb.mps_norm2(_device_copies(host), "lpr"))
    torch.cuda.synchronize()
    torch.cuda._sleep(SLEEP_CYCLES)
    got = to_host(qb.mps_norm2(host, "lpr"))
    assert_bits(got, ref, "main delayed before the call")
    E = None
    for i, s in enumerate(qmps.stream_sites(host, torch.cuda.Stream())):
        torch.cuda._sleep(SLEEP_CYCLES // 20)
        A = qmps.site_lpr(s, "lpr", i, len(host))
        E = ops.eye(A.shape[0], dtype=A.dtype, device=A.device) if E is None else E
        E = qmps.norm_step(E, A)
    assert_bits(to_host(E.reshape(())), ref, "main delayed at every site")


def test_norm_after_a_staged_call_that_raised():
    """A call that fails midway abandons copies into the shared ring; the next
    call must still be exact.  The failed call's copy stream is held back by a
    sleep (~40 ms), and the next call spends its first ~90 ms on a large
    device site before it reads its first staged one."""
    rng = np.random.default_rng(42)
    chi, d = 4096, 16
    gen = torch.Generator(device="cuda").manual_seed(42)
    big = torch.randn((chi, d, chi), dtype=torch.float64, device="cuda", generator=gen) / chi
    good = np.ascontiguousarray(rng.standard_normal((chi, d, 1)))
    junk = [torch.from_numpy(np.full((chi, d, 1), 7.0)).pin_memory() for _ in range(3)]
    bad = [randn(rng, (1, d, chi)), randn(rng, (chi, d))] + junk   # site 1: wrong rank
    ref = to_host(qb.mps_norm2([big, dev(good)], "lpr"))
    host = [big, torch.from_numpy(good).pin_memory()]
    qb.mps_norm2(host, "lpr")                 # ring and pinned buffers exist before the race
    slow = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(slow):
        torch.cuda._sleep(SLEEP_CYCLES * 4 // 5)
    with pytest.raises(ValueError, match="site 1"):
        qb.mps_norm2(bad, "lpr", copy_stream=slow)
    got = to_host(qb.mps_norm2(host, "lpr"))
    assert_bits(got, ref, "first call after the failure")
    assert_bits(to_host(qb.mps_norm2(host, "lpr")), ref, "second call after the failure")
