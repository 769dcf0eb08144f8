"""CPU tier: host logic of the product (planner, tree finder, option parsing)
and the C-ABI surface.  No kernels are launched here."""

import ctypes
import itertools
import json
import os
import re

import numpy as np
import pytest

import quimb_b200 as qb
from quimb_b200 import _lib, split, tree
from oracle import contract_np as cn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "quimb_b200.h")).read()
    names = set(re.findall(r"\b(qb_[a-z0-9_]+)\s*\(", header))
    assert len(names) >= 20
    missing = [n for n in sorted(names) if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.qb_abi_version() == 1


def _strides(shape):
    st, acc = [], 1
    for s in reversed(shape):
        st.append(acc)
        acc *= s
    return list(reversed(st))


@pytest.mark.parametrize("case", [
    ("ab", "bc", "ac", dict(a=37, b=45, c=29)),
    ("abcd", "cdef", "abef", dict(a=6, b=5, c=4, d=3, e=7, f=2)),
    ("acbd", "dfce", "abef", dict(a=6, b=5, c=4, d=3, e=7, f=2)),
    ("gab", "gbc", "gac", dict(g=3, a=4, b=5, c=6)),
    ("abc", "abc", "", dict(a=3, b=4, c=5)),
    ("ab", "cd", "abcd", dict(a=2, b=3, c=4, d=5)),
    ("abe", "bc", "ac", dict(a=3, b=4, c=5, e=6)),
])
def test_planner_gemm_view(case):
    ea, eb, ec, sz = case
    L = {c: i for i, c in enumerate("abcdefgh")}
    sa, sb, sc = ([sz[c] for c in e] for e in (ea, eb, ec))
    plan = qb.plan_pair(sa, _strides(sa), [L[c] for c in ea], sb, _strides(sb),
                        [L[c] for c in eb], sc, _strides(sc), [L[c] for c in ec])
    batch = [c for c in ea if c in eb and c in ec]
    m = [c for c in ea if c in ec and c not in eb]
    n = [c for c in eb if c in ec and c not in ea]
    k = [c for c in set(ea + eb) if c not in ec]
    prod = lambda cs: int(np.prod([sz[c] for c in cs])) if cs else 1  # noqa: E731
    assert plan["M"] == prod(m)
    assert plan["N"] == prod(n)
    assert plan["K"] == prod(k)
    assert plan["batch"] == prod(batch)


def test_planner_merges_contiguous_modes():
    # (a b) and (c d) are jointly contiguous everywhere -> single modes
    plan = qb.plan_pair([6, 5, 4, 3], [60, 12, 3, 1], [0, 1, 2, 3],
                        [4, 3, 7, 2], [42, 14, 2, 1], [2, 3, 4, 5],
                        [6, 5, 7, 2], [70, 14, 2, 1], [0, 1, 4, 5])
    assert (plan["n_m"], plan["n_n"], plan["n_k"]) == (1, 1, 1)
    assert plan["vecB"] == 1 and plan["vecC"] == 1


def test_planner_errors():
    with pytest.raises(ValueError):
        qb.plan_pair([3, 4], [4, 1], [0, 1], [5, 6], [6, 1], [1, 2], [3, 6], [6, 1], [0, 2])
    with pytest.raises(ValueError):  # output label in neither input
        qb.plan_pair([3], [1], [0], [3], [1], [0], [2], [1], [7])


def test_gen_output_inds_matches_reference_rule():
    assert tree.gen_output_inds("abc" "cd" "ea") == ("b", "d", "e")
    with pytest.raises(ValueError) as e:
        tree.gen_output_inds(list("ab") + list("bc") + list("bd"))
    meta = json.load(open(os.path.join(ROOT, "tests", "golden", "contract.json")))
    assert str(e.value) == meta["_triple_index_error"]


def test_tree_finder_cost_not_worse_than_oracle():
    rng = np.random.default_rng(0)
    for trial in range(20):
        n = rng.integers(3, 7)
        letters = "abcdefghij"
        sizes = {c: int(rng.integers(2, 6)) for c in letters}
        inputs = []
        for _ in range(n):
            r = rng.integers(1, 4)
            inputs.append(tuple(rng.choice(list(letters), size=r, replace=False)))
        flat = list(itertools.chain.from_iterable(inputs))
        if any(flat.count(c) > 2 for c in set(flat)):
            continue
        out = cn.gen_output_inds(flat)
        t = tree.find_tree(inputs, out, sizes, "optimal")
        path = cn.find_path(inputs, out, sizes, "optimal")
        fl, _ = cn.path_cost(inputs, out, sizes, path)
        assert 2 * t.contraction_cost() <= fl + 1e-9


def test_parse_split_opts_codes_match_reference():
    meta = json.load(open(os.path.join(ROOT, "tests", "golden", "decomp.json")))
    for c in meta["parse_split_opts"]:
        kw = dict(c["kw"])
        if kw.get("method", "auto") in ("auto", "svd", "qr", "lq"):
            method, opts = split.parse_split_opts(**kw)
            assert method == c["method"]
            ref = dict(c["opts"])
            for k, v in ref.items():
                assert opts[k] == v, (kw, k)


def test_svals_to_keep_c_matches_reference():
    meta = json.load(open(os.path.join(ROOT, "tests", "golden", "decomp.json")))
    s = np.array(meta["svals_to_keep"]["s"])
    for cutoff, mode, expect in meta["svals_to_keep"]["cases"]:
        n_keep, _, _ = split.svals_to_keep(s, cutoff, mode, -1, 0)
        assert n_keep == expect
    # renorm known answers (reference tests: 385 / 55 preserved)
    s = np.arange(10, 0, -1.0)
    n_keep, f, err = split.svals_to_keep(s, 1e-9, 3, 5, 2)
    assert n_keep == 5 and np.isclose(np.sum((s[:5] * f) ** 2), 385.0)
    assert np.isclose(err, np.sqrt(np.sum(s[5:] ** 2)))
    n_keep, f, _ = split.svals_to_keep(s, 1e-9, 5, 5, 1)
    assert np.isclose(np.sum(s[:5] * f), 55.0)


def test_no_cpu_fallback():
    import torch
    a = torch.zeros(3, 3, dtype=torch.float64)
    with pytest.raises(_lib.QuimbB200Error):
        qb.contract_pair(a, [0, 1], a, [1, 2], [0, 2])


def test_fuse_perm_and_shape_match_reference_rule():
    """calc_fuse_perm_and_shape is pure index bookkeeping: bit-exact against
    the oracle restatement and the documented example of array_ops.py:150-160."""
    from quimb_b200 import ops
    from oracle import decomp_np as dn
    perm, shape = ops.calc_fuse_perm_and_shape((2, 3, 4, 5, 6, 7, 8, 9, 10), ((5, 3), (7, 2, 6)))
    assert perm == (0, 1, 5, 3, 7, 2, 6, 4, 8)
    assert shape == (2, 3, 7 * 5, 9 * 4 * 8, 6, 10)
    assert ops.calc_fuse_perm_and_shape((2, 3, 4), ((0,), (1,), (2,))) == (None, None)
    assert ops.calc_fuse_perm_and_shape((2, 3, 4), ((0, 1),)) == (None, (6, 4))
    rng = np.random.default_rng(0)
    for _ in range(50):
        nd = int(rng.integers(2, 7))
        shape = tuple(int(v) for v in rng.integers(1, 5, size=nd))
        axes = list(rng.permutation(nd))
        k = int(rng.integers(1, nd + 1))
        cut = int(rng.integers(0, k + 1))
        groups = tuple(g for g in (tuple(int(a) for a in axes[:cut]),
                                   tuple(int(a) for a in axes[cut:k])) if g)
        perm, new_shape = ops.calc_fuse_perm_and_shape(shape, groups)
        operm, oshape = dn.calc_fuse_perm_and_shape(shape, groups)
        assert (tuple(range(nd)) if perm is None else perm) == operm
        assert (shape if new_shape is None else new_shape) == oshape


def test_find_slices_reduces_width_and_partitions_the_sum():
    from tests.circuit_util import random_grid_circuit_amplitude
    arrays, inputs, output, amp = random_grid_circuit_amplitude(3, 3, 8, seed=1)
    sz = {ix: 2 for t in inputs for ix in t}
    tr = tree.find_tree(inputs, output, sz, "greedy")
    w0 = tr.contraction_width()
    sl, n, w, cost = tree.find_slices(tr, target_width=w0 - 3)
    assert w <= w0 - 3 and n == 2 ** len(sl) and len(set(sl)) == len(sl)
    assert not set(sl) & set(output)
    sl8, n8, _, _ = tree.find_slices(tr, min_slices=8)
    assert n8 >= 8
    # the sliced contractions sum to the full one (numpy stand-in executor)
    import itertools as it
    total = 0.0
    for vals in it.product(*[range(2) for _ in sl]):
        fix = dict(zip(sl, vals))
        sub = [a[tuple(fix[ix] if ix in fix else slice(None) for ix in t)]
               for a, t in zip(arrays, inputs)]
        red = [tuple(ix for ix in t if ix not in fix) for t in inputs]
        total += complex(cn.array_contract(sub, red, output, "greedy"))
    assert abs(total - amp) < 1e-10
    assert tree.find_slices(tr) == ((), 1, w0, tr.contraction_cost())


def _run_tree_numpy(tr, arrays):
    """Execute a quimb_b200 Tree with the oracle's pairwise numpy contraction."""
    nodes = dict(enumerate(arrays))
    inds = dict(enumerate(tr.inputs))
    for i, j, k, res in tr.steps:
        nodes[k] = cn.contract_pair(nodes.pop(i), inds[i], nodes.pop(j), inds[j], res)
        inds[k] = res
    (out,) = nodes.values()
    return out


def test_random_greedy_finder_is_valid_and_not_worse():
    from tests.circuit_util import random_grid_circuit_amplitude, random_circuit_amplitude
    for arrays, inputs, output, amp in (random_grid_circuit_amplitude(3, 3, 8, seed=2),
                                        random_circuit_amplitude(9, 6, 4)):
        sz = {ix: 2 for t in inputs for ix in t}
        g = tree.find_tree(inputs, output, sz, "greedy")
        r = tree.find_tree(inputs, output, sz, "random-greedy")
        r2 = tree.find_tree(inputs, output, sz, "random-greedy")
        assert r.steps == r2.steps                       # fixed seed: reproducible
        assert len(r.steps) == len(arrays) - 1
        assert r.contraction_cost() <= g.contraction_cost() * 1.5
        val = complex(_run_tree_numpy(r, arrays))
        assert abs(val - amp) < 1e-10
    # larger grid: the noisy trials find a markedly cheaper tree than plain greedy
    arrays, inputs, output, _ = random_grid_circuit_amplitude(4, 4, 12, dense=False)
    sz = {ix: 2 for t in inputs for ix in t}
    g = tree.find_tree(inputs, output, sz, "greedy")
    r = tree.find_tree(inputs, output, sz, "random-greedy")
    assert r.contraction_cost() <= g.contraction_cost()
    # disconnected networks and open outputs
    ins = [("a", "b"), ("b", "c"), ("x", "y"), ("y",)]
    t = tree.find_tree(ins, ("a", "c", "x"), dict(a=2, b=3, c=4, x=5, y=6), "random-greedy")
    rng = np.random.default_rng(0)
    arrs = [rng.standard_normal((2, 3)), rng.standard_normal((3, 4)),
            rng.standard_normal((5, 6)), rng.standard_normal(6)]
    if len(ins) > 9:
        pass
    ref = np.einsum("ab,bc,xy,y->acx", *arrs)
    t = tree.Tree(ins, ("a", "c", "x"), dict(a=2, b=3, c=4, x=5, y=6),
                  tree._greedy_heap_ssa(ins, ("a", "c", "x"), dict(a=2, b=3, c=4, x=5, y=6)))
    np.testing.assert_allclose(_run_tree_numpy(t, arrs), ref, atol=1e-12)


def test_planner_randomised_signatures():
    """The C++ planner (host code of the product) on 300 random signatures:
    batch / contracted / free / summed-out labels, size-1 modes, permuted and
    padded strides.  M, N, K and batch must equal the products the einsum
    semantics define; invalid signatures must be rejected, not planned."""
    rng = np.random.default_rng(7)
    letters = list(range(12))
    n_ok = 0
    for trial in range(300):
        sizes = {l: int(rng.choice([1, 2, 3, 4, 5, 7])) for l in letters}
        ra, rb = int(rng.integers(0, 5)), int(rng.integers(0, 5))
        la = [int(x) for x in rng.choice(letters, size=ra, replace=False)]
        lb = [int(x) for x in rng.choice(letters, size=rb, replace=False)]
        cand = list(dict.fromkeys(la + lb))
        keep = [l for l in cand if rng.random() < 0.6]
        lc = [int(x) for x in rng.permutation(keep)] if keep else []

        def shape_strides(ls, pad):
            shape = [sizes[l] for l in ls]
            order = list(rng.permutation(len(ls)))        # arbitrary memory order
            st, acc = [0] * len(ls), 1
            for ax in order:
                st[ax] = acc
                acc *= shape[ax] + (pad if rng.random() < 0.3 else 0)
            return shape, st
        sa, sta = shape_strides(la, 1)
        sb, stb = shape_strides(lb, 2)
        sc, stc = shape_strides(lc, 0)
        plan = qb.plan_pair(sa, sta, la, sb, stb, lb, sc, stc, lc)
        inA, inB, inC = set(la), set(lb), set(lc)
        prod = lambda ls: int(np.prod([sizes[l] for l in ls])) if ls else 1  # noqa: E731
        batch = [l for l in cand if l in inA and l in inB and l in inC]
        m = [l for l in cand if l in inA and l not in inB and l in inC]
        n = [l for l in cand if l in inB and l not in inA and l in inC]
        k = [l for l in cand if l not in inC]
        assert plan["batch"] == prod(batch), (la, lb, lc)
        assert plan["M"] == prod(m), (la, lb, lc)
        assert plan["N"] == prod(n), (la, lb, lc)
        assert plan["K"] == prod(k), (la, lb, lc)
        n_ok += 1
    assert n_ok == 300
    # a label of C that is in neither input / mismatched extents are rejected
    with pytest.raises(ValueError):
        qb.plan_pair([2, 3], [3, 1], [0, 1], [3, 4], [4, 1], [1, 2], [2, 5], [5, 1], [0, 9])
    with pytest.raises(ValueError):
        qb.plan_pair([2, 3], [3, 1], [0, 1], [4, 4], [4, 1], [1, 2], [2, 4], [4, 1], [0, 2])


def test_planner_diagonal_and_summed_labels():
    # trace-like: A[i, i, j] B[j, k] -> C[i, k]: the repeated label is ONE mode
    plan = qb.plan_pair([4, 4, 3], [12, 3, 1], [0, 0, 1], [3, 5], [5, 1], [1, 2],
                        [4, 5], [5, 1], [0, 2])
    assert (plan["M"], plan["N"], plan["K"], plan["batch"]) == (4, 5, 3, 1)
    # full trace against a scalar operand
    plan = qb.plan_pair([6, 6], [6, 1], [0, 0], [], [], [], [], [], [])
    assert plan["M"] * plan["N"] * plan["batch"] == 1 and plan["K"] == 6
    # label only in A and not in C: summed over
    plan = qb.plan_pair([3, 7], [7, 1], [0, 1], [3, 2], [2, 1], [0, 2], [2], [1], [2])
    assert plan["K"] == 21 and plan["N"] == 2 and plan["M"] == 1
    # repeated label with different extents is an error
    with pytest.raises(ValueError):
        qb.plan_pair([4, 5], [5, 1], [0, 0], [], [], [], [4], [1], [0])


def _route(sa, la, sb, lb, sc, lc, dtype=_lib.QB_F64, engine=0):
    return qb.route_pair(sa, _strides(sa), la, sb, _strides(sb), lb, sc, _strides(sc), lc,
                         dtype, engine)


def test_route_report_engines():
    """qb_contract_pair_route: one decision for every engine."""
    r = _route([0, 4], [0, 1], [4, 3], [1, 2], [0, 3], [0, 2])
    assert r["kind"] == "empty" and r["launches"] == 0
    r = _route([3, 0], [0, 1], [0, 2], [1, 2], [3, 2], [0, 2])
    assert r["kind"] == "zero_fill" and r["launches"] == 1
    # single precision: int8 engine above its minimum, widened below it
    assert _route([128, 128], [0, 1], [128, 64], [1, 2], [128, 64], [0, 2],
                  _lib.QB_F32)["kind"] == "int8"
    assert _route([127, 128], [0, 1], [128, 64], [1, 2], [127, 64], [0, 2],
                  _lib.QB_F32)["kind"] == "widen"
    # float64: the int8 engine only on request (5 launches), streaming engine
    # for small operators only on request
    sq = ([256, 256], [0, 1], [256, 256], [1, 2], [256, 256], [0, 2])
    assert _route(*sq)["kind"] == "dmma"
    r = _route(*sq, engine=_lib.QB_ENGINE_OZAKI)
    assert r["kind"] == "int8" and r["launches"] == 5
    small = ([4096, 8], [0, 1], [8, 8], [1, 2], [4096, 8], [0, 2])
    assert _route(*small, engine=_lib.QB_ENGINE_STREAM)["kind"] == "stream"
    assert _route(*small)["kind"] == "dmma"
    # split-K launches the reduction kernel too
    r = _route([130, 4096], [0, 1], [4096, 130], [1, 2], [130, 130], [0, 2])
    assert r["kind"] == "dmma" and r["splitk"] > 1 and r["launches"] == 2
    # the K limit of the int8 engine: f K < 65536 real units
    kl = lambda K, dt: _route([128, K], [0, 1], [K, 64], [1, 2], [128, 64], [0, 2], dt,  # noqa: E731
                              _lib.QB_ENGINE_OZAKI)["kind"]
    assert kl(65535, _lib.QB_F64) == "int8" and kl(65536, _lib.QB_F64) == "dmma"
    assert kl(65535, _lib.QB_F32) == "int8" and kl(65536, _lib.QB_F32) == "widen"
    assert kl(32767, _lib.QB_C64) == "int8" and kl(32768, _lib.QB_C64) == "widen"


def test_route_pinned_for_baseline_shapes():
    """The routes of the BASELINE shapes at the H100 SXM's 132 SMs (the count
    the planner assumes without a device): a planner change shows up here."""
    chi, d, w = 1024, 2, 5
    r = _route([chi, chi], [0, 1], [chi, d, chi], [1, 2, 3], [chi, d, chi], [0, 2, 3])
    if r["sms"] != 132:
        pytest.skip(f"this device has {r['sms']} SMs; the pinned routes are for 132")
    big = dict(cfg=0, splitk=1, bk=32, sms=132, launches=1)
    # MPS norm (bench): ket step E[a, b] A[b, p, b'] -- 128 tiles fill 132 SMs
    # well enough for the classic launch
    assert r == dict(kind="dmma", streamk=0, sk_head=0, layout=2, **big)
    # bra step A[a, p, a'] T[a, p, b']: stream-K, both operands [k][row]
    r = _route([chi, d, chi], [0, 1, 2], [chi, d, chi], [0, 1, 3], [chi, chi], [2, 3])
    assert r == dict(kind="dmma_streamk", streamk=132, sk_head=4, layout=0, **big)
    # DMRG L . x (5120 x 1024 x 4096)
    r = _route([chi, w, chi], [0, 1, 2], [chi, d, d, chi], [2, 3, 4, 5], [chi, w, d, d, chi],
               [0, 1, 3, 4, 5])
    assert r == dict(kind="dmma", streamk=0, sk_head=0, layout=2, **big)
    # 4096^3
    n = 4096
    r = _route([n, n], [0, 1], [n, n], [1, 2], [n, n], [0, 2])
    assert r == dict(kind="dmma", streamk=0, sk_head=0, layout=2, **big)


def test_route_search_reaches_every_route():
    """The GPU route matrix (tests/test_gpu_routes.py) finds a grid shape for
    every route; here at the SM count the planner sees on this machine."""
    from tests import route_oracle as ro
    found = ro.search_routes()
    missing = ro.required_keys() - set(found)
    assert not missing, sorted(missing, key=str)
    assert max(ro.macs(*v[:4], k[0]) for k, v in found.items()) <= ro.MAX_MACS


def test_nonfinite_class_oracle_matches_numpy():
    """The class oracle of the route tests agrees with numpy's own
    element-by-element arithmetic (einsum without BLAS)."""
    import warnings
    from tests import route_oracle as ro
    rng = np.random.default_rng(0)
    for dt in ("float64", "complex128"):
        a, b = ro.plant_nonfinite(ro.normal_operand(rng, (9, 7), dt),
                                  ro.normal_operand(rng, (7, 6), dt))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = np.einsum("ab,bc->ac", a, b, optimize=False)
        cls = ro.nonfinite_class(a, b)
        if dt == "complex128":
            np.testing.assert_array_equal(cls[0], ro.classify(ref.real))
            np.testing.assert_array_equal(cls[1], ro.classify(ref.imag))
        else:
            np.testing.assert_array_equal(cls, ro.classify(ref))
            assert set(np.unique(cls)) == {0, 1, 2, 3}


def test_svd_trunc_and_p2p_argument_errors_without_a_device():
    """Argument checks of the new entry points run before any CUDA call."""
    import ctypes
    lib = _lib.load()
    nk, err, nn, sw = ctypes.c_int64(0), ctypes.c_double(0.0), ctypes.c_int64(0), ctypes.c_int(0)
    args = lambda dt, m, n, mode, ws, wsb: (dt, m, n, None, 0.0, mode, -1, 0, 0, None, None, None,
                                            ctypes.byref(nk), ctypes.byref(err), ctypes.byref(nn),
                                            ws, wsb, ctypes.byref(sw), None)
    assert lib.qb_svd_trunc(*args(_lib.QB_F32, 8, 4, 4, None, 0)) == -1       # f64 only
    assert "only f64" in _lib.last_error()
    assert lib.qb_svd_trunc(*args(_lib.QB_F64, 4, 8, 4, None, 0)) == -2       # m >= n
    assert lib.qb_svd_trunc(*args(_lib.QB_F64, 8, 4, 4, None, 0)) == -8       # workspace
    assert lib.qb_svd_workspace(_lib.QB_F64, 2048, 2048) > 0
    assert lib.qb_svd_workspace(_lib.QB_F64, 20000, 64) < 0                  # beyond the register panels
    assert lib.qb_p2p_block_bytes(32 << 20) >= (64 << 20) + 65536
    assert lib.qb_p2p_data_offset(32 << 20, 1) - lib.qb_p2p_data_offset(32 << 20, 0) == 32 << 20
    bufs = (ctypes.c_void_p * 2)(0, 0)
    assert lib.qb_p2p_allgather(bufs, 2, 0, None, 16, 0, 1024, 1, None, None) == -2   # null peer
    assert lib.qb_p2p_allgather(bufs, 40, 0, None, 16, 0, 1024, 1, None, None) == -1  # world > 16


def test_p2p_exchange_argument_errors_without_a_device():
    """Every malformed exchange call is refused with its own negative code
    before any CUDA call.  The pointers are dummies that are never touched, and
    nothing is launched."""
    lib = _lib.load()
    vp = ctypes.c_void_p
    peers = (vp * 17)(*([0x7f0000000000] * 17))
    x, scratch = 0x7f1000000000, 0x7f2000000000
    n0 = _lib.launch_count()

    def ag(world=2, rank=0, x=x, nbytes=256, dst_off=0, gather=1000, epoch=1, scratch=scratch,
           bufs=peers):
        return lib.qb_p2p_allgather(bufs, world, rank, vp(x), nbytes, dst_off, gather, epoch,
                                    vp(scratch), None)

    def ar(world=2, rank=0, x=x, m=24, epoch=1, scratch=scratch, bufs=peers):
        return lib.qb_p2p_allreduce_small(bufs, world, rank, vp(x), m, epoch, vp(scratch), None)

    def refused(rc, code, fragment):
        assert rc == code, (rc, code, _lib.last_error())
        assert fragment in _lib.last_error(), _lib.last_error()

    for call in (ag, ar):
        for world in (0, 17):
            refused(call(world=world), -1, "out of range")
        for rank in (-1, 2):
            refused(call(rank=rank), -1, "out of range")
        holes = (vp * 2)(0x7f0000000000, None)
        refused(call(bufs=holes), -2, "null peer buffer 1")
        refused(call(scratch=0), -3, "scratch is null")
        refused(call(epoch=0), -4, "epoch must be >= 1")
    refused(ag(x=x + 8), -5, "16-byte aligned")
    refused(ag(nbytes=264), -5, "multiple of 16")
    refused(ag(dst_off=8), -5, "16-byte aligned")
    for nbytes, dst_off in ((-16, 0), (-256, 512), (16, -16), (256, -65536)):
        refused(ag(nbytes=nbytes, dst_off=dst_off), -5, "negative")
    refused(ag(x=0, nbytes=16), -5, "null pointer")
    # the gather buffer is gather_bytes rounded up to 256: 1000 -> 1024
    refused(ag(nbytes=1040), -6, "exceeds the gather buffer")
    refused(ag(nbytes=16, dst_off=1024), -6, "exceeds the gather buffer")
    refused(ag(nbytes=512, dst_off=528), -6, "exceeds the gather buffer")
    refused(ag(nbytes=16, dst_off=(1 << 62)), -6, "exceeds the gather buffer")
    refused(ag(gather=-256, nbytes=0), -6, "exceeds the gather buffer")
    for m in (-1, 65):
        refused(ar(m=m), -5, "outside [0, 64]")
    refused(ar(x=x + 4), -5, "8-byte aligned")
    refused(ar(x=0), -5, "non-null")
    assert _lib.launch_count() == n0


def test_path_to_sequence_linear_and_ssa():
    from quimb_b200.compressed import path_to_sequence
    # linear (opt_einsum) path over 4 tensors: contract (0,1) -> appended; then (0,1) again ...
    assert path_to_sequence([(0, 1), (0, 1), (0, 1)], 4) == [(0, 1), (2, 3), (1, 3)]
    # the same tree in SSA form: ids 4, 5, 6 are the intermediates
    assert path_to_sequence([(0, 1), (2, 3), (4, 5)], 4) == [(0, 1), (2, 3), (1, 3)]


def test_bond_shard_exchange_argument():
    from quimb_b200.dist import BondShard
    s = BondShard(rank=0, world_size=1)
    assert not s.active and s.exchange_name == "none"
    assert s.slab(10) == (0, 10)
    with pytest.raises(ValueError):
        BondShard(rank=0, world_size=1, exchange="mpi")


def test_decomposition_routes_pinned_for_benchmark_shapes():
    """The DMRG split of the benchmark (a 2048 x 2048 svd_trunc, right sweep:
    absorb 'right' mirrored onto the accumulation-free left family) and the
    TSQR of the boundary configuration's (chi d D^2) x (chi D) tensors."""
    from quimb_b200 import linalg
    r = linalg.route_svd((2048, 2048), absorb=1)
    assert (r["mirror"], r["transpose"], r["qr_first"], r["absorb"]) == (True, False, None, -1)
    assert (r["npad"], r["nblk"], r["groups"], r["cluster"], r["chunk"], r["stages"]) == \
        (2048, 128, 4, 2, 64, 4)
    assert (r["epilogue"], r["graph_sweeps"], r["qr_panel_mask"], r["qr_wy_t"]) == \
        ("left", 24, 0b0001, False)
    assert linalg.route_svd((2048, 2048))["epilogue"] == "accumulate"
    q = linalg.route_qr((128 * 4 * 64, 128 * 8))          # chi = 128, d = 4, D = 8
    assert q["path"] == "tsqr" and q["tsqr_blocks"] == 2
    assert [k["shape"] for k in q["kernels"]] == [(16384, 1024), (2048, 1024)]
    assert (q["panel_mask"], q["wy_t"]) == (0b1001, True)


def test_decomposition_route_search_reaches_every_route():
    """The GPU decomposition route tests find a grid shape for every route."""
    from tests import decomp_oracle as do
    found = do.search_routes()
    missing = [k for k in do.QR_KEYS + do.SVD_KEYS if k not in found]
    assert not missing, missing
    assert found[("svd", "groups", "fallback")][3]["nblk"] == 66


def test_decomposition_oracle_is_exact():
    """The dyadic constructions are exact and orthogonal in integer
    arithmetic, and the numpy / mpmath references agree with them."""
    from tests import decomp_oracle as do
    rng = np.random.default_rng(3)
    for m, k in ((1, 1), (17, 5), (100, 48), (2049, 33)):
        X, J = do.isometry(m, k, rng)
        G = X.astype(object).T.dot(X.astype(object))          # exact integers
        assert all(G[i, j] == (4 ** J if i == j else 0) for i in range(k) for j in range(k))
    A, Q0, R0, kappa = do.qr_case(100, 40, rng)
    assert kappa <= 11 and np.array_equal(Q0 @ R0, A)
    q, r = np.linalg.qr(A)
    sg = np.sign(np.diag(r))
    do.check_qr(A, q * sg, r * sg[:, None], kappa=kappa, Q0=Q0, R0=R0)
    for kind in ("separated", "clusters", "zeros", "graded", "gap"):
        A, U0, s, V0 = do.svd_case(60, 40, kind, rng)
        assert np.array_equal((U0 * s) @ V0.T, A)
        u, ss, vh = np.linalg.svd(A, full_matrices=False)
        do.check_svd(A, u, ss, vh, s, U0, V0)
    pytest.importorskip("mpmath")
    B = rng.standard_normal((30, 20))
    np.testing.assert_allclose(do.mp_svd(B), np.linalg.svd(B, compute_uv=False), rtol=1e-13)
    r = np.linalg.qr(B)[1]
    np.testing.assert_allclose(do.mp_qr_r(B), r * np.sign(np.diag(r))[:, None], atol=1e-13)


def test_route_pins_every_stream_variant():
    """The streaming engine's compiled (KMAX, NMAX) variant in the route
    report: one shape per variant, each at a limit, and the DMMA fallback of
    shapes past a variant's reach (complex operators past 16, real past 32)."""
    from tests import route_oracle as ro
    S = ro.ENGINE_STREAM

    def rk(K, N, dt="float64"):
        r = ro.route_of("ab,bc", ro.STREAM_M, K, N, dt, S)
        return r["kind"], r.get("stream_k", 0), r.get("stream_n", 0)

    for dt in ("float64", "complex128"):
        assert rk(4, 4, dt) == ("stream", 4, 4)
        assert rk(5, 4, dt) == ("stream", 16, 4)
        assert rk(16, 1, dt) == ("stream", 16, 4)
        assert rk(4, 5, dt) == ("stream", 4, 16)
        assert rk(1, 16, dt) == ("stream", 4, 16)
        assert rk(5, 5, dt) == ("stream", 16, 16)
        assert rk(16, 16, dt) == ("stream", 16, 16)
    assert rk(17, 1) == ("stream", 32, 32)
    assert rk(32, 32) == ("stream", 32, 32)
    for K, N in ((17, 4), (4, 17), (17, 17), (32, 32)):
        assert rk(K, N, "complex128") == ("dmma", 0, 0)
    assert rk(33, 4) == ("dmma", 0, 0)
    # without the request the same shape takes DMMA and reports no variant,
    # neither in the C report's slots nor as keys of the Python dict
    r = ro.route_of("ab,bc", ro.STREAM_M, 16, 16, "float64")
    assert r["kind"] == "dmma" and "stream_k" not in r and "stream_n" not in r
    sa, sb, sc = [ro.STREAM_M, 16], [16, 16], [ro.STREAM_M, 16]
    out = (ctypes.c_int64 * 16)(*([-7] * 16))
    for eng, want in ((0, (0, 0)), (S, (16, 16))):
        rc = _lib.load().qb_contract_pair_route(
            _lib.np_desc(sa, _strides(sa), _lib.QB_F64), _lib.labels([0, 1]),
            _lib.np_desc(sb, _strides(sb), _lib.QB_F64), _lib.labels([1, 2]),
            _lib.np_desc(sc, _strides(sc), _lib.QB_F64), _lib.labels([0, 2]), eng, out)
        assert rc == 0 and (out[9], out[10]) == want


def test_stream_route_search_reaches_every_variant():
    """The streaming grid reaches all 9 variants, each at its largest
    operator, with a lower-edge shape just past the previous variant."""
    from tests import route_oracle as ro
    want = {(dt, "stream", k, n) for dt, vs in ro.STREAM_VARIANTS.items() for k, n in vs}
    assert len(want) == 9
    found = ro.stream_shapes()
    assert set(found) == want
    top = ro.search_routes()
    low = ro.stream_lower_edges()
    for key in want:
        _, _, K, N, _, _ = top[key]
        assert (K, N) == key[2:], (key, K, N)
        _, _, K, N, _, _ = low[key]
        assert max(K, N) in (1, 5, 17), (key, K, N)


def test_exact_dot_reference_is_correctly_rounded():
    """route_oracle.exact_dot against rational arithmetic: the correctly
    rounded value of sum x_i y_i for random pairs of wide dynamic range."""
    from fractions import Fraction
    from tests import route_oracle as ro
    rng = np.random.default_rng(7)
    for trial in range(300):
        n = int(rng.integers(1, 40))
        x = np.ldexp(rng.standard_normal(n), rng.integers(-60, 60, size=n))
        y = np.ldexp(rng.standard_normal(n), rng.integers(-60, 60, size=n))
        if trial % 3 == 0:                 # heavy cancellation
            y[-1] = -float(np.dot(x[:-1], y[:-1])) / x[-1]
        exact = sum(Fraction(a) * Fraction(b) for a, b in zip(x.tolist(), y.tolist()))
        got = ro.exact_dot(x, y)
        assert Fraction(got) == Fraction(float(exact)), (trial, got, float(exact))
    z = rng.standard_normal(8) + 1j * rng.standard_normal(8)
    w = rng.standard_normal(8) + 1j * rng.standard_normal(8)
    got, scale = ro.exact_vdot(z, w)
    assert abs(got - np.vdot(z, w)) <= 1e-14 * scale
