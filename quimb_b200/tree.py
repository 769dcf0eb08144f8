"""Contraction-tree executor: the host-side mirror of what cotengra does for
``quimb.tensor.contraction.array_contract`` (contraction.py:272-292) and
``array_contract_expression`` (:296-299).

A tree is a list of SSA steps ``(i, j) -> k``.  Every step is ONE launch of
the pairwise contraction kernel, with the output written directly in the
index order the next consumer wants -- so, unlike the numpy path
(tensordot + transpose per node), no standalone transpose ever runs.

External trees are accepted unchanged: anything with a ``get_path()`` method
(cotengra.ContractionTree) or an explicit opt_einsum-style linear path.
"""

import itertools
import math

from . import ops
from .array import Array
from .contract import contract_pair


# ------------------------------------------------------------- bookkeeping --
def gen_output_inds(all_inds):
    """Indices appearing exactly once in first-appearance order; an index
    appearing more than twice is an error unless output_inds is given
    (mirrors quimb/tensor/tensor_core.py:158-170)."""
    freq = {}
    for ix in all_inds:
        freq[ix] = freq.get(ix, 0) + 1
    for ix, f in freq.items():
        if f > 2:
            raise ValueError(
                f"The index {ix} appears more than twice! If this is "
                "intentionally a 'hyper' tensor network you will need to "
                "explicitly supply `output_inds` when contracting for example."
            )
    return tuple(ix for ix, f in freq.items() if f == 1)


class Tree:
    """SSA contraction tree over ``inputs`` with per-node index tuples."""

    def __init__(self, inputs, output, size_dict, ssa_steps):
        self.inputs = [tuple(t) for t in inputs]
        self.output = tuple(output)
        self.size_dict = dict(size_dict)
        self.steps = []  # (i, j, k, inds_k)
        self._build(ssa_steps)

    def _build(self, ssa_steps):
        n = len(self.inputs)
        inds = {i: t for i, t in enumerate(self.inputs)}
        alive = set(range(n))
        # appearance counts to know which indices are still needed
        nxt = n
        for i, j in ssa_steps:
            alive.discard(i)
            alive.discard(j)
            need = set(self.output)
            for a in alive:
                need.update(inds[a])
            ti, tj = inds[i], inds[j]
            res = tuple(ix for ix in dict.fromkeys(ti + tj) if ix in need)
            inds[nxt] = res
            self.steps.append((i, j, nxt, res))
            alive.add(nxt)
            nxt += 1
        if self.steps:
            # last node is produced directly in the requested output order
            i, j, k, res = self.steps[-1]
            if set(res) != set(self.output):
                raise ValueError("tree does not produce the requested output")
            self.steps[-1] = (i, j, k, self.output)
        self.node_inds = inds

    def contraction_cost(self):
        """sum over nodes of M*N*K (scalar multiply-adds), cotengra's
        ``contraction_cost`` convention."""
        inds = dict(enumerate(self.inputs))
        tot = 0
        for i, j, k, res in self.steps:
            allix = set(inds[i]) | set(inds[j])
            tot += math.prod(self.size_dict[ix] for ix in allix)
            inds[k] = res
        return tot

    def contraction_width(self):
        w = 1
        for _, _, _, res in self.steps:
            w = max(w, math.prod(self.size_dict[ix] for ix in res))
        return math.log2(w)


def find_slices(tree, target_width=None, min_slices=None, max_slices=1 << 20):
    """Choose indices to slice (fix to each of their values and sum) so that
    the largest intermediate of ``tree`` has at most ``2**target_width``
    elements and / or there are at least ``min_slices`` independent
    contractions -- the unit multi-GPU runs shard (quimb/tensor/
    tensor_core.py:255-259; the role of cotengra's SliceFinder).  Greedy: the
    index whose removal shrinks the widest intermediates most, ties broken by
    total cost.  Returns ``(sliced_inds, n_slices, width, cost_per_slice)``.
    Host-only."""
    out_set = set(tree.output)
    node_inds = dict(enumerate(tree.inputs))
    steps = []
    for i, j, k, res in tree.steps:
        steps.append((tuple(node_inds[i]), tuple(node_inds[j]), tuple(res)))
        node_inds[k] = res
    sz = dict(tree.size_dict)

    def measure(removed):
        width, cost = 1, 0
        for a, b, r in steps:
            w = math.prod(sz[ix] for ix in r if ix not in removed)
            c = math.prod(sz[ix] for ix in set(a) | set(b) if ix not in removed)
            width = max(width, w)
            cost += c
        return width, cost

    sliced, nsl = [], 1
    width, cost = measure(set())

    def done():
        ok_w = target_width is None or width <= 2 ** target_width
        ok_n = min_slices is None or nsl >= min_slices
        return ok_w and ok_n

    while not done():
        removed = set(sliced)
        # candidates: indices of the widest intermediates (or any inner index
        # when only the slice count is short)
        cands = set()
        for a, b, r in steps:
            w = math.prod(sz[ix] for ix in r if ix not in removed)
            if w == width or target_width is None or width <= 2 ** (target_width or 0):
                cands.update(ix for ix in r if ix not in removed and ix not in out_set)
        if not cands:
            for a, b, r in steps:
                cands.update(ix for ix in set(a) | set(b)
                             if ix not in removed and ix not in out_set)
        cands = {ix for ix in cands if sz[ix] > 1}
        if not cands:
            break
        best = None
        for ix in sorted(cands, key=str):
            w, c = measure(removed | {ix})
            key = (w, c * sz[ix])
            if best is None or key < best[0]:
                best = (key, ix, w, c)
        _, ix, width, cost = best
        sliced.append(ix)
        nsl *= sz[ix]
        if nsl > max_slices:
            raise ValueError(f"find_slices: more than {max_slices} slices would be "
                             "needed; use a better contraction tree")
    return tuple(sliced), nsl, math.log2(width), cost


def linear_to_ssa(path, n):
    ids = list(range(n))
    nxt = n
    ssa = []
    for con in path:
        con = sorted(con)
        if len(con) != 2:
            raise ValueError("only pairwise contraction paths are supported")
        i, j = con
        a, b = ids[i], ids[j]
        ssa.append((a, b))
        ids = [x for k, x in enumerate(ids) if k not in (i, j)] + [nxt]
        nxt += 1
    return ssa


# ---------------------------------------------------------------- finders ---
def _greedy_ssa(inputs, output, size_dict):
    """Greedy: repeatedly contract the pair sharing an index that minimises
    size(result) - size(a) - size(b) (opt_einsum's heuristic); disconnected
    components are joined by outer products at the end.  Candidates are
    generated from an index -> tensors map, so the cost per step is
    proportional to the number of neighbouring pairs, not all pairs."""
    inds = {i: tuple(t) for i, t in enumerate(inputs)}
    where = {}
    for i, t in inds.items():
        for ix in set(t):
            where.setdefault(ix, set()).add(i)
    out_set = set(output)
    sz = lambda t: math.prod(size_dict[ix] for ix in t)  # noqa: E731

    def result(a, b):
        sa, sb = set(inds[a]), set(inds[b])
        keep = []
        for ix in dict.fromkeys(inds[a] + inds[b]):
            # needed later if it is an output or lives on a third tensor
            if ix in out_set or (where[ix] - {a, b}):
                keep.append(ix)
        return tuple(keep), sa | sb

    ssa, nxt = [], len(inputs)
    while len(inds) > 1:
        cands = set()
        for ix, ts in where.items():
            if len(ts) >= 2:
                tl = sorted(ts)
                for x in range(len(tl)):
                    for y in range(x + 1, len(tl)):
                        cands.add((tl[x], tl[y]))
        best = None
        if cands:
            for a, b in cands:
                res, union = result(a, b)
                key = (sz(res) - sz(inds[a]) - sz(inds[b]),
                       math.prod(size_dict[ix] for ix in union), a, b)
                if best is None or key < best[0]:
                    best = (key, a, b, res)
        else:
            # no shared indices left: outer product of the two smallest
            ks = sorted(inds, key=lambda k: (sz(inds[k]), k))[:2]
            a, b = ks
            res, _ = result(a, b)
            best = (None, a, b, res)
        _, a, b, res = best
        ssa.append((a, b))
        for k in (a, b):
            for ix in set(inds[k]):
                where[ix].discard(k)
            del inds[k]
        inds[nxt] = res
        for ix in set(res):
            where.setdefault(ix, set()).add(nxt)
        nxt += 1
    return ssa


def _greedy_heap_ssa(inputs, output, size_dict, costmod=1.0, temperature=0.0, rng=None):
    """Heap-based greedy with optional Boltzmann (Gumbel) noise: the trial
    generator of the 'random-greedy' strategy (the approach of opt_einsum's /
    cotengra's RandomGreedy).  Pair score = size(result) - costmod * (size(a) +
    size(b)), compared on a signed-log scale with noise ``temperature``."""
    import heapq
    inds = {i: frozenset(t) for i, t in enumerate(inputs)}
    order = {i: tuple(t) for i, t in enumerate(inputs)}
    where = {}
    for i, t in inds.items():
        for ix in t:
            where.setdefault(ix, set()).add(i)
    out_set = set(output)
    log2 = math.log2

    def lsize(t):
        return sum(log2(size_dict[ix]) for ix in t)

    def result(a, b):
        keep = [ix for ix in dict.fromkeys(order[a] + order[b])
                if ix in out_set or (where[ix] - {a, b})]
        return tuple(keep)

    def score(a, b):
        res = result(a, b)
        c = 2.0 ** lsize(res) - costmod * (2.0 ** lsize(inds[a]) + 2.0 ** lsize(inds[b]))
        sc = math.copysign(math.log1p(abs(c)), c)
        if temperature > 0.0:
            u = rng.random()
            sc -= temperature * (-math.log(-math.log(u + 1e-300) + 1e-300))
        return sc

    heap = []
    seen = set()
    for ix, ts in where.items():
        tl = sorted(ts)
        for x in range(len(tl)):
            for y in range(x + 1, len(tl)):
                key = (tl[x], tl[y])
                if key not in seen:
                    seen.add(key)
                    heapq.heappush(heap, (score(*key), key[0], key[1]))
    ssa, nxt = [], len(inputs)
    while len(inds) > 1:
        a = b = None
        while heap:
            _, x, y = heapq.heappop(heap)
            if x in inds and y in inds:
                a, b = x, y
                break
        if a is None:
            # disconnected components: outer product of the two smallest
            ks = sorted(inds, key=lambda k: (lsize(inds[k]), k))[:2]
            a, b = ks
        res = result(a, b)
        ssa.append((a, b))
        for k in (a, b):
            for ix in inds[k]:
                where[ix].discard(k)
            del inds[k], order[k]
        inds[nxt], order[nxt] = frozenset(res), res
        nbrs = set()
        for ix in res:
            nbrs.update(where.setdefault(ix, set()))
            where[ix].add(nxt)
        for k in nbrs:
            if k != nxt:
                heapq.heappush(heap, (score(k, nxt), k, nxt))
        nxt += 1
    return ssa


def _random_greedy_ssa(inputs, output, size_dict, trials=32, seed=0, minimize="flops"):
    """Best of a deterministic greedy run and ``trials`` noisy ones (fixed
    seed: reproducible), judged by total cost then width."""
    import random
    rng = random.Random(seed)
    best = None
    for t in range(trials + 1):
        if t == 0:
            ssa = _greedy_heap_ssa(inputs, output, size_dict)
        else:
            costmod = math.exp(rng.uniform(math.log(0.1), math.log(4.0)))
            temp = math.exp(rng.uniform(math.log(1e-3), math.log(1.0)))
            ssa = _greedy_heap_ssa(inputs, output, size_dict, costmod, temp, rng)
        tr = Tree(inputs, output, size_dict, ssa)
        key = ((tr.contraction_cost(), tr.contraction_width()) if minimize == "flops"
               else (tr.contraction_width(), tr.contraction_cost()))
        if best is None or key < best[0]:
            best = (key, ssa)
    return best[1]


def _optimal_ssa(inputs, output, size_dict):
    """Exact minimum-flop tree by dynamic programming over subsets."""
    n = len(inputs)
    inputs = [tuple(t) for t in inputs]

    def boundary(mask):
        outside = set(output)
        for k in range(n):
            if not mask >> k & 1:
                outside.update(inputs[k])
        seen = []
        for k in range(n):
            if mask >> k & 1:
                for ix in inputs[k]:
                    if ix in outside and ix not in seen:
                        seen.append(ix)
        return tuple(seen)

    bnd = {1 << k: inputs[k] for k in range(n)}
    cost = {1 << k: (0, None) for k in range(n)}
    for r in range(2, n + 1):
        for combo in itertools.combinations(range(n), r):
            mask = 0
            for k in combo:
                mask |= 1 << k
            bnd[mask] = boundary(mask)
            best = None
            sub = (mask - 1) & mask
            while sub:
                oth = mask ^ sub
                if sub > oth:
                    fl = math.prod(size_dict[ix]
                                   for ix in set(bnd[sub]) | set(bnd[oth]))
                    c = cost[sub][0] + cost[oth][0] + fl
                    if best is None or c < best[0]:
                        best = (c, sub, oth)
                sub = (sub - 1) & mask
            cost[mask] = (best[0], (best[1], best[2]))
    ssa, ids, counter = [], {1 << k: k for k in range(n)}, [n]

    def rec(mask):
        if mask in ids:
            return ids[mask]
        a, b = cost[mask][1]
        ia, ib = rec(a), rec(b)
        ssa.append((ia, ib))
        ids[mask] = counter[0]
        counter[0] += 1
        return ids[mask]

    rec((1 << n) - 1)
    return ssa


# multiply-add equivalents charged per intermediate element by the 'combo'
# objective of the device-targeted searches: a complex128 element written and
# read back costs 2 x 16 B / (HBM bytes/s) against 8 flop / (fp64 flop/s) per
# multiply-add; 16 is that ratio rounded for an HBM-bandwidth to fp64-rate
# ratio like the H100 data sheet's (3.35 TB/s, 67 TFLOP/s)
DEVICE_COMBO = ("combo", 16.0)


def _hq_candidates(inputs, output, size_dict, trials=64, subtree_size=8, minimize="flops"):
    """Refined candidate trees over the rank-simplified network: noisy greedy
    (good for shallow / tree-like networks) and the spectral sweep (good for
    deep circuits and strips), each polished by simulated annealing over tree
    rotations and exact subtree reconfiguration.
    Yields ``(log2 cost, log2 width, ssa over the ORIGINAL inputs)``."""
    from . import treeopt
    n = len(inputs)
    prefix, red, ids = treeopt.simplify_inputs(inputs, output, size_dict)
    if len(red) < 3:
        sub = [(0, 1)] if len(red) == 2 else []
        full = treeopt.compose_ssa(prefix, n, ids, sub)
        yield treeopt.tree_stats(inputs, output, size_dict, full) + (full,)
        return
    starts = [_random_greedy_ssa(red, output, size_dict, trials=trials),
              treeopt.spectral_ssa(red, output, size_dict)]
    for k, sub in enumerate(starts):
        sub = treeopt.reconfigure(red, output, size_dict, sub, subtree_size=6, minimize=minimize)
        sub = treeopt.anneal(red, output, size_dict, sub, sweeps=300, seed=k, minimize=minimize)
        sub = treeopt.reconfigure(red, output, size_dict, sub, subtree_size=subtree_size,
                                  minimize=minimize)
        c, w = treeopt.tree_stats(red, output, size_dict, sub)
        yield c, w, treeopt.compose_ssa(prefix, n, ids, sub)


def _hq_ssa(inputs, output, size_dict):
    return min(_hq_candidates(inputs, output, size_dict), key=lambda t: t[:2])[2]


def find_sliced_tree(inputs, output, size_dict, target_width, min_slices=None,
                     optimize="auto-hq", subtree_size=8, minimize=DEVICE_COMBO):
    """Tree + sliced indices found TOGETHER for a memory target (the job of
    cotengra's ``slicing_reconf_opts``): candidates from ``optimize`` are each
    sliced index by index with the tree of the sliced network re-optimised
    after every cut, and the cheapest total (cost per slice x slices) wins.
    ``minimize`` defaults to the device-targeted objective (multiply-adds + 16 x
    intermediate elements: most big steps of a circuit tree are HBM-bound).
    Returns ``(Tree over the sliced inputs, sliced_inds)``; ``min_slices``
    (e.g. the world size) adds slices with :func:`find_slices` when the width
    target alone gives fewer.  Host-only."""
    from . import treeopt
    orig_inputs = [tuple(t) for t in inputs]
    orig_output, orig_sizes = tuple(output), size_dict
    inputs, output, size_dict, names = _canonical(orig_inputs, orig_output, size_dict)
    if optimize == "auto-hq":
        cands = [c[2] for c in _hq_candidates(inputs, output, size_dict, subtree_size=subtree_size,
                                              minimize=minimize)]
    else:
        cands = [[(i, j) for i, j, _, _ in find_tree(inputs, output, size_dict, optimize).steps]]
    best = None
    for ssa in cands:
        ssa2, sl = treeopt.slice_and_reconfigure(inputs, output, size_dict, ssa,
                                                 target_width, subtree_size=subtree_size,
                                                 minimize=minimize)
        s = set(sl)
        red = [tuple(ix for ix in t if ix not in s) for t in inputs]
        c, w = treeopt.tree_stats(red, output, size_dict, ssa2)
        sw = treeopt._size_weight(minimize)
        if sw:
            c = math.log2(2.0 ** c + sw * 2.0 ** treeopt.tree_traffic(red, output, size_dict, ssa2) / 3)
        tot = c + sum(math.log2(size_dict[ix]) for ix in sl)
        if best is None or (w > target_width, tot) < best[0]:
            best = ((w > target_width, tot), ssa2, sl, red)
    _, ssa, sl, red = best
    tr = Tree(red, output, size_dict, ssa)
    if min_slices is not None and math.prod(size_dict[ix] for ix in sl) < min_slices:
        more = find_slices(tr, None, -(-min_slices // math.prod(size_dict[ix] for ix in sl)))[0]
        sl = tuple(sl) + tuple(more)
    # back to the caller's index names
    sl = tuple(names[ix] for ix in sl)
    s = set(sl)
    red = [tuple(ix for ix in t if ix not in s) for t in orig_inputs]
    return Tree(red, orig_output, orig_sizes, ssa), sl


def _canonical(inputs, output, size_dict):
    """Index names -> integers in first-appearance order.  The finders keep
    indices in sets; with string names their iteration order depends on the
    process's hash seed, and the ranks of a multi-GPU run (which each find the
    tree and the slices for themselves) must take identical decisions."""
    table = {}
    for t in inputs:
        for ix in t:
            table.setdefault(ix, len(table))
    for ix in output:
        table.setdefault(ix, len(table))
    cin = [tuple(table[ix] for ix in t) for t in inputs]
    cout = tuple(table[ix] for ix in output)
    csz = {table[ix]: size_dict[ix] for ix in table}
    names = list(table)
    return cin, cout, csz, names


def find_tree(inputs, output, size_dict, optimize="auto"):
    n = len(inputs)
    orig = (inputs, output, size_dict)
    if isinstance(optimize, (str, type(None))) and n > 1:
        inputs, output, size_dict, _ = _canonical(inputs, output, size_dict)
    if hasattr(optimize, "get_path"):          # cotengra.ContractionTree
        ssa = linear_to_ssa(optimize.get_path(), n)
    elif isinstance(optimize, Tree):
        return optimize
    elif isinstance(optimize, (list, tuple)):  # explicit linear path
        ssa = linear_to_ssa(optimize, n)
    elif n <= 1:
        ssa = []
    elif optimize in ("optimal", "dp") or (
            optimize in ("auto", "auto-hq", "random-greedy", None) and n <= 9):
        ssa = _optimal_ssa(inputs, output, size_dict)
    elif optimize == "auto-hq":
        ssa = _hq_ssa(inputs, output, size_dict)
    elif optimize == "spectral":
        from . import treeopt
        ssa = treeopt.spectral_ssa(inputs, output, size_dict)
    elif optimize == "random-greedy":
        ssa = _random_greedy_ssa(inputs, output, size_dict, trials=32)
    elif optimize in ("auto", None):
        ssa = _random_greedy_ssa(inputs, output, size_dict, trials=8)
    elif optimize == "greedy":
        ssa = _greedy_ssa(inputs, output, size_dict)
    else:
        raise ValueError(f"unknown optimize strategy {optimize!r}")
    return Tree(orig[0], orig[1], orig[2], ssa)


# --------------------------------------------------------------- executor ---
def _labels(inds, table):
    return [table.setdefault(ix, len(table)) for ix in inds]


class _Exponent:
    """Running log10 scale of a contraction with ``strip_exponent=True``
    (quimb tensor_core.py:330-336 -> cotengra: every intermediate is divided
    by its largest magnitude and the log10 of that factor accumulated).  The
    factor never leaves the device: ``qb_scale`` divides by a device scalar,
    the exponent is read once at the end."""

    def __init__(self):
        self.total = None

    def strip(self, out, own=True):
        import torch
        # own=False: `out` aliases a caller's array -> scale a copy
        out = ops.materialize(ops.asarray(out), force=not own)
        factor = out.t.abs().amax() if out.t.numel() else None
        if factor is None:
            return out
        if factor.dtype != torch.float64:
            factor = factor.double()
        ops.scale_(out, 1.0, div_by=Array(factor))
        lg = torch.log10(factor)
        self.total = lg if self.total is None else self.total + lg
        return out

    def value(self):
        return 0.0 if self.total is None else float(self.total.item())


def execute(tree, arrays, strip_exponent=False):
    expo = _Exponent() if strip_exponent else None
    out = _execute(tree, arrays, expo)
    if expo is not None:
        return out, expo.value()
    return out


def _execute(tree, arrays, expo):
    table = {}
    nodes = {i: ops.asarray(a) for i, a in enumerate(arrays)}
    inds = dict(enumerate(tree.inputs))
    if not tree.steps:
        (x,) = nodes.values()
        t = inds[0]
        if t == tree.output:
            return x if expo is None else expo.strip(x, own=False)
        one = ops.ones((), dtype=x.dtype, device=x.device)
        res = Array(contract_pair(x.t, _labels(t, table), one.t, [],
                                  _labels(tree.output, table), conj_a=x.cj))
        return res if expo is None else expo.strip(res)
    for i, j, k, res in tree.steps:
        a, b = nodes.pop(i), nodes.pop(j)
        if a.dtype != b.dtype:
            import numpy as np
            dt = np.result_type(a.dtype, b.dtype)
            a, b = a.astype(dt, copy=False), b.astype(dt, copy=False)
        out = contract_pair(a.t, _labels(inds[i], table), b.t,
                            _labels(inds[j], table), _labels(res, table),
                            conj_a=a.cj, conj_b=b.cj)
        nodes[k] = Array(out) if expo is None else expo.strip(Array(out))
        inds[k] = res
    (out,) = nodes.values()
    return out


def _sizes(inputs, arrays):
    size_dict = {}
    for t, x in zip(inputs, arrays):
        if len(t) != len(x.shape):
            raise ValueError(f"indices {t} do not match array rank {x.shape}")
        for ix, d in zip(t, x.shape):
            if size_dict.setdefault(ix, int(d)) != int(d):
                raise ValueError(f"size mismatch on index {ix}")
    return size_dict


def array_contract(arrays, inputs, output=None, optimize="auto", strip_exponent=False):
    """Contract device arrays labelled by hashable indices.  With
    ``strip_exponent`` returns ``(mantissa, exponent)`` with the result equal
    to ``mantissa * 10**exponent`` and ``max|mantissa| == 1``."""
    arrays = [ops.asarray(a) for a in arrays]
    inputs = [tuple(t) for t in inputs]
    if output is None:
        output = gen_output_inds(itertools.chain.from_iterable(inputs))
    tree = find_tree(inputs, tuple(output), _sizes(inputs, arrays), optimize)
    return execute(tree, arrays, strip_exponent=strip_exponent)


def tensor_contract(arrays, inds, output_inds=None, optimize="auto",
                    strip_exponent=False, exponent=None):
    """Array-level mirror of ``quimb.tensor.tensor_contract``
    (tensor_core.py:224-358) for raw device arrays: returns
    ``(data, inds_out)``; the output indices are those appearing exactly once,
    in first-appearance order, unless ``output_inds`` is given.  With
    ``strip_exponent`` the data is ``(mantissa, exponent)``; a base
    ``exponent`` is added to the stripped one, or multiplies the plain result
    by ``10**exponent`` (tensor_core.py:330-341)."""
    inds = [tuple(t) for t in inds]
    if output_inds is None:
        inds_out = gen_output_inds(itertools.chain.from_iterable(inds))
    else:
        inds_out = tuple(output_inds)
    out = array_contract(arrays, inds, inds_out, optimize=optimize,
                         strip_exponent=strip_exponent)
    if strip_exponent:
        data, e = out
        if exponent is not None:
            e = e + exponent
        return (data, e), inds_out
    if exponent is not None:
        out = ops.scale_(ops.materialize(out, force=True), 10.0 ** exponent)
    return out, inds_out


class ContractExpression:
    """Reusable contraction (quimb's ``get='expression'`` with ``constants``,
    tensor_core.py:176-193): the tree is found once, constants stay resident
    on the device."""

    def __init__(self, inputs, output, shapes, optimize="auto", constants=None):
        self.inputs = [tuple(t) for t in inputs]
        self.output = tuple(output)
        size_dict = {}
        for t, s in zip(self.inputs, shapes):
            for ix, d in zip(t, s):
                size_dict[ix] = int(d)
        self.tree = find_tree(self.inputs, self.output, size_dict, optimize)
        self.constants = {i: ops.asarray(c) for i, c in (constants or {}).items()}
        self.var_pos = [i for i in range(len(self.inputs))
                        if i not in self.constants]

    def __call__(self, *arrays):
        if len(arrays) != len(self.var_pos):
            raise ValueError("wrong number of variable arrays")
        full = [None] * len(self.inputs)
        for i, c in self.constants.items():
            full[i] = c
        for i, a in zip(self.var_pos, arrays):
            full[i] = a
        return execute(self.tree, full)


class GraphedContraction:
    """A whole contraction tree captured ONCE into a CUDA graph and replayed.

    Trees over many small tensors (circuit amplitudes, PEPS/MPS sweeps) are
    launch- and host-bound: hundreds of kernels of a few microseconds each.
    quimb/cotengra cache the *expression* per geometry
    (tests/test_tensor/test_contract.py:155-175); here the cached object is
    the captured launch sequence itself, so a repeat contraction with new
    input values costs one graph launch.  Input arrays are copied into static
    device buffers; the output buffer is reused (clone it to keep it).  The
    graph owns its scratch (``contract.capture_graph``), so plans may be
    replayed in any order and on different streams at once.
    """

    def __init__(self, inputs, output, example_arrays, optimize="auto"):
        from .contract import capture_graph
        arrays = [ops.materialize(ops.asarray(a), force=True) for a in example_arrays]
        self.inputs = [tuple(t) for t in inputs]
        self.output = tuple(output)
        self.tree = find_tree(self.inputs, self.output, _sizes(self.inputs, arrays),
                              optimize)
        self.static_in = arrays
        self.graph, self.out, self._scratch = capture_graph(
            lambda: execute(self.tree, self.static_in))
        self.n_nodes = len(self.tree.steps)

    def __call__(self, *arrays):
        if len(arrays) != len(self.static_in):
            raise ValueError("wrong number of arrays")
        for s, a in zip(self.static_in, arrays):
            a = ops.asarray(a)
            if a.shape != s.shape:
                raise ValueError("shape mismatch with the captured contraction")
            s.t.copy_(a.resolve())
        self.graph.replay()
        return self.out
