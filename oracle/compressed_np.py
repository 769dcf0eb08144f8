"""ORACLE (test infrastructure, never imported by the product package).

numpy restatement of compressed contraction along a given sequence,
``TensorNetwork._contract_compressed_tid_sequence``
(quimb/tensor/tensor_core.py:8429-8718) with ``compress_mode='basic'`` and
``tree_gauge_distance=0``, for arrays labelled by index names -- the input
convention of quimb_b200/compressed.py.  The bond operations and the trace
are those of oracle/boundary_np.py; one trace record per factorisation, with
the step's pair as the bond.
"""

import math

import numpy as np

from oracle import boundary_np as bnp
from oracle import contract_np as cnp


class Network:
    """tid -> labelled tensor in ``tensor_map`` order, and the accumulated
    log10 exponent."""

    def __init__(self, arrays, inputs):
        self.t = {tid: bnp.T(np.asarray(a), inds) for tid, (a, inds) in
                  enumerate(zip(arrays, inputs))}
        self.exponent = 0.0

    def neighbors(self, tid):
        """_get_neighbor_tids (:7216-7242): the union over the tensor's
        indices of the tids on each index, in the order they joined it (which
        is tensor_map order: a contracted tensor re-joins at the end)."""
        out = []
        for ix in self.t[tid].inds:
            for other, t in self.t.items():
                if other != tid and ix in t.inds and other not in out:
                    out.append(other)
        return out

    def strip_exponent(self, tid, value=True):
        """TensorNetwork.strip_exponent (:10809-10841) without check_zero:
        divide by the Frobenius norm over ``value``, keep its log10."""
        value = 1.0 if value is True else float(value)
        t = self.t[tid]
        f = np.linalg.norm(t.data) / value
        t.modify(t.data / f)
        self.exponent += math.log10(f)


def _fuse_squeeze(ta, tb):
    """tensor_fuse_squeeze (:1241-1265)."""
    _, bond, _ = bnp.make_single_bond(ta, tb)
    if bond is not None and ta.size(bond) == 1:
        for t in (ta, tb):
            ax = t.inds.index(bond)
            t.modify(np.squeeze(t.data, axis=ax))
            t.inds = t.inds[:ax] + t.inds[ax + 1:]


def contract_compressed(arrays, inputs, output, seq, max_bond=None, cutoff=1e-10,
                        compress_late=True, compress_min_size=None, compress_span=False,
                        compress_matrices=True, compress_exclude=None, compress_opts=None,
                        equalize_norms="auto", strip_exponent=False):
    """Returns ``(value, info)``: ``value`` is the output array in ``output``
    order, or ``(mantissa, exponent)`` with ``strip_exponent``; ``info`` has
    ``max_bond_seen``, ``n_compress`` and ``trace``."""
    compress_opts = dict(compress_opts or {})
    if equalize_norms == "auto":
        equalize_norms = strip_exponent
    net = Network(arrays, inputs)
    output = tuple(output)
    seq = [tuple(s) for s in seq]
    info = {"max_bond_seen": 1, "n_compress": 0, "trace": []}
    if not compress_span:
        dont = {frozenset(s[:2]) for s in seq}
    else:
        compress_span = int(compress_span)
        dont = {frozenset(s[:2]) for s in seq[:compress_span]}
    chi_fn = max_bond if callable(max_bond) else (lambda d: max_bond)
    eps_fn = cutoff if callable(cutoff) else (lambda d: cutoff)

    def skip(a, b):
        """_should_skip_compression (:8568-8597)."""
        if compress_exclude is not None and b in compress_exclude:
            return True
        if frozenset((a, b)) in dont:
            return True
        if not compress_matrices and len(net.neighbors(a)) <= 2:
            return True
        if compress_min_size is not None:
            ta, tb = net.t[a], net.t[b]
            new = ta.data.size * tb.data.size
            for ix in bnp.group_inds(ta, tb)[1]:
                new //= ta.size(ix)
            if new < compress_min_size:
                return True
        return False

    def compress_neighbors(tid, d):
        """_compress_neighbors (:8614-8654) and _compress_between_tids."""
        chi, eps = chi_fn(d), eps_fn(d)
        if max_bond is None and eps == 0.0:
            return
        for nb in net.neighbors(tid):
            ta, tb = net.t[tid], net.t[nb]
            _fuse_squeeze(ta, tb)
            if skip(tid, nb):
                continue
            size = ta.size_of(bnp.group_inds(ta, tb)[1])
            info["max_bond_seen"] = max(info["max_bond_seen"], size)
            if chi is None or size > chi:
                bnp.compress_between(ta, tb, max_bond=chi, cutoff=eps, trace=info["trace"],
                                     label=(tid, nb), **compress_opts)
                info["n_compress"] += 1
                if equalize_norms:
                    net.strip_exponent(tid, equalize_norms)
                    net.strip_exponent(nb, equalize_norms)

    for i, step in enumerate(seq):
        a, b = step[0], step[1]
        d = step[2] if len(step) > 2 else float("inf")
        if compress_span:
            for s in seq[i + compress_span - 1:i + compress_span]:
                dont.add(frozenset(s[:2]))
        if a == b:
            continue
        if compress_late:
            compress_neighbors(a, d)
            compress_neighbors(b, d)
        # _contract_between_tids (:6206-6243), compute_contracted_inds
        # (:10656-10675): keep what another tensor or the output still needs
        ta, tb = net.t.pop(a), net.t.pop(b)
        needed = set(output)
        for t in net.t.values():
            needed.update(t.inds)
        keep = tuple(dict.fromkeys(ix for ix in ta.inds + tb.inds if ix in needed))
        net.t[b] = bnp.T(cnp.contract_pair(ta.data, ta.inds, tb.data, tb.inds, keep), keep)
        if equalize_norms:
            net.strip_exponent(b, equalize_norms)
        if not compress_late:
            compress_neighbors(b, d)

    # maybe_unwrap (:1833-1900)
    if equalize_norms is True and strip_exponent:
        for tid in net.t:
            net.strip_exponent(tid, 1.0)
    rest = list(net.t.values())
    data, _ = cnp.tensor_contract([t.data for t in rest], [t.inds for t in rest],
                                  output_inds=output)
    data = np.asarray(data)
    if strip_exponent:
        nrm = np.linalg.norm(data)
        return (data / nrm, net.exponent + math.log10(nrm)), info
    return data * 10.0 ** net.exponent, info


def greedy_sequence(arrays, inputs, output):
    """A greedy pairwise sequence over connected pairs, smallest result first
    (the one the fixtures of oracle/make_golden.py use): ``(tid1, tid2)``
    steps, the result living on under the second id."""
    sizes = {ix: d for a, t in zip(arrays, inputs) for ix, d in zip(t, np.shape(a))}
    live = {k: set(t) for k, t in enumerate(inputs)}
    seq = []
    while len(live) > 1:
        best = None
        keys = list(live)
        for x in range(len(keys)):
            for y in range(x + 1, len(keys)):
                a, b = keys[x], keys[y]
                if not (live[a] & live[b]):
                    continue
                other = set(output)
                for k, v in live.items():
                    if k not in (a, b):
                        other |= v
                res = {ix for ix in live[a] | live[b] if ix in other}
                cost = int(np.prod([sizes[ix] for ix in res])) if res else 1
                if best is None or cost < best[0]:
                    best = (cost, a, b, res)
        if best is None:                 # disconnected: outer product of the first two
            best = (0, keys[0], keys[1], live[keys[0]] | live[keys[1]])
        _, a, b, res = best
        seq.append((a, b))
        del live[a], live[b]
        live[b] = res
    return seq
