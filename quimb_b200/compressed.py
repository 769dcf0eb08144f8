"""Compressed contraction along a given contraction sequence on the device:
the array-level mirror of ``TensorNetwork._contract_compressed_tid_sequence``
(quimb/tensor/tensor_core.py:8429-8718) behind ``contract_compressed``
(:8839-9080), SURVEY.md 8(f) rank 3.

What is mirrored is the reference's control flow for ``compress_mode='basic'``
with ``tree_gauge_distance=0`` (no tree gauging): for every step
``(tid1, tid2)`` of the sequence

  * ``compress_late=True`` (default): first look at the neighbours of both
    tensors -- fuse accumulated multibonds, squeeze size-1 bonds
    (``tensor_fuse_squeeze`` :1241-1265) and, where a (fused) bond exceeds
    ``max_bond``, compress it (``_compress_between_tids`` :6667-6762 incl. the
    QR-only shortcut for ``cutoff == 0``; ``tensor_compress_bond`` :864-1094),
    skipping pairs that the sequence contracts anyway (``compress_span``),
    pairs of effective matrices (``compress_matrices``), small results
    (``compress_min_size``) and excluded tensors;
  * contract the pair, the new tensor taking the place of ``tid2``
    (``_contract_between_tids`` :6206-6243); output indices of the step are
    the ones that appear elsewhere in the network or in ``output_inds``;
  * ``compress_late=False``: compress the new tensor with its neighbours
    instead.

Every contraction is one launch of the pairwise kernel, every compression the
QR / truncated-SVD kernels (``quimb_b200.split.tensor_compress_bond``); the
network bookkeeping (which tensors share which index) is host Python over
index names, exactly the information quimb keeps in ``ind_map``.

The virtual-tree / full-bond / local-fit compression modes and simple-update
gauges of the reference are TN-level algorithms on top of the same primitives;
quimb's own implementation of them runs on this backend unchanged (DESIGN 1),
they are not duplicated here and raise ``NotImplementedError``.
"""

import math

from . import ops
from .array import Array
from .boundary import LTensor, _contract, compress_between, make_single_bond


class _Network:
    """tid -> labelled tensor, plus the index -> tids map quimb keeps."""

    def __init__(self, arrays, inputs):
        self.t = {}
        for tid, (a, inds) in enumerate(zip(arrays, inputs)):
            self.t[tid] = LTensor(ops.asarray(a), tuple(inds))
        self.exponent = 0.0

    def ind_map(self):
        m = {}
        for tid, t in self.t.items():
            for ix in t.inds:
                m.setdefault(ix, []).append(tid)
        return m

    def neighbors(self, tid):
        """tids sharing an index with ``tid``, in first-appearance order
        (``_get_neighbor_tids`` :5012-5040)."""
        mine = self.t[tid].inds
        out = []
        for ix in mine:
            for other, t in self.t.items():
                if other != tid and ix in t.inds and other not in out:
                    out.append(other)
        return out

    def bonds_size(self, a, b):
        ta, tb = self.t[a], self.t[b]
        n = 1
        for ix in ta.inds:
            if ix in tb.inds:
                n *= ta.ind_size(ix)
        return n

    def strip_exponent(self, tid, value):
        """Rescale tensor ``tid`` to Frobenius norm ``value`` (True: 1.0),
        accumulating log10 of the factor (``TensorNetwork.strip_exponent``,
        tensor_core.py:10809-10841).  The norm sets the scale the next
        compression's absolute cutoffs see, so it must be the reference's.
        A zero or non-finite norm leaves the tensor as it is (DESIGN 4.7)."""
        t = self.t[tid]
        target = 1.0 if value is True else float(value)
        nrm = _norm(t.data)
        if nrm == 0.0 or not math.isfinite(nrm):
            return
        f = nrm / target
        t.data = t.data / f
        self.exponent += math.log10(f)


def _norm(data):
    return float(ops.norm_fro(data).item()) if data.size else 0.0


def _fuse_squeeze(net, a, b):
    ta, tb = net.t[a], net.t[b]
    _, bond, _ = make_single_bond(ta, tb)
    if bond is not None and ta.ind_size(bond) == 1:
        for t in (ta, tb):
            ax = t.inds.index(bond)
            t.data = t.data.reshape(*[s for i, s in enumerate(t.data.shape) if i != ax])
            t.inds = tuple(ix for ix in t.inds if ix != bond)
            t.left_inds = None


def path_to_sequence(path, n):
    """Linear (opt_einsum style) or SSA path -> the (tid1, tid2) sequence the
    reference walks: the result of a step lives on under the second id."""
    path = [tuple(p) for p in path]
    ssa = any(max(p) >= n - i for i, p in enumerate(path)) if path else False
    seq = []
    if ssa:
        alias = {i: i for i in range(n)}
        nxt = n
        for i, j in path:
            seq.append((alias[i], alias[j]))
            alias[nxt] = alias[j]
            nxt += 1
        return seq
    cur = list(range(n))
    for p in path:
        i, j = sorted(p)
        a, b = cur[i], cur[j]
        seq.append((a, b))
        cur.pop(j); cur.pop(i)
        cur.append(b)
    return seq


def contract_compressed(arrays, inputs, output, seq, max_bond=None, cutoff=1e-10,
                        tree_gauge_distance=0, compress_mode="basic", compress_late=True,
                        compress_min_size=None, compress_span=False, compress_matrices=True,
                        compress_exclude=None, compress_opts=None, equalize_norms="auto",
                        strip_exponent=False, gauges=None, info=None):
    """Contract the network ``(arrays, inputs) -> output`` along ``seq``,
    compressing bonds larger than ``max_bond`` on the way.

    ``seq``: steps ``(tid1, tid2[, distance])`` over the positions of
    ``arrays`` (the result of a step replaces ``tid2``); use
    :func:`path_to_sequence` for opt_einsum / cotengra paths.  ``max_bond`` and
    ``cutoff`` may be callables of the step's distance, as in the reference.
    Returns a device Array (0-d for a scalar network); with
    ``strip_exponent=True`` the pair ``(mantissa, log10 exponent)``.
    ``info`` (dict) receives ``max_bond_seen`` and ``n_compress``.
    ``equalize_norms='auto'`` (the reference's default) follows
    ``strip_exponent``: tensors are then divided by their Frobenius norm after
    every contraction and compression.
    """
    if tree_gauge_distance not in (0, None) or gauges not in (None, False):
        raise NotImplementedError(
            "quimb_b200.contract_compressed: tree gauging / simple-update gauges are "
            "TN-level algorithms of quimb (run them through quimb on this backend); "
            "the mirror covers compress_mode='basic' with tree_gauge_distance=0")
    if compress_mode not in ("basic", "auto"):
        raise NotImplementedError(f"compress_mode={compress_mode!r} is not mirrored")
    compress_opts = dict(compress_opts or {})
    compress_opts.pop("mode", None)
    if equalize_norms == "auto":
        equalize_norms = strip_exponent
    net = _Network(arrays, inputs)
    output = tuple(output)
    seq = [tuple(s) for s in seq]
    stats = {"max_bond_seen": 1, "n_compress": 0}

    if not compress_span:
        dont = {frozenset(s[:2]) for s in seq}
    else:
        compress_span = int(compress_span)
        dont = {frozenset(s[:2]) for s in seq[:compress_span]}
    chi_fn = max_bond if callable(max_bond) else (lambda d: max_bond)
    eps_fn = cutoff if callable(cutoff) else (lambda d: cutoff)

    def skip(a, b):
        if compress_exclude is not None and b in compress_exclude:
            return True
        if frozenset((a, b)) in dont:
            return True
        if (not compress_matrices) and len(net.neighbors(a)) <= 2:
            return True             # the reference tests tid1 twice (:8586-8589)
        if compress_min_size is not None:
            ta, tb = net.t[a], net.t[b]
            new = ta.data.size * tb.data.size
            for ix in ta.inds:
                if ix in tb.inds:
                    new //= ta.ind_size(ix)
            if new < compress_min_size:
                return True
        return False

    def compress_neighbors(tid, d):
        chi, eps = chi_fn(d), eps_fn(d)
        if max_bond is None and eps == 0.0:
            return
        for nb in net.neighbors(tid):
            _fuse_squeeze(net, tid, nb)
            if skip(tid, nb):
                continue
            size = net.bonds_size(tid, nb)
            stats["max_bond_seen"] = max(stats["max_bond_seen"], size)
            if chi is None or size > chi:
                compress_between(net.t[tid], net.t[nb], max_bond=chi, cutoff=eps,
                                 **compress_opts)
                stats["n_compress"] += 1
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
        ta, tb = net.t.pop(a), net.t.pop(b)
        # indices that survive the step: needed by another tensor or the output
        elsewhere = set(output)
        for t in net.t.values():
            elsewhere.update(t.inds)
        # (compute_contracted_inds :10656-10675: first-appearance order over
        # the two tensors; an index seen nowhere else and not in the output is
        # summed over, shared or not)
        keep, seen = [], set()
        for ix in ta.inds + tb.inds:
            if ix in seen:
                continue
            seen.add(ix)
            if ix in elsewhere:
                keep.append(ix)
        net.t[b] = _contract([ta, tb], output_inds=tuple(keep))
        if equalize_norms:
            net.strip_exponent(b, equalize_norms)
        if not compress_late:
            compress_neighbors(b, d)

    tensors = list(net.t.values())
    res = tensors[0] if len(tensors) == 1 else _contract(tensors, output_inds=output)
    if tuple(res.inds) != output:
        res = _contract([res], output_inds=output)
    if info is not None:
        info.update(stats)
    data = res.data
    if strip_exponent:
        # maybe_unwrap (tensor_core.py:1891-1894): mantissa of unit Frobenius norm
        nrm = _norm(data)
        if nrm > 0.0 and math.isfinite(nrm):
            data = data / nrm
            net.exponent += math.log10(nrm)
        return data, net.exponent
    if net.exponent:
        data = data * (10.0 ** net.exponent)
    return data


__all__ = ["contract_compressed", "path_to_sequence"]
