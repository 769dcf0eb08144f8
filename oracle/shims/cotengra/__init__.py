"""TEST INFRASTRUCTURE ONLY -- minimal functional stand-in for `cotengra`.

cotengra 0.8.2 (pixi.lock:1022 of the reference) owns the contraction-tree
executor of quimb's hot path but cannot be installed offline.  This shim
provides the entry points quimb calls (quimb/tensor/contraction.py:285-313)
on top of the numpy oracle in oracle/contract_np.py, so that the unmodified
reference can be run here to generate golden vectors.  Never imported by the
product package.
"""
import math
import os
import sys

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from oracle import contract_np as _cn  # noqa: E402

from . import utils  # noqa: E402,F401
from . import cotengra  # noqa: E402,F401

__version__ = "0.0.shim"


def get_symbol(i):
    if i < 26:
        return "abcdefghijklmnopqrstuvwxyz"[i]
    if i < 52:
        return "ABCDEFGHIJKLMNOPQRSTUVWXYZ"[i - 26]
    return chr(i + 140)


def get_symbol_map(inputs):
    symbol_map = {}
    c = 0
    for term in inputs:
        for ind in term:
            if ind not in symbol_map:
                symbol_map[ind] = get_symbol(c)
                c += 1
    return symbol_map


class PathOptimizer:
    pass


class ContractionTree:
    """Just enough of a tree: a linear path plus cost queries."""

    def __init__(self, inputs, output, size_dict, path):
        self.inputs = tuple(tuple(t) for t in inputs)
        self.output = tuple(output)
        self.size_dict = dict(size_dict)
        self._path = list(path)
        self.sliced_inds = {}
        self.multiplicity = 1

    def get_path(self):
        return tuple(self._path)

    def contraction_cost(self, log=None):
        fl, _ = _cn.path_cost(self.inputs, self.output, self.size_dict, self._path)
        c = fl // 2
        return math.log(c, log) if log else c

    def contraction_width(self, log=2):
        _, w = _cn.path_cost(self.inputs, self.output, self.size_dict, self._path)
        return math.log(max(w, 1), log) if log else w

    def max_size(self, log=None):
        _, w = _cn.path_cost(self.inputs, self.output, self.size_dict, self._path)
        return w

    def contract(self, arrays, backend=None, **kw):
        return _cn.array_contract(arrays, self.inputs, self.output,
                                  optimize=self._path, size_dict=self.size_dict)


class ContractionTreeCompressed(ContractionTree):
    pass


def _sizes(inputs, shapes):
    size_dict = {}
    for t, s in zip(inputs, shapes):
        for ix, d in zip(t, s):
            size_dict[ix] = int(d)
    return size_dict


def _resolve(optimize, inputs, output, size_dict):
    if isinstance(optimize, ContractionTree):
        return optimize.get_path()
    if optimize is None:
        optimize = "auto"
    if isinstance(optimize, str):
        return _cn.find_path(inputs, output, size_dict, optimize)
    return [tuple(p) for p in optimize]


def array_contract_tree(inputs, output=None, size_dict=None, shapes=None,
                        optimize="auto", **kwargs):
    inputs = tuple(tuple(t) for t in inputs)
    if size_dict is None:
        size_dict = _sizes(inputs, shapes)
    if output is None:
        output = _cn.gen_output_inds(ix for t in inputs for ix in t)
    path = _resolve(optimize, inputs, output, size_dict)
    return ContractionTree(inputs, output, size_dict, path)


def array_contract_path(inputs, output=None, size_dict=None, shapes=None,
                        optimize="auto", **kwargs):
    return array_contract_tree(inputs, output, size_dict, shapes, optimize).get_path()


def _strip(x):
    xmax = np.max(np.abs(x))
    if xmax == 0.0:
        return x, 0.0
    return x / xmax, float(np.log10(xmax))


def _all_numpy(arrays):
    return all(isinstance(a, (np.ndarray, np.generic, float, complex, int)) for a in arrays)


def _dispatched_contract(arrays, inputs, output, path, size_dict, strip_exponent=False,
                         backend=None):
    """The pairwise loop as cotengra runs it for a non-numpy backend: every
    node is ``do("tensordot")`` (+ ``do("transpose")``) when the pair is a
    pure tensordot and ``do("einsum")`` otherwise, dispatched by autoray on
    the array type (or ``backend``).  Used when the unmodified reference is
    driven with device arrays as ``Tensor._data``."""
    from autoray import do
    arrays = list(arrays)
    terms = [tuple(t) for t in inputs]
    output = tuple(output)
    expo = 0.0

    def strip(x):
        nonlocal expo
        if not strip_exponent:
            return x
        f = do("max", do("abs", x, like=backend), like=backend)
        f = float(f.item() if hasattr(f, "item") else f)
        if f == 0.0:
            return x
        expo += math.log10(f)
        return x / f

    def single(x, t):
        if t == output:
            return x
        if len(set(t)) == len(t) and set(t) == set(output):
            return do("transpose", x, tuple(t.index(ix) for ix in output), like=backend)
        sym = get_symbol_map([t])
        return do("einsum", "".join(sym[i] for i in t) + "->" + "".join(sym[i] for i in output),
                  x, like=backend)

    if len(arrays) == 1:
        res = strip(single(arrays[0], terms[0]))
        return (res, expo) if strip_exponent else res
    for i, j in path:
        need = _cn._needed_elsewhere(terms, (i, j), output)
        last = len(terms) == 2
        iout = output if last else _cn._pair_result(terms[i], terms[j], need)
        ia, ib = terms[i], terms[j]
        sa, sb, so = set(ia), set(ib), set(iout)
        pure = (len(sa) == len(ia) and len(sb) == len(ib) and not (sa & sb & so)
                and (sa - sb) <= so and (sb - sa) <= so)
        if pure:
            shared = [ix for ix in ia if ix in sb]
            res = do("tensordot", arrays[i], arrays[j],
                     axes=([ia.index(ix) for ix in shared], [ib.index(ix) for ix in shared]),
                     like=backend)
            ires = tuple(ix for ix in ia if ix not in sb) + tuple(ix for ix in ib if ix not in sa)
            if ires != tuple(iout):
                res = do("transpose", res, tuple(ires.index(ix) for ix in iout), like=backend)
        else:
            sym = get_symbol_map([ia, ib, tuple(iout)])
            eq = "{},{}->{}".format("".join(sym[x] for x in ia), "".join(sym[x] for x in ib),
                                    "".join(sym[x] for x in iout))
            res = do("einsum", eq, arrays[i], arrays[j], like=backend)
        res = strip(res)
        arrays = [x for k, x in enumerate(arrays) if k not in (i, j)] + [res]
        terms = [t for k, t in enumerate(terms) if k not in (i, j)] + [tuple(iout)]
    return (arrays[0], expo) if strip_exponent else arrays[0]


def array_contract(arrays, inputs, output=None, optimize="auto", backend=None,
                   strip_exponent=False, cache_expression=True, **kwargs):
    inputs = tuple(tuple(t) for t in inputs)
    shapes = [tuple(a.shape) if hasattr(a, "shape") else np.shape(a) for a in arrays]
    size_dict = _sizes(inputs, shapes)
    if output is None:
        output = _cn.gen_output_inds(ix for t in inputs for ix in t)
    path = _resolve(optimize, inputs, tuple(output), size_dict)
    if not _all_numpy(arrays) or backend not in (None, "numpy"):
        return _dispatched_contract(arrays, inputs, tuple(output), path, size_dict,
                                    strip_exponent, backend)
    return _cn.array_contract(arrays, inputs, tuple(output), optimize=path,
                              size_dict=size_dict, strip_exponent=strip_exponent)


def array_contract_expression(inputs, output=None, size_dict=None, shapes=None,
                              optimize="auto", constants=None, **kwargs):
    inputs = tuple(tuple(t) for t in inputs)
    if size_dict is None:
        size_dict = _sizes(inputs, shapes)
    if output is None:
        output = _cn.gen_output_inds(ix for t in inputs for ix in t)
    output = tuple(output)
    path = _resolve(optimize, inputs, output, size_dict)
    constants = dict(constants or {})
    var_pos = [i for i in range(len(inputs)) if i not in constants]

    def expr(*arrays, backend=None, **kw):
        full = [None] * len(inputs)
        for i, c in constants.items():
            full[i] = c
        for i, a in zip(var_pos, arrays):
            full[i] = a
        if not _all_numpy(full) or backend not in (None, "numpy"):
            return _dispatched_contract(full, inputs, output, path, size_dict, False, backend)
        return _cn.array_contract(full, inputs, output, optimize=path,
                                  size_dict=size_dict)

    expr.path = path
    return expr


def get_hypergraph(*a, **k):
    raise NotImplementedError("cotengra shim: hypergraph tools unavailable")


HyperGraph = None
