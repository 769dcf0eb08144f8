"""Function surface of the ``quimb_b200`` array backend (what
``autoray.do(name, ..., like="quimb_b200")`` resolves to).

Hot-path functions (``tensordot``, ``einsum``, ``transpose``, ``reshape``,
``linalg.qr``, ``linalg.svd`` and the fused quimb drivers) run on the CUDA
kernels behind the C ABI.  Cold element-wise helpers forward to torch on the
wrapped tensor (torch is the container library here).
"""

import builtins
import ctypes
import numbers

import numpy as np
import torch

from . import _lib
from .array import Array, default_device, torch_dtype
from .contract import contract_pair

# this module shadows min / all / any with array versions further down
builtins_min, builtins_all, builtins_any = builtins.min, builtins.all, builtins.any


# ------------------------------------------------------------ conversion ---
def asarray(x, dtype=None, device=None):
    if isinstance(x, Array):
        return x if dtype is None else x.astype(dtype, copy=False)
    if isinstance(x, torch.Tensor):
        t = x
    else:
        xn = np.asarray(x)
        if not xn.flags.writeable:
            xn = xn.copy()          # torch cannot wrap read-only host memory
        t = torch.as_tensor(xn)
    dev = device or (t.device if t.device.type == "cuda" else default_device())
    if t.device != dev:
        if t.device.type == "cpu" and t.numel() * t.element_size() >= (1 << 20):
            t = t.pin_memory()
        t = t.to(dev, non_blocking=True)
    if dtype is not None:
        t = t.to(torch_dtype(dtype))
    return Array(t)


array = asarray


def to_numpy(x):
    return x.__array__() if isinstance(x, Array) else np.asarray(x)


def _t(x):
    return x.resolve() if isinstance(x, Array) else x


def _wrap(fn):
    def wrapped(*args, **kwargs):
        args = [_t(a) for a in args]
        kwargs = {k: _t(v) for k, v in kwargs.items()}
        if "axis" in kwargs:
            ax = kwargs.pop("axis")
            if ax is not None:
                kwargs["dim"] = ax
        out = fn(*args, **kwargs)
        if isinstance(out, torch.Tensor):
            return Array(out)
        if isinstance(out, tuple) and hasattr(out, "_fields"):
            return out[0] if not isinstance(out[0], torch.Tensor) else Array(out[0])
        return out
    return wrapped


# ------------------------------------------------------------- layout ------
def materialize(x, force=False):
    """Contiguous copy of a strided / lazily conjugated view through the
    permute kernel (this is quimb's fuse transpose-copy)."""
    if not isinstance(x, Array):
        x = asarray(x)
    t = x.t
    if not force and not x.cj and t.is_contiguous():
        return x
    _lib.require_cuda(t)
    if t.dim() > 10:
        # a general permutation of a high-rank tensor (to_dense of a 20-qubit
        # state, fuse over interleaved axes) can exceed the permute kernel's
        # mode limit: take the multi-pass route then
        from .contract import PERMUTE_MAX_MODES, permute_contiguous, permute_modes
        if permute_modes(t) > PERMUTE_MAX_MODES:
            return Array(permute_contiguous(t, list(range(t.dim())), conj=x.cj))
    out = torch.empty(t.shape, dtype=t.dtype, device=t.device)
    if t.numel():
        lib = _lib.load()
        rc = lib.qb_permute(_lib.desc(t), _lib.desc(out), int(x.cj),
                            _lib.stream_ptr())
        _lib.check(rc, "qb_permute")
    return Array(out)


def reshape(x, shape):
    if not isinstance(x, Array):
        x = asarray(x)
    if isinstance(shape, numbers.Integral):
        shape = (shape,)
    shape = tuple(int(s) for s in shape)
    try:
        return Array(x.t.view(shape), x.cj)  # free when strides allow it
    except RuntimeError:
        return Array(materialize(x).t.view(shape))


def calc_fuse_perm_and_shape(shape, axes_groups):
    """quimb/tensor/array_ops.py:95-145 (bit-exact index bookkeeping): the
    fused axes are inserted at the minimum index of any fused axis, ungrouped
    axes keep their order; ``perm`` / ``new_shape`` are None for no-ops."""
    shape = tuple(shape)
    ndim = len(shape)
    num_groups = len(axes_groups)
    ax2group = {ax: g for g, axes in enumerate(axes_groups) for ax in axes}
    position = builtins_min(g for gax in axes_groups for g in gax)
    axes_before = tuple(ax for ax in range(position)
                        if ax2group.setdefault(ax, None) is None)
    axes_after = tuple(ax for ax in range(position, ndim)
                       if ax2group.setdefault(ax, None) is None)
    perm = (*axes_before, *(ax for g in axes_groups for ax in g), *axes_after)
    new_axes = {ax: ax for ax in axes_before}
    for i, g in enumerate(axes_groups):
        for ax in g:
            new_axes[ax] = position + i
    for i, ax in enumerate(axes_after):
        new_axes[ax] = position + num_groups + i
    new_shape = [1] * (len(axes_before) + num_groups + len(axes_after))
    for i, d in enumerate(shape):
        new_shape[new_axes[i]] *= d
    if builtins_all(i == ax for i, ax in enumerate(perm)):
        perm = None
    new_shape = tuple(new_shape)
    if shape == new_shape:
        new_shape = None
    return perm, new_shape


def fuse(x, *axes_groups, backend=None):
    """quimb's ``fuse`` (array_ops.py:148-180): transpose + reshape, i.e. at
    most ONE permute-copy kernel (and none when the strides already allow the
    view)."""
    x = asarray(x)
    axes_groups = tuple(map(tuple, axes_groups))
    if not builtins_any(axes_groups):
        return x
    perm, new_shape = calc_fuse_perm_and_shape(x.shape, axes_groups)
    if perm is not None:
        x = x.transpose(*perm)
    if new_shape is not None:
        x = reshape(x, new_shape)
    return x


def unfuse(x, axis, axis_dims, backend=None):
    """array_ops.py:183-217: split one axis back into ``axis_dims`` (a view)."""
    axis_dims = tuple(axis_dims)
    if len(axis_dims) == 1:
        return x
    x = asarray(x)
    shape = x.shape
    return reshape(x, (*shape[:axis], *axis_dims, *shape[axis + 1:]))


def transpose(x, axes=None):
    if not isinstance(x, Array):
        x = asarray(x)
    return x.transpose() if axes is None else x.transpose(*axes)


def swapaxes(x, a, b):
    return x.swapaxes(a, b)


def moveaxis(x, src, dst):
    return Array(torch.movedim(x.t, src, dst), x.cj)


def conj(x):
    return x.conj() if isinstance(x, Array) else np.conj(x)


conjugate = conj


def real(x):
    return x.real


def imag(x):
    return x.imag


def shape(x):
    return tuple(x.shape)


def ndim(x):
    return x.ndim


def size(x):
    return x.size


def squeeze(x, axis=None):
    return x.squeeze(axis)


def expand_dims(x, axis):
    return Array(x.t.unsqueeze(axis), x.cj)


def ravel(x):
    return x.ravel()


def astype(x, dtype, **kw):
    return x.astype(dtype)


def copy(x):
    return x.copy()


# ---------------------------------------------------------- contraction ----
def tensordot(a, b, axes=2):
    """numpy.tensordot semantics; one kernel launch, no transposes."""
    a, b = asarray(a), asarray(b)
    if a.dtype != b.dtype:
        dt = np.result_type(a.dtype, b.dtype)
        a, b = a.astype(dt, copy=False), b.astype(dt, copy=False)
    na, nb = a.ndim, b.ndim
    if isinstance(axes, numbers.Integral):
        axa = list(range(na - axes, na))
        axb = list(range(axes))
    else:
        axa, axb = axes
        axa = [axa] if isinstance(axa, numbers.Integral) else list(axa)
        axb = [axb] if isinstance(axb, numbers.Integral) else list(axb)
    axa = [ax % na if na else ax for ax in axa]
    axb = [ax % nb if nb else ax for ax in axb]
    if len(axa) != len(axb):
        raise ValueError("shape-mismatch for sum")
    for i, j in zip(axa, axb):
        if a.shape[i] != b.shape[j]:
            raise ValueError("shape-mismatch for sum")
    la = list(range(na))
    lb = [na + j for j in range(nb)]
    for i, j in zip(axa, axb):
        lb[j] = la[i]
    lc = [l for i, l in enumerate(la) if i not in axa] + [
        l for j, l in enumerate(lb) if j not in axb
    ]
    out = contract_pair(a.t, la, b.t, lb, lc, conj_a=a.cj, conj_b=b.cj)
    return Array(out)


def matmul(a, b):
    a, b = asarray(a), asarray(b)
    if a.ndim <= 2 and b.ndim <= 2:
        if a.ndim == 0 or b.ndim == 0:
            raise ValueError("matmul: scalar operands")
        return tensordot(a, b, axes=((a.ndim - 1,), (0,)))
    # broadcast batched matmul via einsum labels (numpy.matmul semantics:
    # 1-d operands are promoted, size-1 batch dims broadcast)
    if a.dtype != b.dtype:
        dt = np.result_type(a.dtype, b.dtype)
        a, b = a.astype(dt, copy=False), b.astype(dt, copy=False)
    vec_a, vec_b = a.ndim == 1, b.ndim == 1
    if vec_a:
        a = expand_dims(a, 0)
    if vec_b:
        b = expand_dims(b, b.ndim)
    nb = builtins.max(a.ndim, b.ndim) - 2
    la = list(range(nb - (a.ndim - 2), nb)) + [100, 101]
    lb = list(range(nb - (b.ndim - 2), nb)) + [101, 102]
    lc = list(range(nb)) + [100, 102]
    # a size-1 batch dim facing a larger one is summed over (extent 1) under a
    # private label instead of being a batch label: that is the broadcast
    fresh = 200
    for pos in range(nb):
        ia, ib = pos - (nb - (a.ndim - 2)), pos - (nb - (b.ndim - 2))
        sa = a.shape[ia] if ia >= 0 else None
        sb = b.shape[ib] if ib >= 0 else None
        if sa is not None and sb is not None and sa != sb:
            if sa == 1:
                la[ia] = fresh
            elif sb == 1:
                lb[ib] = fresh
            else:
                raise ValueError(f"matmul: batch dims {sa} and {sb} do not broadcast")
            fresh += 1
    out = Array(contract_pair(a.t, la, b.t, lb, lc, conj_a=a.cj, conj_b=b.cj))
    if vec_a:
        out = out.squeeze(out.ndim - 2)
    if vec_b:
        out = out.squeeze(out.ndim - 1)
    return out


def dot(a, b):
    return matmul(a, b)


def _parse_einsum(eq, nops):
    eq = eq.replace(" ", "")
    if "..." in eq:
        raise NotImplementedError("einsum ellipsis is not supported")
    if "->" in eq:
        lhs, rhs = eq.split("->")
    else:
        lhs = eq
        counts = {}
        for c in lhs.replace(",", ""):
            counts[c] = counts.get(c, 0) + 1
        rhs = "".join(sorted(c for c, n in counts.items() if n == 1))
    terms = lhs.split(",")
    if len(terms) != nops:
        raise ValueError("einsum: operand count does not match equation")
    return terms, rhs


def einsum(eq, *operands):
    """einsum for any number of operands: unary/pairwise cases are one kernel
    launch (batch, summed and diagonal indices included); more operands go
    through the tree executor."""
    ops = [asarray(o) for o in operands]
    terms, rhs = _parse_einsum(eq, len(ops))
    sym = {}
    for c in "".join(terms) + rhs:
        sym.setdefault(c, len(sym))
    if len(ops) == 1:
        x = ops[0]
        one = Array(torch.ones((), dtype=x.t.dtype, device=x.t.device))
        out = contract_pair(x.t, [sym[c] for c in terms[0]], one.t, [],
                            [sym[c] for c in rhs], conj_a=x.cj)
        return Array(out)
    if len(ops) == 2:
        a, b = ops
        if a.dtype != b.dtype:
            dt = np.result_type(a.dtype, b.dtype)
            a, b = a.astype(dt, copy=False), b.astype(dt, copy=False)
        out = contract_pair(a.t, [sym[c] for c in terms[0]], b.t,
                            [sym[c] for c in terms[1]], [sym[c] for c in rhs],
                            conj_a=a.cj, conj_b=b.cj)
        return Array(out)
    from .tree import array_contract
    return array_contract(ops, [tuple(t) for t in terms], tuple(rhs))


def trace(x, axis1=0, axis2=1):
    x = asarray(x)
    lab = list(range(x.ndim))
    lab[axis2] = lab[axis1]
    out_l = [l for i, l in enumerate(lab) if i not in (axis1, axis2)]
    one = torch.ones((), dtype=x.t.dtype, device=x.t.device)
    return Array(contract_pair(x.t, lab, one, [], out_l, conj_a=x.cj))


def diagonal(x, offset=0, axis1=0, axis2=1):
    return Array(torch.diagonal(x.resolve(), offset, axis1, axis2))


def diag(x, k=0):
    return Array(torch.diag(x.resolve(), k))


# ------------------------------------------------- element-wise / reductions
sqrt = _wrap(torch.sqrt)
exp = _wrap(torch.exp)
log = _wrap(torch.log)
log2 = _wrap(torch.log2)
log10 = _wrap(torch.log10)
sin = _wrap(torch.sin)
cos = _wrap(torch.cos)
tanh = _wrap(torch.tanh)
sign = _wrap(torch.sgn)
count_nonzero = _wrap(torch.count_nonzero)
where = _wrap(torch.where)
clip = _wrap(torch.clamp)
isfinite = _wrap(torch.isfinite)
isnan = _wrap(torch.isnan)
argmax = _wrap(torch.argmax)
argmin = _wrap(torch.argmin)
kron = _wrap(torch.kron)
equal = _wrap(torch.eq)
power = _wrap(torch.pow)
multiply = _wrap(torch.mul)
add = _wrap(torch.add)
subtract = _wrap(torch.sub)
divide = _wrap(torch.div)


def abs(x):  # noqa: A001
    return Array(torch.abs(x.t)) if isinstance(x, Array) else np.abs(x)


absolute = abs


def _reduce(x, axis, keepdims, full, along):
    t = _t(asarray(x))
    if axis is None:
        out = full(t)
        if keepdims:
            out = out.reshape((1,) * t.ndim)
        return Array(out)
    return Array(along(t, axis, bool(keepdims)))


def sum(x, axis=None, keepdims=False, **kw):  # noqa: A001
    return _reduce(x, axis, keepdims, lambda t: t.sum(),
                   lambda t, ax, kd: t.sum(dim=ax, keepdim=kd))


def max(x, axis=None, keepdims=False):  # noqa: A001
    return _reduce(x, axis, keepdims, lambda t: t.max(),
                   lambda t, ax, kd: t.amax(dim=ax, keepdim=kd))


def min(x, axis=None, keepdims=False):  # noqa: A001
    return _reduce(x, axis, keepdims, lambda t: t.min(),
                   lambda t, ax, kd: t.amin(dim=ax, keepdim=kd))


def mean(x, axis=None, keepdims=False):
    return _reduce(x, axis, keepdims, lambda t: t.mean(),
                   lambda t, ax, kd: t.mean(dim=ax, keepdim=kd))


def all(x):  # noqa: A001
    return bool(_t(x).all().item())


def any(x):  # noqa: A001
    return bool(_t(x).any().item())


def allclose(a, b, rtol=1e-5, atol=1e-8):
    a, b = _t(asarray(a)), _t(asarray(b))
    return bool(torch.allclose(a, b.to(a.dtype), rtol=rtol, atol=atol))


def stack(arrays, axis=0):
    return Array(torch.stack([_t(asarray(a)) for a in arrays], dim=axis))


def concatenate(arrays, axis=0):
    return Array(torch.cat([_t(asarray(a)) for a in arrays], dim=axis))


def pad(x, pad_width, mode="constant", constant_values=0):
    flat = []
    for lo, hi in reversed(list(pad_width)):
        flat += [lo, hi]
    return Array(torch.nn.functional.pad(_t(x), flat, value=constant_values))


def zeros(shape, dtype="float64", device=None):
    return Array(torch.zeros(shape, dtype=torch_dtype(dtype),
                             device=device or default_device()))


def ones(shape, dtype="float64", device=None):
    return Array(torch.ones(shape, dtype=torch_dtype(dtype),
                            device=device or default_device()))


def empty(shape, dtype="float64", device=None):
    return Array(torch.empty(shape, dtype=torch_dtype(dtype),
                             device=device or default_device()))


def eye(n, m=None, dtype="float64", device=None):
    return Array(torch.eye(n, m if m is not None else n,
                           dtype=torch_dtype(dtype),
                           device=device or default_device()))


def arange(*args, dtype="int64", device=None):
    return Array(torch.arange(*args, dtype=torch_dtype(dtype),
                              device=device or default_device()))


def zeros_like(x):
    return Array(torch.zeros_like(x.t))


def ones_like(x):
    return Array(torch.ones_like(x.t))


# ---------------------------------------------- Lanczos vector algebra -----
_DOT_WS = {}


def _dot_ws(dev):
    """Stage-1 partials of ``qb_dot``, one buffer per (device, stream): dot
    products running on two streams at once must not share them."""
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
    ws = _DOT_WS.get(key)
    if ws is None:
        n = _lib.load().qb_dot_workspace(0)
        ws = torch.empty(n, dtype=torch.uint8, device=dev)
        _DOT_WS[key] = ws
    return ws


def vdot(x, y):
    """<x|y> = sum conj(x) * y as a 0-d device Array (deterministic)."""
    x, y = materialize(asarray(x)), materialize(asarray(y))
    lib = _lib.load()
    out = torch.empty((), dtype=x.t.dtype, device=x.t.device)
    rc = lib.qb_dot(_lib.qb_dtype(x.t.dtype), x.t.numel(), x.t.data_ptr(),
                    y.t.data_ptr(), out.data_ptr(), _dot_ws(x.t.device).data_ptr(),
                    _lib.stream_ptr())
    _lib.check(rc, "qb_dot")
    return Array(out)


def axpby(alpha, x, beta, y):
    """y <- alpha * x + beta * y in place (contiguous); returns y."""
    lib = _lib.load()
    a = (ctypes.c_double * 2)(complex(alpha).real, complex(alpha).imag)
    b = (ctypes.c_double * 2)(complex(beta).real, complex(beta).imag)
    if not (x.t.is_contiguous() and y.t.is_contiguous()) or x.cj or y.cj:
        raise ValueError("axpby needs contiguous, resolved operands")
    rc = lib.qb_axpby(_lib.qb_dtype(x.t.dtype), x.t.numel(), a, x.t.data_ptr(),
                      b, y.t.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "qb_axpby")
    return y


def scale_(x, alpha=1.0, div_by=None):
    """x <- x * alpha / div_by (div_by: 0-d real device Array) in place."""
    lib = _lib.load()
    a = (ctypes.c_double * 2)(complex(alpha).real, complex(alpha).imag)
    if not x.t.is_contiguous() or x.cj:
        raise ValueError("scale_ needs a contiguous, resolved operand")
    dptr = None if div_by is None else ctypes.c_void_p(div_by.t.data_ptr())
    rc = lib.qb_scale(_lib.qb_dtype(x.t.dtype), x.t.numel(), a, dptr,
                      x.t.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "qb_scale")
    return x


def scale_into(y, x, alpha=1.0, div_by=None):
    """y <- x * alpha / div_by (contiguous, same dtype / size; real factor);
    returns y."""
    lib = _lib.load()
    if not (x.t.is_contiguous() and y.t.is_contiguous()) or x.cj or y.cj:
        raise ValueError("scale_into needs contiguous, resolved operands")
    if x.t.numel() != y.t.numel() or x.t.dtype != y.t.dtype:
        raise ValueError("scale_into: size / dtype mismatch")
    dptr = None if div_by is None else ctypes.c_void_p(div_by.t.data_ptr())
    rc = lib.qb_scale_into(_lib.qb_dtype(x.t.dtype), x.t.numel(), float(alpha), dptr,
                           x.t.data_ptr(), y.t.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "qb_scale_into")
    return y


# --------------------------------- remaining names of the backend surface ---
# (SURVEY 8(b): cold helpers quimb's drivers reach through ``do``; they
# forward to torch on the wrapped tensor like the element-wise block above)
log2 = _wrap(torch.log2)
log10 = _wrap(torch.log10)
argsort = _wrap(torch.argsort)


def sort(x, axis=-1):
    return Array(torch.sort(_t(asarray(x)), dim=axis).values)


outer = _wrap(torch.outer)


def dag(x):
    """conjugate transpose of the last two axes (lazy flag + view)."""
    x = asarray(x)
    return swapaxes(conj(x), x.ndim - 2, x.ndim - 1)


def identity(n, dtype="float64", device=None):
    return eye(n, dtype=dtype, device=device)


def full(shape, fill_value, dtype=None, device=None):
    if dtype is None:
        dtype = "complex128" if isinstance(fill_value, complex) else "float64"
    if isinstance(shape, numbers.Integral):
        shape = (shape,)
    return Array(torch.full(tuple(shape), fill_value, dtype=torch_dtype(dtype),
                            device=device or default_device()))


def indices(dimensions, dtype="int64", device=None):
    """numpy.indices: grid index arrays, shape (len(dimensions), *dimensions)."""
    dev = device or default_device()
    grids = torch.meshgrid(*[torch.arange(int(d), dtype=torch_dtype(dtype), device=dev)
                             for d in dimensions], indexing="ij")
    if not grids:
        return Array(torch.empty((0,), dtype=torch_dtype(dtype), device=dev))
    return Array(torch.stack(grids, dim=0))


def finfo(dtype):
    """numpy.finfo of a dtype given as a name, a numpy / torch dtype or an
    Array (quimb's safe_inverse / diag shifts ask the backend for eps)."""
    if isinstance(dtype, Array):
        dtype = dtype.dtype
    if isinstance(dtype, torch.dtype):
        dtype = str(dtype).replace("torch.", "")
    return np.finfo(np.dtype(dtype))


def multiply_diagonal(x, v, axis, backend=None):
    """x with the vector v multiplied in along ``axis`` as if contracting with
    diag(v) (quimb/tensor/array_ops.py:226-231)."""
    x = asarray(x)
    shape = tuple(-1 if i == axis % x.ndim else 1 for i in range(x.ndim))
    return x * reshape(asarray(v), shape)


def align_axes(*arrays, axes, backend=None):
    """dense arrays need no sector alignment (array_ops.py:234-243)."""
    return arrays


def norm_fro(x):
    """Frobenius norm through the deterministic dot kernel (array_ops.py:255-262)."""
    from .linalg import norm
    return norm(x)


# ---- numpy-signature versions of helpers whose torch signature differs ------
def take(x, indices, axis=None):
    """numpy.take: an integer index drops the axis, a sequence keeps it."""
    t = _t(asarray(x))
    if axis is None:
        t, axis = t.reshape(-1), 0
    if isinstance(indices, numbers.Integral):
        return Array(t.select(axis, int(indices)))
    idx = _t(indices) if isinstance(indices, Array) else torch.as_tensor(
        np.asarray(indices), device=t.device)
    idx = idx.to(torch.int64)
    out = t.index_select(axis, idx.reshape(-1))
    if idx.ndim != 1:
        shape = list(t.shape)
        out = out.reshape(shape[:axis] + list(idx.shape) + shape[axis + 1:])
    return Array(out)


def flip(x, axis=None):
    t = _t(asarray(x))
    if axis is None:
        dims = tuple(range(t.ndim))
    elif isinstance(axis, numbers.Integral):
        dims = (int(axis),)
    else:
        dims = tuple(int(a) for a in axis)
    return Array(torch.flip(t, dims))


def cumsum(x, axis=None):
    t = _t(asarray(x))
    if axis is None:
        t, axis = t.reshape(-1), 0
    return Array(torch.cumsum(t, dim=axis))


def tril(x, k=0):
    return Array(torch.tril(_t(asarray(x)), diagonal=k))


def triu(x, k=0):
    return Array(torch.triu(_t(asarray(x)), diagonal=k))


def prod(x, axis=None, keepdims=False):
    return _reduce(x, axis, keepdims, lambda t: t.prod(),
                   lambda t, ax, kd: t.prod(dim=ax, keepdim=kd))
