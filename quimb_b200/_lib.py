"""ctypes binding of ``libquimb_b200.so`` (see ``include/quimb_b200.h``).

The product path has no CPU fallback: if the shared object is missing or a
kernel is requested on a machine without a GPU, we raise.
"""

import ctypes
import os

import numpy as np
import torch

QB_MAX_RANK = 32
QB_F32, QB_F64, QB_C64, QB_C128 = 0, 1, 2, 3
QB_ENGINE_AUTO, QB_ENGINE_DMMA, QB_ENGINE_OZAKI, QB_ENGINE_STREAM = 0, 1, 2, 3
QB_ENGINE_WS_ZEROED = 0x100
QB_PLAQ_DESC_WORDS = 12

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libquimb_b200.so")

_TORCH2QB = {
    torch.float32: QB_F32,
    torch.float64: QB_F64,
    torch.complex64: QB_C64,
    torch.complex128: QB_C128,
}
_REAL_OF = {
    torch.float32: torch.float32,
    torch.float64: torch.float64,
    torch.complex64: torch.float32,
    torch.complex128: torch.float64,
}


class qb_tensor_t(ctypes.Structure):
    _fields_ = [
        ("ptr", ctypes.c_void_p),
        ("dtype", ctypes.c_int32),
        ("rank", ctypes.c_int32),
        ("shape", ctypes.c_int64 * QB_MAX_RANK),
        ("stride", ctypes.c_int64 * QB_MAX_RANK),
    ]


class QuimbB200Error(RuntimeError):
    pass


_lib = None


def load(build_if_missing=True):
    """Load (building first if necessary) the C-ABI library."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise QuimbB200Error(
                f"{LIB_PATH} is missing: run `python -m quimb_b200.csrc.build`"
            )
        from .csrc.build import build

        build()
    lib = ctypes.CDLL(LIB_PATH)
    P = ctypes.POINTER
    T = P(qb_tensor_t)
    I32P = P(ctypes.c_int32)
    vp = ctypes.c_void_p
    i64 = ctypes.c_int64
    ci = ctypes.c_int
    dblp = P(ctypes.c_double)

    def sig(name, res, args):
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args

    sig("qb_abi_version", ci, [])
    sig("qb_last_error", ctypes.c_char_p, [])
    sig("qb_launch_count", i64, [])
    sig("qb_contract_pair", ci,
        [T, I32P, T, I32P, T, I32P, ci, ci, ci, vp, ctypes.c_size_t, vp])
    sig("qb_contract_pair_ab", ci,
        [T, I32P, T, I32P, T, I32P, ci, ci, ctypes.c_double, ctypes.c_double,
         vp, ctypes.c_size_t, vp])
    sig("qb_contract_pair_workspace", i64, [T, I32P, T, I32P, T, I32P, ci])
    sig("qb_contract_pair_plan", ci, [T, I32P, T, I32P, T, I32P, P(i64)])
    sig("qb_contract_pair_route", ci, [T, I32P, T, I32P, T, I32P, ci, P(i64)])
    sig("qb_contract_pair_feed", ci, [T, I32P, T, I32P, T, I32P, P(i64)])
    sig("qb_contract_pair_schedule", ci, [T, I32P, T, I32P, T, I32P, P(i64)])
    sig("qb_contract_batched", ci,
        [T, I32P, T, I32P, T, I32P, vp, vp, vp, i64, ci, ci, vp])
    sig("qb_permute", ci, [T, T, ci, vp])
    sig("qb_axpby", ci, [ci, i64, dblp, vp, dblp, vp, vp])
    sig("qb_scale", ci, [ci, i64, dblp, vp, vp, vp])
    sig("qb_scale_into", ci, [ci, i64, ctypes.c_double, vp, vp, vp, vp])
    sig("qb_dot", ci, [ci, i64, vp, vp, vp, vp, vp])
    sig("qb_dot_workspace", i64, [i64])
    sig("qb_scale_diag", ci, [ci, i64, i64, vp, vp, ci, ci, vp])
    sig("qb_convert", ci, [ci, ci, i64, vp, vp, vp])
    sig("qb_embed_complex", ci, [i64, i64, vp, vp, vp])
    sig("qb_extract_complex", ci, [i64, i64, i64, vp, i64, vp, vp])
    sig("qb_multi_dot", ci, [ci, ci, i64, vp, i64, vp, vp, vp, vp])
    sig("qb_multi_dot_workspace", i64, [])
    sig("qb_multi_axpy", ci, [ci, ci, i64, vp, i64, vp, ctypes.c_double, vp, vp])
    sig("qb_sample_select", ci, [ci, i64, i64, i64, vp, vp, i64, vp, i64, vp, vp, vp])
    sig("qb_rdm_workspace", i64, [i64, i64, i64, i64])
    sig("qb_rdm_reduce", ci, [ci, i64, i64, i64, i64, vp, P(i64), vp, P(i64), vp, vp, i64, vp])
    sig("qb_plaquette_expec", ci, [ci, i64, P(i64), vp, vp, i64, vp, i64, vp, vp])
    sig("qb_sketch_env", ci, [ci, i64, i64, i64, i64, i64, i64, vp, P(i64), vp, P(i64), vp,
                              P(i64), vp, P(i64), vp])
    for name, res, args in (
        ("qb_qr_stab", ci, [ci, i64, i64, vp, vp, vp, ci, vp, ctypes.c_size_t, vp]),
        ("qb_qr_workspace", i64, [ci, i64, i64]),
        ("qb_qr_route", ci, [i64, i64, P(i64)]),
        ("qb_svd_route", ci, [i64, i64, ci, P(i64)]),
        ("qb_svd", ci, [ci, i64, i64, vp, vp, vp, vp, vp, ctypes.c_size_t,
                        P(ci), vp]),
        ("qb_svd_workspace", i64, [ci, i64, i64]),
        ("qb_debug_jacobi_schedule", i64, [ci, ci, I32P, i64, P(ci)]),
        ("qb_svd_trunc", ci, [ci, i64, i64, vp, ctypes.c_double, ci, i64, ci, ci, vp, vp, vp,
                              P(i64), dblp, P(i64), vp, ctypes.c_size_t, P(ci), vp]),
        ("qb_svals_to_keep", ci, [dblp, i64, ctypes.c_double, ci, i64, ci,
                                  P(i64), dblp, dblp]),
        ("qb_measure_dmma_peak", ci, [dblp, vp]),
        ("qb_p2p_block_bytes", i64, [i64]),
        ("qb_p2p_data_offset", i64, [i64, ci]),
        ("qb_p2p_alloc", ci, [i64, P(vp)]),
        ("qb_p2p_free", ci, [vp]),
        ("qb_p2p_export", ci, [vp, P(ctypes.c_ubyte)]),
        ("qb_p2p_import", ci, [P(ctypes.c_ubyte), P(vp)]),
        ("qb_p2p_unimport", ci, [vp]),
        ("qb_p2p_allgather", ci, [P(vp), ci, ci, vp, i64, i64, i64, ctypes.c_uint64, vp, vp]),
        ("qb_p2p_allreduce_small", ci, [P(vp), ci, ci, vp, ci, ctypes.c_uint64, vp, vp]),
        ("qb_debug_trace_read", ci, [vp, i64]),
        ("qb_debug_contract_stream_host", ci,
         [T, I32P, T, I32P, T, I32P, ci, ci, ctypes.c_double, ctypes.c_double]),
    ):
        if hasattr(lib, name):
            sig(name, res, args)
    if lib.qb_abi_version() != 1:
        raise QuimbB200Error("libquimb_b200.so ABI version mismatch")
    _lib = lib
    return lib


def last_error():
    return load().qb_last_error().decode()


def check(rc, what):
    if rc != 0:
        msg = last_error()
        if rc < 0:
            raise ValueError(f"{what}: invalid argument (code {rc}): {msg}")
        raise QuimbB200Error(f"{what}: failed (code {rc}): {msg}")


def launch_count():
    return int(load().qb_launch_count())


def qb_dtype(dt):
    try:
        return _TORCH2QB[dt]
    except KeyError:
        raise TypeError(f"quimb_b200 does not support dtype {dt}") from None


def require_cuda(t, what="operand"):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor, got {type(t)}")
    if t.device.type != "cuda":
        raise QuimbB200Error(
            f"{what} lives on '{t.device}': quimb_b200 has no CPU fallback, "
            "move the data to a CUDA device first"
        )


_DESC_CACHE = {}
_LABEL_CACHE = {}


def desc(t, ptr_override=None):
    """C descriptor of a (strided) torch tensor view.  Descriptors are plain
    values the library only reads, so they are memoised on (pointer, dtype,
    shape, strides): trees over many small tensors are host-bound and filling
    a 528-byte ctypes struct costs ~4 us."""
    ptr = t.data_ptr() if ptr_override is None else ptr_override
    key = (ptr, t.dtype, t.shape, t.stride())
    d = _DESC_CACHE.get(key)
    if d is not None:
        return d
    rank = t.dim()
    if rank > QB_MAX_RANK:
        raise ValueError(f"tensor rank {rank} exceeds QB_MAX_RANK")
    d = qb_tensor_t()
    d.ptr = ptr
    d.dtype = qb_dtype(t.dtype)
    d.rank = rank
    if rank:
        d.shape[:rank] = list(t.shape)
        d.stride[:rank] = list(t.stride())
    if len(_DESC_CACHE) >= 8192:
        _DESC_CACHE.clear()
    _DESC_CACHE[key] = d
    return d


def labels(seq):
    """int32 label array (memoised per label tuple)."""
    key = tuple(seq)
    arr = _LABEL_CACHE.get(key)
    if arr is None:
        arr = (ctypes.c_int32 * max(len(key), 1))(*key)
        if len(_LABEL_CACHE) >= 8192:
            _LABEL_CACHE.clear()
        _LABEL_CACHE[key] = arr
    return arr


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def np_desc(shape, strides, dtype_code, ptr=0x10000000):
    """Descriptor for host-only planner tests (no memory is touched)."""
    d = qb_tensor_t()
    d.ptr = ptr
    d.dtype = dtype_code
    d.rank = len(shape)
    for i, (s, st) in enumerate(zip(shape, strides)):
        d.shape[i] = s
        d.stride[i] = st
    return d
