"""TEST INFRASTRUCTURE ONLY -- a host emulation of the kernel-launching entry
points of ``libquimb_b200.so`` so that the *host layer* of the product (tree
executor, split drivers, complex embedding, Lanczos, DMRG2, sharding logic)
can be exercised in the CPU tier (``-m "not gpu"``), where no CUDA device
exists.

Nothing under ``quimb_b200/`` imports this module and the product never routes
through it: without the fixture below every kernel call on a host tensor
raises (``tests/test_host_cpu.py::test_no_cpu_fallback``).  The emulator obeys
the C ABI of ``include/quimb_b200.h`` literally -- it receives the same
``qb_tensor_t`` descriptors, raw pointers, label arrays, workspaces and return
codes the CUDA library does and reads / writes the memory behind the raw
pointers (host memory here) -- so pointer, stride, label and dtype conventions
of the Python layer are checked as they are on the device.  Host-only entry
points (planner, workspace queries, truncation rule, error string) are served
by the real shared library.

Arithmetic is numpy (einsum / LAPACK); it says nothing about the CUDA kernels,
which are covered by the ``-m gpu`` tier against the oracle.
"""

import collections
import contextlib
import ctypes

import numpy as np
import torch

from quimb_b200 import _lib

_NP = {_lib.QB_F32: np.float32, _lib.QB_F64: np.float64,
       _lib.QB_C64: np.complex64, _lib.QB_C128: np.complex128}
_REAL = {_lib.QB_F32: np.float32, _lib.QB_F64: np.float64,
         _lib.QB_C64: np.float32, _lib.QB_C128: np.float64}

_HOST_ONLY = {
    "qb_abi_version", "qb_last_error", "qb_contract_pair_plan", "qb_contract_pair_route",
    "qb_contract_pair_workspace", "qb_dot_workspace", "qb_multi_dot_workspace",
    "qb_qr_workspace", "qb_svd_workspace", "qb_svals_to_keep", "qb_qr_route", "qb_svd_route",
}


def _addr(p):
    if p is None:
        return 0
    if isinstance(p, int):
        return p
    if isinstance(p, ctypes.c_void_p):
        return p.value or 0
    if hasattr(p, "contents") or isinstance(p, ctypes.Array):
        return ctypes.addressof(p.contents if hasattr(p, "contents") else p)
    raise TypeError(f"emulator: cannot take the address of {type(p)}")


def _flat(ptr, n, dtype):
    """1-d numpy view of n elements at a raw address."""
    ptr = _addr(ptr)
    dtype = np.dtype(dtype)
    if n == 0:
        return np.empty(0, dtype)
    if not ptr:
        raise ValueError("emulator: NULL pointer dereference")
    buf = (ctypes.c_char * (n * dtype.itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=n)


def _view(d, ptr=None):
    """Strided numpy view described by a qb_tensor_t."""
    if hasattr(d, "contents"):
        d = d.contents
    dt = np.dtype(_NP[d.dtype])
    shape = tuple(d.shape[i] for i in range(d.rank))
    stride = tuple(d.stride[i] for i in range(d.rank))
    if any(s < 0 for s in stride):
        raise ValueError("emulator: negative strides")
    if 0 in shape:
        return np.empty(shape, dt)
    extent = 1 + sum((n - 1) * s for n, s in zip(shape, stride))
    base = _flat(d.ptr if ptr is None else ptr, extent, dt)
    return np.lib.stride_tricks.as_strided(
        base, shape=shape, strides=tuple(s * dt.itemsize for s in stride))


def _labels(p, rank):
    if rank == 0:
        return []
    if isinstance(p, (list, tuple)):
        return list(p[:rank])
    return [int(p[i]) for i in range(rank)]


class EmulatedLib:
    """Drop-in for the ``ctypes.CDLL`` object returned by ``_lib.load()``."""

    def __init__(self, real):
        self._real = real
        self.calls = collections.Counter()
        self._launches = 0
        self._err = b""

    # ---- library -------------------------------------------------------
    def __getattr__(self, name):
        if name in _HOST_ONLY:
            return getattr(self._real, name)
        raise AttributeError(f"emulator: {name} is not emulated")

    def qb_last_error(self):
        return self._err or self._real.qb_last_error()

    def qb_launch_count(self):
        return self._launches

    def _fail(self, rc, msg):
        self._err = msg.encode()
        return rc

    def _tick(self, name, n=1):
        self.calls[name] += 1
        self._launches += n
        self._err = b""

    # ---- contraction ---------------------------------------------------
    def _contract(self, A, la, B, lb, C, lc, conjA, conjB, alpha, beta,
                  a_ptr=None, b_ptr=None, c_ptr=None):
        a, b, c = _view(A, a_ptr), _view(B, b_ptr), _view(C, c_ptr)
        la, lb, lc = (_labels(l, v.ndim) for l, v in ((la, a), (lb, b), (lc, c)))
        if a.dtype != b.dtype or a.dtype != c.dtype:
            return self._fail(-3, "dtype mismatch between operands")
        if c.size == 0:
            return 0
        single = a.dtype in (np.float32, np.complex64)
        if single:
            # the native single-precision engine accumulates exactly and rounds
            # once (eligibility was decided by the real planner beforehand)
            wide = np.float64 if a.dtype == np.float32 else np.complex128
            a, b = a.astype(wide), b.astype(wide)
        remap = {}
        for l in la + lb + lc:
            remap.setdefault(l, len(remap))
        sa, sb, sc = ([remap[l] for l in ls] for ls in (la, lb, lc))
        x = a.conj() if conjA else a
        y = b.conj() if conjB else b
        if a.size == 0 or b.size == 0:
            res = np.zeros(c.shape, c.dtype)
        else:
            res = np.einsum(x, sa, y, sb, sc, optimize=True)
        if single and beta != 0.0:
            res = alpha * res + beta * c.astype(res.dtype)
            c[...] = res.astype(c.dtype)
            return 0
        if beta == 0.0:
            c[...] = alpha * res if alpha != 1.0 else res
        else:
            c[...] = alpha * res + beta * c
        return 0

    def qb_contract_pair(self, A, la, B, lb, C, lc, conjA, conjB, engine, ws,
                         ws_bytes, stream):
        need = self._real.qb_contract_pair_workspace(A, la, B, lb, C, lc,
                                                     engine & 0xff)
        if need < 0:
            return int(need)
        if need > 0 and (not _addr(ws) or ws_bytes < need):
            return self._fail(-10, f"workspace too small: need {need} bytes")
        if need > 0 and engine & _lib.QB_ENGINE_WS_ZEROED:
            # the zeroed-header contract the caller signed
            assert not _flat(ws, 1024, np.uint8).any(), "workspace header dirty"
        self._tick("qb_contract_pair")
        return self._contract(A, la, B, lb, C, lc, conjA, conjB, 1.0, 0.0)

    def qb_contract_pair_ab(self, A, la, B, lb, C, lc, conjA, conjB, alpha,
                            beta, ws, ws_bytes, stream):
        need = self._real.qb_contract_pair_workspace(A, la, B, lb, C, lc, 0)
        if need < 0:
            return int(need)
        if need > 0 and (not _addr(ws) or ws_bytes < need):
            return self._fail(-10, f"workspace too small: need {need} bytes")
        self._tick("qb_contract_pair_ab")
        return self._contract(A, la, B, lb, C, lc, conjA, conjB, alpha, beta)

    def qb_contract_batched(self, A0, la, B0, lb, C0, lc, dA, dB, dC, count,
                            conjA, conjB, stream):
        a0 = A0.contents if hasattr(A0, "contents") else A0
        if a0.dtype in (_lib.QB_F32, _lib.QB_C64):
            return self._fail(-101, "qb_contract_batched: single precision has no "
                              "batched engine: widen")
        out = (ctypes.c_int64 * 16)()
        rc = self._real.qb_contract_pair_plan(A0, la, B0, lb, C0, lc, out)
        if rc:
            return rc
        if out[7]:
            return self._fail(-2, "qb_contract_batched: batch labels are not "
                              "allowed inside the per-item signature")
        self._tick("qb_contract_batched")
        pa = _flat(dA, count, np.int64)
        pb = _flat(dB, count, np.int64)
        pc = _flat(dC, count, np.int64)
        for i in range(count):
            rc = self._contract(A0, la, B0, lb, C0, lc, conjA, conjB, 1.0, 0.0,
                                int(pa[i]), int(pb[i]), int(pc[i]))
            if rc:
                return rc
        return 0

    # ---- layout / element-wise ------------------------------------------
    def qb_permute(self, src, dst, conj, stream):
        s, d = _view(src), _view(dst)
        if s.ndim != d.ndim or s.dtype != d.dtype:
            return self._fail(-2, "qb_permute: rank/dtype mismatch")
        if s.shape != d.shape:
            return self._fail(-2, "qb_permute: shape mismatch")
        self._tick("qb_permute")
        d[...] = s.conj() if conj else s
        return 0

    def qb_axpby(self, dtype, n, alpha, x, beta, y, stream):
        self._tick("qb_axpby")
        xv, yv = _flat(x, n, _NP[dtype]), _flat(y, n, _NP[dtype])
        if dtype in (_lib.QB_C64, _lib.QB_C128):
            a, b = complex(alpha[0], alpha[1]), complex(beta[0], beta[1])
        else:
            a, b = alpha[0], beta[0]
        yv[...] = (a * xv + b * yv).astype(yv.dtype)
        return 0

    def qb_scale(self, dtype, n, alpha, div, x, stream):
        self._tick("qb_scale")
        f, g = alpha[0], alpha[1]
        if _addr(div):
            d = _flat(div, 1, _REAL[dtype])[0]
            f, g = (0.0, 0.0) if d == 0 else (f / d, g / d)
        xv = _flat(x, n, _NP[dtype])
        if dtype in (_lib.QB_C64, _lib.QB_C128) and g != 0.0:
            xv[...] = (xv * complex(f, g)).astype(xv.dtype)
        else:
            xv[...] = (xv * f).astype(xv.dtype)
        return 0

    def qb_scale_into(self, dtype, n, alpha, div, x, y, stream):
        self._tick("qb_scale_into")
        f = float(alpha)
        if _addr(div):
            d = _flat(div, 1, _REAL[dtype])[0]
            f = 0.0 if d == 0 else f / d
        yv = _flat(y, n, _NP[dtype])
        yv[...] = (_flat(x, n, _NP[dtype]) * f).astype(yv.dtype)
        return 0

    def qb_dot(self, dtype, n, x, y, out, ws, stream):
        if not _addr(ws):
            return self._fail(-6, "qb_dot: workspace required")
        self._tick("qb_dot", 2)
        xv, yv = _flat(x, n, _NP[dtype]), _flat(y, n, _NP[dtype])
        _flat(out, 1, _NP[dtype])[0] = np.vdot(xv, yv)
        return 0

    def qb_multi_dot(self, dtype, m, n, V, ldv, w, out, ws, stream):
        if dtype != _lib.QB_F64:
            return self._fail(-1, "qb_multi_dot: f64 only")
        if not 1 <= m <= 16:
            return self._fail(-2, "qb_multi_dot: 1 <= m <= 16")
        if not _addr(ws):
            return self._fail(-8, "qb_multi_dot: workspace required")
        self._tick("qb_multi_dot", 2)
        Vv = _flat(V, (m - 1) * ldv + n, np.float64)
        Vm = np.lib.stride_tricks.as_strided(Vv, (m, n), (ldv * 8, 8))
        _flat(out, m, np.float64)[...] = Vm @ _flat(w, n, np.float64)
        return 0

    def qb_multi_axpy(self, dtype, m, n, V, ldv, h, alpha, w, stream):
        if dtype != _lib.QB_F64:
            return self._fail(-1, "qb_multi_axpy: f64 only")
        if not 1 <= m <= 16:
            return self._fail(-2, "qb_multi_axpy: 1 <= m <= 16")
        self._tick("qb_multi_axpy")
        Vv = _flat(V, (m - 1) * ldv + n, np.float64)
        Vm = np.lib.stride_tricks.as_strided(Vv, (m, n), (ldv * 8, 8))
        wv = _flat(w, n, np.float64)
        wv += alpha * (_flat(h, m, np.float64) @ Vm)
        return 0

    def qb_scale_diag(self, dtype, rows, cols, x, d, side, sqrt_d, stream):
        if rows * cols <= 0:
            return 0
        self._tick("qb_scale_diag")
        xv = _flat(x, rows * cols, _NP[dtype]).reshape(rows, cols)
        dv = _flat(d, cols if side else rows, _REAL[dtype])
        f = np.sqrt(dv) if sqrt_d else dv
        if side:
            xv *= f[None, :]
        else:
            xv *= f[:, None]
        return 0

    def qb_convert(self, src_dtype, dst_dtype, n, src, dst, stream):
        ok = {(_lib.QB_F32, _lib.QB_F64), (_lib.QB_F64, _lib.QB_F32),
              (_lib.QB_C64, _lib.QB_C128), (_lib.QB_C128, _lib.QB_C64)}
        if (src_dtype, dst_dtype) not in ok:
            return self._fail(-1, "qb_convert: unsupported conversion")
        if n <= 0:
            return 0
        self._tick("qb_convert")
        _flat(dst, n, _NP[dst_dtype])[...] = _flat(src, n, _NP[src_dtype])
        return 0

    def qb_embed_complex(self, m, n, z, E, stream):
        if m * n <= 0:
            return 0
        self._tick("qb_embed_complex")
        zv = _flat(z, m * n, np.complex128).reshape(m, n)
        Ev = _flat(E, 4 * m * n, np.float64).reshape(2 * m, 2 * n)
        Ev[0::2, 0::2] = zv.real
        Ev[0::2, 1::2] = -zv.imag
        Ev[1::2, 0::2] = zv.imag
        Ev[1::2, 1::2] = zv.real
        return 0

    def qb_extract_complex(self, m, ncols, col_step, E, ld, out, stream):
        if m * ncols <= 0:
            return 0
        self._tick("qb_extract_complex")
        extent = (2 * m - 1) * ld + (ncols - 1) * col_step + 1
        Ev = _flat(E, extent, np.float64)
        Em = np.lib.stride_tricks.as_strided(
            Ev, (2 * m, ncols), (ld * 8, col_step * 8))
        o = _flat(out, m * ncols, np.complex128).reshape(m, ncols)
        o[...] = Em[0::2] + 1j * Em[1::2]
        return 0

    # ---- decompositions ---------------------------------------------------
    def qb_qr_stab(self, dtype, m, n, X, Q, R, stabilized, ws, ws_bytes, stream):
        if dtype != _lib.QB_F64:
            return self._fail(-1, "qb_qr_stab: only f64 is implemented")
        if m <= 0 or n <= 0:
            return 0
        need = self._real.qb_qr_workspace(dtype, m, n)
        if need < 0:
            return self._fail(-2, f"qb_qr_stab: unsupported shape {m} x {n}")
        if not _addr(ws) or ws_bytes < need:
            return self._fail(-8, "qb_qr_stab: workspace too small")
        self._tick("qb_qr_stab")
        x = _flat(X, m * n, np.float64).reshape(m, n)
        # the kernel factors 2^-e x outside max|x| in [2^-200, 2^200]
        mx = np.abs(x).max()
        e = int(np.frexp(mx)[1]) - 1 if np.isfinite(mx) and mx > 0 else 0
        e = e if abs(e) > 200 else 0
        q, r = np.linalg.qr(np.ldexp(x, -e))
        r = np.ldexp(r, e)
        if stabilized:
            sg = np.where(np.diag(r) < 0, -1.0, 1.0)
            q = q * sg[None, :]
            r = r * sg[:, None]
        if _addr(Q):
            _flat(Q, m * n, np.float64).reshape(m, n)[...] = q
        if _addr(R):
            _flat(R, n * n, np.float64).reshape(n, n)[...] = r
        return 0

    def qb_svd(self, dtype, m, n, X, U, S, VH, ws, ws_bytes, sweeps_out, stream):
        if dtype != _lib.QB_F64:
            return self._fail(-1, "qb_svd: only f64 is implemented")
        if m <= 0 or n <= 0:
            return 0
        need = self._real.qb_svd_workspace(dtype, m, n)
        if need < 0:
            return self._fail(-2, f"qb_svd: unsupported shape {m} x {n}")
        if not _addr(ws) or ws_bytes < need:
            return self._fail(-8, "qb_svd: workspace too small")
        if m < n:
            return self._fail(-2, "qb_svd: m < n -- pass the transpose")
        x = _flat(X, m * n, np.float64).reshape(m, n)
        if not np.all(np.isfinite(x)):
            return self._fail(-9, "qb_svd: the input contains NaN or Inf")
        self._tick("qb_svd")
        u, s, vh = np.linalg.svd(x, full_matrices=False)
        _flat(U, m * n, np.float64).reshape(m, n)[...] = u
        _flat(S, n, np.float64)[...] = s
        _flat(VH, n * n, np.float64).reshape(n, n)[...] = vh
        if sweeps_out is not None:
            tgt = getattr(sweeps_out, "_obj", None)
            if tgt is not None:
                tgt.value = 1
        return 0

    def qb_svd_trunc(self, dtype, m, n, X, cutoff, cutoff_mode, max_bond, absorb, renorm,
                     U, S, VH, n_keep, trunc_error, n_null, ws, ws_bytes, sweeps_out, stream):
        """Same contract as csrc/svd_jacobi.cu:qb_svd_trunc, incl. what the
        Jacobi kernel does for exactly-zero singular values (null rows of VH)."""
        if dtype != _lib.QB_F64:
            return self._fail(-1, "qb_svd_trunc: only f64 is implemented")
        if m < n:
            return self._fail(-2, "qb_svd_trunc: m < n -- pass the transpose")
        need = self._real.qb_svd_workspace(dtype, m, n)
        if need < 0:
            return self._fail(-2, f"qb_svd_trunc: unsupported shape {m} x {n}")
        if not _addr(ws) or ws_bytes < need:
            return self._fail(-8, "qb_svd_trunc: workspace too small")
        plan = {100: (0, 0, 1, 1, 1), 2: (0, 0, 0, 0, 1), -1: (1, 0, 1, 1, 0),
                -10: (1, 0, 1, 0, 0), -11: (0, 0, 0, 1, 0), 0: (.5, .5, 1, 1, 0),
                -12: (.5, 0, 1, 0, 0), 12: (0, .5, 0, 1, 0), 1: (0, 1, 1, 1, 0),
                10: (0, 0, 1, 0, 0), 11: (0, 1, 0, 1, 0)}.get(absorb)
        if plan is None:
            return self._fail(-8, f"qb_svd_trunc: invalid absorb code {absorb}")
        lpow, rpow, want_l, want_r, want_s = plan
        x = _flat(X, m * n, np.float64).reshape(m, n)
        if not np.all(np.isfinite(x)):
            return self._fail(-9, "qb_svd: the input contains NaN or Inf")
        self._tick("qb_svd_trunc")
        u, s, vh = np.linalg.svd(x, full_matrices=False)
        s = np.where(s > 1e-300 * max(s[0], 1e-300), s, 0.0) if s.size else s
        nk = ctypes.c_int64(0)
        f = ctypes.c_double(1.0)
        err = ctypes.c_double(0.0)
        sc = np.ascontiguousarray(s, dtype=np.float64)
        rc = self._real.qb_svals_to_keep(
            sc.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), sc.size, float(cutoff),
            int(cutoff_mode), int(max_bond), int(renorm), ctypes.byref(nk), ctypes.byref(f),
            ctypes.byref(err))
        if rc:
            return rc
        k = int(nk.value)
        sk = s[:k] * f.value
        for ref, val in ((n_keep, k), (trunc_error, err.value),
                         (n_null, int(np.sum(~(s[:k] > 0.0))))):
            tgt = getattr(ref, "_obj", None)
            if tgt is not None:
                tgt.value = val
        vk = vh[:k].copy()
        vk[~(s[:k] > 0.0)] = 0.0             # the kernel: W[:, c] / s with s == 0 -> 0
        if want_l and _addr(U):
            _flat(U, m * k, np.float64).reshape(m, k)[...] = u[:, :k] * (sk ** lpow if lpow else 1.0)
        if want_r and _addr(VH):
            scale = (sk ** rpow)[:, None] if rpow else 1.0
            _flat(VH, k * n, np.float64).reshape(k, n)[...] = vk * scale
        if want_s and _addr(S):
            _flat(S, k, np.float64)[...] = sk
        tgt = getattr(sweeps_out, "_obj", None)
        if tgt is not None:
            tgt.value = 1
        return 0


class _FakeStream:
    cuda_stream = 0

    def wait_stream(self, other):
        pass

    def wait_event(self, ev):
        pass


@contextlib.contextmanager
def emulated_abi():
    """Install the emulator: the host layer allocates on the CPU device and
    every kernel-launching ABI call is served by :class:`EmulatedLib`."""
    import importlib
    qarray = importlib.import_module("quimb_b200.array")
    qops = importlib.import_module("quimb_b200.ops")
    qmps = importlib.import_module("quimb_b200.mps")

    real = _lib.load()
    emu = EmulatedLib(real)
    cpu = torch.device("cpu")
    stream = _FakeStream()
    saved = [
        (_lib, "_lib", _lib._lib),
        (_lib, "require_cuda", _lib.require_cuda),
        (_lib, "stream_ptr", _lib.stream_ptr),
        (qarray, "default_device", qarray.default_device),
        (qops, "default_device", qops.default_device),
        (torch.cuda, "current_stream", torch.cuda.current_stream),
        (torch.Tensor, "record_stream", torch.Tensor.record_stream),
        (qmps, "_is_host", qmps._is_host),
    ]

    def require_tensor(t, what="operand"):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{what} must be a torch.Tensor, got {type(t)}")

    _lib._lib = emu
    _lib.require_cuda = require_tensor
    _lib.stream_ptr = lambda: None
    qarray.default_device = lambda: cpu
    qops.default_device = lambda: cpu
    torch.cuda.current_stream = lambda device=None: stream
    torch.Tensor.record_stream = lambda self, s: None
    qmps._is_host = lambda x: False   # no H2D staging: everything is "resident"
    try:
        yield emu
    finally:
        for obj, name, val in saved:
            setattr(obj, name, val)
        # workspaces cached per (device, stream) must not leak into real runs
        qcontract = importlib.import_module("quimb_b200.contract")
        qlanczos = importlib.import_module("quimb_b200.lanczos")
        qlinalg = importlib.import_module("quimb_b200.linalg")
        qcontract._WS.clear()
        qlinalg._WS.clear()
        qlanczos._MD_WS.clear()
        qops._DOT_WS.clear()
