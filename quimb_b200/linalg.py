"""``quimb_b200.linalg`` -- what ``do("linalg.svd" | "linalg.qr" | ...,
like="quimb_b200")`` resolves to.  SVD and QR run on the dedicated CUDA
kernels (``csrc/linalg.cu``: cluster-resident Householder panels, one-sided
block Jacobi); nothing here falls back to a CPU or library factorization.

dtypes: float64 natively.  float32 / complex64 are widened exactly, factored
in double precision and rounded once.  complex128 runs on the same real
kernels through the interleaved real embedding
``E[2i+a, 2j+b] = [[re, -im], [im, re]]``:

* the stabilised real QR of E *is* the embedding of the stabilised complex QR
  (QR with positive diagonal is unique), so Q and R are read off its even
  columns;
* every real singular vector of E is the image of a complex singular vector
  of x, each singular value appears twice; one vector per pair is kept (for
  clusters of equal singular values a small complex Gram matrix decides which
  candidates are independent and re-orthonormalises them).
"""

import ctypes
import functools
import math

import numpy as np
import torch

from . import _lib, ops
from .array import Array

_WS = {}


def _workspace(nbytes, device):
    key = ("linalg", device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _WS.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _WS[key] = buf
    return buf


_WIDE = {torch.float32: torch.float64, torch.complex64: torch.complex128}


def _narrow(fn):
    """float32 / complex64 input: widen exactly, factor in double precision,
    round the factors once (dtype is preserved end to end, as the reference
    does)."""

    @functools.wraps(fn)
    def wrapped(x, *args, **kwargs):
        x = ops.asarray(x)
        if x.t.dtype not in _WIDE:
            return fn(x, *args, **kwargs)
        from .contract import convert
        src = x.t.dtype
        real_src = torch.float32
        wide = Array(convert(ops.materialize(x).t, _WIDE[src]))
        outs = fn(wide, *args, **kwargs)
        res = []
        for o in outs:
            if isinstance(o, Array):
                t = ops.materialize(o).t
                res.append(Array(convert(t, src if t.dtype.is_complex else real_src)))
            else:
                res.append(o)
        return tuple(res)
    return wrapped


def _as_matrix(x):
    x = ops.materialize(ops.asarray(x))
    if x.ndim != 2:
        raise ValueError("quimb_b200.linalg: only 2-d arrays are supported "
                         f"(got shape {x.shape})")
    if x.t.dtype not in (torch.float64, torch.complex128):
        raise TypeError(f"quimb_b200.linalg: dtype {x.dtype} is not supported")
    _lib.require_cuda(x.t)
    return x


def _embed(x):
    """complex (m, n) -> real (2m, 2n) interleaved embedding (one kernel)."""
    m, n = x.shape
    E = torch.empty((2 * m, 2 * n), dtype=torch.float64, device=x.t.device)
    rc = _lib.load().qb_embed_complex(m, n, x.t.data_ptr(), E.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "qb_embed_complex")
    return E


def _extract(E, m, ncols, col_step):
    """complex (m, ncols) with out[i,c] = E[2i, c*step] + 1j E[2i+1, c*step]."""
    out = torch.empty((m, ncols), dtype=torch.complex128, device=E.device)
    rc = _lib.load().qb_extract_complex(m, ncols, col_step, E.data_ptr(), E.stride(0),
                                        out.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "qb_extract_complex")
    return out


@_narrow
def qr(x, stabilized=False, want_q=True, want_r=True):
    """Thin QR of a 2-d device array: Q (m, k), R (k, n), k = min(m, n).
    ``stabilized`` makes diag(R) >= 0 (quimb's qr_stabilized convention);
    complex input is always returned stabilised (diag(R) real, >= 0)."""
    x = _as_matrix(x)
    m, n = x.shape
    k = min(m, n)
    if x.t.dtype == torch.complex128:
        Qe, Re = qr(Array(_embed(x)), stabilized=True, want_q=want_q, want_r=True)
        # The real QR of the embedding is the embedding of the complex QR only
        # through uniqueness, i.e. for full column rank; its deviation from the
        # embedded structure grows like eps * cond(x).  The diagonal of R
        # (k doubles, one host read) tells: ill-conditioned or rank-deficient
        # input (redundant MPS bonds, products of thin factors, ...) takes the
        # SVD route, which is accurate there.
        d = Re.t.diagonal()[0:2 * k:2].abs()
        dh = d.cpu().numpy() if k else np.ones(1)
        if dh.size and dh.min() <= _QR_COMPLEX_COND * dh.max():
            return _qr_complex_via_svd(x, want_q, want_r)
        Q = Array(_extract(Qe.t, m, k, 2)) if want_q else None
        R = Array(_extract(Re.t, k, n, 2)) if want_r else None
        return Q, R
    lib = _lib.load()
    dev = x.t.device
    path = _qr_path(m, n)
    if path == "tsqr":
        return _tsqr(x, stabilized, want_q, want_r)
    if path == "wide":
        # QR of the leading m x m block, R2 = Q^T X[:, m:]
        q, r1 = qr(Array(x.t[:, :m]), stabilized=stabilized)
        r2 = ops.tensordot(q, Array(x.t[:, m:]), axes=((0,), (0,)))
        r = torch.cat([r1.t, r2.t], dim=1)
        return (q if want_q else None), (Array(r) if want_r else None)
    need = lib.qb_qr_workspace(_lib.QB_F64, m, n)
    if need < 0:
        raise ValueError(f"quimb_b200.linalg.qr: unsupported shape {x.shape}")
    ws = _workspace(need, dev)
    Q = torch.empty((m, k), dtype=x.t.dtype, device=dev) if want_q else None
    R = torch.empty((k, n), dtype=x.t.dtype, device=dev) if want_r else None
    rc = lib.qb_qr_stab(_lib.QB_F64, m, n, x.t.data_ptr(),
                        Q.data_ptr() if want_q else None,
                        R.data_ptr() if want_r else None,
                        int(bool(stabilized)), ws.data_ptr(), ws.numel(),
                        _lib.stream_ptr())
    _lib.check(rc, "qb_qr_stab")
    return (Array(Q) if want_q else None), (Array(R) if want_r else None)


# the Householder panel kernel keeps one panel row per thread in registers
# (csrc/linalg.cu: qr_geometry); taller matrices are factored by blocks
_QR_MAX_ROWS = 16384


def _qr_path(m, n):
    """Host-layer decision of :func:`qr` for a real m x n matrix: ``"tsqr"``
    (more than ``_QR_MAX_ROWS`` rows: row blocks), ``"wide"`` (m < n: QR of
    the leading m x m block) or ``"kernel"`` (one ``qb_qr_stab`` call)."""
    if m > _QR_MAX_ROWS and m >= n:
        return "tsqr"
    if m < n:
        return "wide"
    return "kernel"


def _tsqr_blocks(m, n):
    """(row blocks, rows per block) of the TSQR of an m x n matrix."""
    nblk = -(-m // _QR_MAX_ROWS)
    rows = -(-m // nblk)
    if rows < n or nblk * n >= m:
        raise ValueError(f"quimb_b200.linalg.qr: shape {(m, n)} is not supported "
                         f"(more than {_QR_MAX_ROWS} rows and {n} columns)")
    return nblk, rows


def _tsqr(x, stabilized, want_q, want_r):
    """Tall-skinny QR for m > 16384 rows (e.g. the (chi d D^2) x (chi D)
    boundary tensors of BASELINE config 5): row blocks are factored
    independently, the stacked R factors are factored again (recursively), and
    Q is assembled with one tensor-core GEMM per block."""
    m, n = x.shape
    nblk, rows = _tsqr_blocks(m, n)
    qs, rs = [], []
    for lo in range(0, m, rows):
        q, r = qr(Array(x.t[lo:lo + rows]), stabilized=False, want_q=want_q)
        qs.append(q)
        rs.append(r.t)
    stacked = Array(torch.cat(rs, dim=0))                  # (nblk * n, n)
    q2, r = qr(stacked, stabilized=stabilized, want_q=want_q, want_r=want_r)
    if not want_q:
        return None, r
    Q = torch.empty((m, n), dtype=x.t.dtype, device=x.t.device)
    for b, (lo, q) in enumerate(zip(range(0, m, rows), qs)):
        blk = ops.tensordot(q, Array(q2.t[b * n:(b + 1) * n]), axes=((1,), (0,)))
        Q[lo:lo + q.shape[0]] = blk.t
    return Array(Q), r


# relative size of the smallest diagonal entry of R below which the complex
# QR leaves the embedding route (structure error ~ eps / this value)
_QR_COMPLEX_COND = 1e-4


def _qr_complex_via_svd(x, want_q, want_r):
    """x = Q R for (numerically) rank-deficient or ill-conditioned complex x:
    Q = U (a complete isometry: the Jacobi kernel accumulates U as a product of
    rotations, also across zero singular values), R = diag(s) V^H.  R is then
    not triangular -- the factorisation is not unique in this regime and no
    caller on the path needs triangularity (canonisation only needs x = Q R
    with isometric Q); for well-conditioned input the embedding route returns
    the unique stabilised QR."""
    from .split import _ldmul
    U, s, VH = svd(x)
    R = Array(_ldmul(s.t, ops.materialize(VH, force=True).t)) if want_r else None
    return (U if want_q else None), R


def _select_complex_pairs(s_host, gram_fn):
    """Choose one real singular vector per complex singular vector.

    ``s_host``: the 2k sorted singular values of the embedding.  Returns
    ``(src, svals, blocks)``: for each of the k output slots ``src[t]`` is the
    column of the embedding's factors to take (or -1 when the candidates of
    its cluster do not span enough independent directions -- a zero / fully
    degenerate cluster whose vectors came back null -- and the slot has to be
    filled by orthonormal completion), ``svals[t]`` the index into ``s_host``
    of its singular value, and ``blocks`` lists ``(start, size, T)`` for
    clusters of more than one complex vector that need the small
    re-orthonormalising transform ``T`` (size x size, complex, host) on the
    ``size`` picked columns starting at output slot ``start``.  Always k slots:
    every cluster of 2d equal values contributes exactly d (the reference's
    thin SVD returns min(m, n) triplets whatever the rank, decomp.py:1101)."""
    n2 = len(s_host)
    smax = s_host[0] if n2 and s_host[0] > 0 else 1.0
    src, svals, blocks = [], [], []
    i = 0
    while i < n2:
        j = i + 1
        while j < n2 and abs(s_host[j] - s_host[i]) <= 1e-10 * smax:
            j += 1
        if (j - i) % 2:
            j = min(j + 1, n2)  # pairs are never split
        size = j - i
        d = size // 2
        if d <= 1:
            chosen = [0]
            if d == 1:
                # a lone pair is normally taken as is; a null candidate (zero
                # matrix) is detected through its norm
                G = gram_fn(i, i + 1)
                if not np.isfinite(G[0, 0].real) or abs(G[0, 0]) < 0.25:
                    chosen = []
        else:
            G = gram_fn(i, j)  # complex Gram of the candidates, host (size x size)
            G = np.where(np.isfinite(G), G, 0.0)
            # d independent candidates by pivoted Cholesky of the Gram matrix
            # (always the candidate with the largest remaining component: the
            # 2d candidates span exactly a d-dimensional complex space)
            resid = np.real(np.diag(G)).copy()
            Lc = np.zeros((size, d), dtype=G.dtype)
            chosen = []
            for t in range(d):
                c = int(np.argmax(resid))
                if resid[c] <= 1e-12:
                    break
                chosen.append(c)
                col = G[:, c] - Lc[:, :t] @ Lc[c, :t].conj()
                Lc[:, t] = col / np.sqrt(resid[c])
                resid = resid - np.abs(Lc[:, t]) ** 2
                resid[chosen] = -1.0
            chosen.sort()
            if len(chosen) > 1 or (chosen and d > 1):
                Gs = G[np.ix_(chosen, chosen)]
                T = np.linalg.inv(np.linalg.cholesky(Gs)).conj().T
                blocks.append((len(src), len(chosen), T))
        src.extend(i + c for c in chosen)
        src.extend([-1] * (d - len(chosen)))
        svals.extend(i + 2 * t for t in range(d))
        i = j
    return src, svals, blocks


def _complete_isometry(Q, missing, rows=False):
    """Fill the columns ``missing`` of the (m, k) matrix ``Q`` (rows of
    a (k, n) matrix when ``rows``) with vectors orthonormal to each other and to
    the remaining columns: random directions, two projection passes (launches of
    the contraction kernel) and the device QR.  Used for the null vectors of
    zero / rank-deficient complex input, where u and v need not be paired."""
    if rows:
        Qt = Q.transpose(0, 1).conj().contiguous()
        _complete_isometry(Qt, missing)
        Q.copy_(Qt.transpose(0, 1).conj())
        return Q
    m, k = Q.shape
    miss = torch.as_tensor(missing, dtype=torch.int64, device=Q.device)
    keep = [c for c in range(k) if c not in set(missing)]
    gen = torch.Generator(device=Q.device)
    gen.manual_seed(0x5eed + m * 131 + len(missing))
    if Q.dtype.is_complex:
        G = torch.view_as_complex(torch.randn((m, len(missing), 2), dtype=torch.float64,
                                              device=Q.device, generator=gen))
    else:
        G = torch.randn((m, len(missing)), dtype=Q.dtype, device=Q.device, generator=gen)
    if keep:
        Qk = Array(Q.index_select(1, torch.as_tensor(keep, dtype=torch.int64,
                                                     device=Q.device)).contiguous())
        for _ in range(2):
            c = ops.tensordot(Qk.conj(), Array(G), axes=((0,), (0,)))
            G = G - ops.tensordot(Qk, c, axes=((1,), (0,))).t
    Qn, _ = qr(Array(G.contiguous()), stabilized=True, want_r=False)
    Q.index_copy_(1, miss, ops.materialize(Qn).t)
    return Q


@_narrow
def svd(x, full_matrices=False, return_sweeps=False):
    """Thin SVD: U (m, k), s (k,) real descending, VH (k, n)."""
    if full_matrices:
        raise NotImplementedError("quimb_b200.linalg.svd: thin SVD only")
    x = _as_matrix(x)
    m, n = x.shape
    if x.t.dtype == torch.complex128:
        return _svd_complex(x, return_sweeps)
    path = _svd_path(m, n)
    if path == "transpose":
        xt = ops.materialize(Array(x.t.t()))
        out = svd(xt, return_sweeps=return_sweeps)
        u, s, vh = out[:3]
        res = (Array(vh.t.t()), s, Array(u.t.t()))
        return res + (out[3],) if return_sweeps else res
    if path == "qr_first":
        # X = Q R (blocked QR), R = Ur s VH (Jacobi), U = Q Ur (one GEMM)
        q, r = qr(x)
        out = svd(r, return_sweeps=return_sweeps)
        res = (ops.tensordot(q, out[0], axes=((1,), (0,))), out[1], out[2])
        return res + (out[3],) if return_sweeps else res
    lib = _lib.load()
    dev = x.t.device
    need = lib.qb_svd_workspace(_lib.QB_F64, m, n)
    if need < 0:
        raise ValueError(f"quimb_b200.linalg.svd: unsupported shape {x.shape}")
    ws = _workspace(need, dev)
    U = torch.empty((m, n), dtype=x.t.dtype, device=dev)
    S = torch.empty((n,), dtype=x.t.dtype, device=dev)
    VH = torch.empty((n, n), dtype=x.t.dtype, device=dev)
    sweeps = ctypes.c_int(0)
    rc = lib.qb_svd(_lib.QB_F64, m, n, x.t.data_ptr(), U.data_ptr(),
                    S.data_ptr(), VH.data_ptr(), ws.data_ptr(), ws.numel(),
                    ctypes.byref(sweeps), _lib.stream_ptr())
    _lib.check(rc, "qb_svd")
    # numerically zero columns come back with s = 0 and null rows of VH
    # (sorted last): complete them, VH is an isometry like LAPACK's
    nnull = int((S == 0).sum())
    if nnull:
        _complete_isometry(VH, list(range(n - nnull, n)), rows=True)
    out = (Array(U), Array(S), Array(VH))
    return out + (sweeps.value,) if return_sweeps else out


_MIRROR_ABSORB = {100: 100, 2: 2, -1: 1, 1: -1, -10: 11, 11: -10, -11: 10, 10: -11,
                  -12: 12, 12: -12, 0: 0}
# absorb codes whose right (resp. left) factor is returned as an isometry
_ISO_RIGHT = (100, -1, -11)
_ISO_LEFT = (100, 1, 10)


def _svd_path(m, n, code=None):
    """Host-layer decision of :func:`svd` (``code`` None) and
    :func:`svd_trunc` (quimb's absorb code) for a real m x n matrix:
    ``"transpose"`` (m < n; for ``svd_trunc`` also square input whose LEFT
    factor is the isometry, which the kernel serves without accumulated
    rotations when mirrored), ``"qr_first"`` (more than ``_QR_MAX_ROWS`` rows:
    blocked QR, then the SVD of R) or ``"kernel"``."""
    if m < n or (code is not None and m == n and code in (1, 10, 11)):
        return "transpose"
    if m > _QR_MAX_ROWS:
        return "qr_first"
    return "kernel"


def _qr_kernel_route(m, n):
    out = (ctypes.c_int64 * 16)()
    _lib.check(_lib.load().qb_qr_route(m, n, out), "qb_qr_route")
    return {"shape": (m, n), "nb": out[0], "nbo": out[1], "outer_panels": out[2],
            "panel_mask": out[3], "wy_t": bool(out[4]), "inner_panels": out[5]}


def route_qr(shape, dtype=torch.float64):
    """Which kernels :func:`qr` runs for a matrix of this shape and dtype,
    from the decisions it takes itself.  ``kernels`` lists the route of every
    ``qb_qr_stab`` call (``qb_qr_route``: inner / outer panel width, the
    panel-instantiation bitmask, whether aggregated T factors are formed);
    ``panel_mask`` / ``wy_t`` are their union.  Complex input runs on its real
    embedding (and leaves it for the SVD route when the data are
    ill-conditioned, which no shape decides)."""
    m, n = (int(s) for s in shape)
    cplx = torch.empty((), dtype=dtype).is_complex()
    if cplx:
        m, n = 2 * m, 2 * n
    path = _qr_path(m, n)
    res = {"complex_embed": cplx, "path": path, "wide": path == "wide", "tsqr_blocks": 0}
    if path == "tsqr":
        nblk, rows = _tsqr_blocks(m, n)
        res["tsqr_blocks"] = nblk
        shapes = sorted({(rows, n), (m - (nblk - 1) * rows, n)})
        kernels = [_qr_kernel_route(*s) for s in shapes]
        kernels += route_qr((nblk * n, n))["kernels"]
    else:
        kernels = [_qr_kernel_route(m, min(m, n))] if path == "wide" else [_qr_kernel_route(m, n)]
    res["kernels"] = kernels
    res["panel_mask"] = functools.reduce(lambda a, k: a | k["panel_mask"], kernels, 0)
    res["wy_t"] = any(k["wy_t"] for k in kernels)
    return res


_EPILOGUES = ("accumulate", "left", "right", "values")


def route_svd(shape, dtype=torch.float64, absorb=None):
    """Which kernels :func:`svd` (``absorb`` None) or :func:`svd_trunc`
    (quimb's absorb code) runs for a matrix of this shape and dtype, from the
    decisions they take themselves: complex embedding, the wide / square
    mirror transpose, the QR preconditioning above ``_QR_MAX_ROWS`` rows, and
    ``qb_svd_route`` of the Jacobi kernel call (padded width, column blocks,
    stream groups, cluster size, chunk rows, stages, epilogue, graph-replayed
    sweeps, round launches per sweep, its QR preconditioner's panel mask and
    aggregation)."""
    m, n = (int(s) for s in shape)
    cplx = torch.empty((), dtype=dtype).is_complex()
    if cplx:
        if absorb is not None:
            raise TypeError("svd_trunc: float64 only (other dtypes go through svd())")
        m, n = 2 * m, 2 * n
    code = None if absorb is None else int(absorb)
    res = {"complex_embed": cplx, "transpose": False, "mirror": False, "qr_first": None}
    if _svd_path(m, n, code) == "transpose":
        res["transpose"] = m < n
        res["mirror"] = m == n
        m, n = n, m
        code = None if code is None else _MIRROR_ABSORB[code]
    if _svd_path(m, n, code) == "qr_first":
        res["qr_first"] = route_qr((m, n))
        m = n
    out = (ctypes.c_int64 * 16)()
    kcode = 100 if code is None else code
    _lib.check(_lib.load().qb_svd_route(m, n, kcode, out), "qb_svd_route")
    res.update({"kernel_shape": (m, n), "absorb": kcode, "npad": out[0], "nblk": out[1],
                "groups": out[2], "cluster": out[3], "chunk": out[4], "stages": out[5],
                "epilogue": _EPILOGUES[out[6]], "graph_sweeps": out[7],
                "qr_panel_mask": out[8], "qr_wy_t": bool(out[9]), "rounds": out[10]})
    return res


def svd_trunc(x, cutoff=-1.0, cutoff_mode=4, max_bond=-1, absorb=0, renorm=0, info=None):
    """``svd_truncated`` (decomp.py:829-898) as ONE library call on a float64
    device matrix: Jacobi SVD, the reference's keep rule / renormalisation and
    the absorption of the kept singular values run inside ``qb_svd_trunc``
    (csrc/svd_jacobi.cu), which writes only the kept rank.  ``absorb`` is
    quimb's integer code (100 = the three parts).  Returns (left, s, right)
    device Arrays (``None`` for parts the mode does not request); the factors
    are views of exactly-sized buffers -- no slicing copies."""
    x = _as_matrix(x)
    if x.t.dtype != torch.float64:
        raise TypeError("svd_trunc: float64 only (other dtypes go through svd())")
    m, n = x.shape
    code = 100 if absorb is None else int(absorb)
    path = _svd_path(m, n, code)
    if path == "transpose":
        # X^T = V s U^T: factor the transpose, swap the roles of the factors.
        # Also taken for SQUARE input whose LEFT factor is to be the isometry
        # ('right' / 'lorthog' / 'rfactor': DMRG's right-moving sweep): the
        # mirrored mode needs no accumulated rotations in the kernel (the
        # isometry is read off the rotated columns, the other factor is one GEMM
        # with the original matrix), which halves the rows the Jacobi apply
        # phase streams; the transpose itself is one 32 MiB permute-copy.
        xt = ops.materialize(Array(x.t.t()))
        l, s, r = svd_trunc(xt, cutoff, cutoff_mode, max_bond, _MIRROR_ABSORB[code],
                            renorm, info)
        left = None if r is None else Array(r.t.t())
        right = None if l is None else Array(l.t.t())
        return left, s, right
    if path == "qr_first":
        # blocked QR first (m beyond the register-panel limit), then the core
        q, rr = qr(x)
        l, s, r = svd_trunc(rr, cutoff, cutoff_mode, max_bond, code, renorm, info)
        if l is not None:
            l = ops.tensordot(q, l, axes=((1,), (0,)))
        return l, s, r
    lib = _lib.load()
    dev = x.t.device
    need = lib.qb_svd_workspace(_lib.QB_F64, m, n)
    if need < 0:
        raise ValueError(f"quimb_b200.linalg.svd_trunc: unsupported shape {x.shape}")
    ws = _workspace(need, dev)
    want_l = code in (100, -1, -10, 0, -12, 1, 10)
    want_r = code in (100, -1, -11, 0, 12, 1, 11)
    want_s = code in (100, 2)
    U = torch.empty((m * n,), dtype=torch.float64, device=dev) if want_l else None
    VH = torch.empty((n * n,), dtype=torch.float64, device=dev) if want_r else None
    S = torch.empty((n,), dtype=torch.float64, device=dev) if want_s else None
    nk, err, nnull = ctypes.c_int64(0), ctypes.c_double(0.0), ctypes.c_int64(0)
    sweeps = ctypes.c_int(0)
    rc = lib.qb_svd_trunc(_lib.QB_F64, m, n, x.t.data_ptr(), float(cutoff), int(cutoff_mode),
                          int(max_bond), code, int(renorm),
                          U.data_ptr() if want_l else None,
                          S.data_ptr() if want_s else None,
                          VH.data_ptr() if want_r else None,
                          ctypes.byref(nk), ctypes.byref(err), ctypes.byref(nnull),
                          ws.data_ptr(), ws.numel(), ctypes.byref(sweeps), _lib.stream_ptr())
    _lib.check(rc, "qb_svd_trunc")
    k = int(nk.value)
    if info is not None:
        if "error" in info:
            info["error"] = float(err.value)
        info["n_keep"] = k
        info["sweeps"] = int(sweeps.value)
    left = U[:m * k].view(m, k) if want_l else None
    right = VH[:k * n].view(k, n) if want_r else None
    if nnull.value and right is not None and code in _ISO_RIGHT:
        # exactly-zero singular values among the kept ones: their rows of VH
        # came back null; complete the right factor to an isometry (the
        # reference's LAPACK V always is one)
        miss = list(range(k - int(nnull.value), k))
        _complete_isometry(right, miss, rows=True)
    if nnull.value and left is not None and code in (1, 10):
        # same for the left isometry of the accumulation-free right family
        # (U = Q1 U_R with U_R the normalised rotated columns: null for s = 0)
        miss = list(range(k - int(nnull.value), k))
        _complete_isometry(left, miss)
    return (None if left is None else Array(left), None if S is None else Array(S[:k]),
            None if right is None else Array(right))


def _svd_complex(x, return_sweeps):
    m, n = x.shape
    k = min(m, n)
    out = svd(Array(_embed(x)), return_sweeps=True)
    Ue, se, VHe, sweeps = out                       # (2m,2k) (2k,) (2k,2n)
    s_host = se.t.cpu().numpy()
    Uc = _extract(ops.materialize(Ue).t, m, 2 * k, 1)           # (m, 2k) complex
    # row j of VHe viewed as complex is v_j^T; VH rows are conj(v_j)
    Vrows = torch.view_as_complex(ops.materialize(VHe).t.reshape(2 * k, n, 2))

    def gram(i, j):
        Z = Array(Uc[:, i:j])
        return ops.tensordot(Z.conj(), Z, axes=((0,), (0,))).to_numpy()

    src, svals, blocks = _select_complex_pairs(s_host, gram)
    missing = [t for t, c in enumerate(src) if c < 0]
    dev = x.t.device
    idx = torch.as_tensor([max(c, 0) for c in src], dtype=torch.int64, device=dev)
    U = Uc.index_select(1, idx).contiguous()                    # (m, k)
    VH = Array(Vrows.index_select(0, idx).contiguous()).conj()  # (k, n), lazy conj
    VH = ops.materialize(VH).t
    S = se.t.index_select(0, torch.as_tensor(svals, dtype=torch.int64, device=dev)).contiguous()
    for start, size, T in blocks:
        Td = ops.asarray(np.ascontiguousarray(T))
        Ub = Array(U[:, start:start + size])
        U[:, start:start + size] = ops.tensordot(Ub, Td, axes=((1,), (0,))).t
        Vb = Array(VH[start:start + size, :])
        VH[start:start + size, :] = ops.tensordot(Td.conj().transpose(1, 0), Vb,
                                                  axes=((1,), (0,))).t
    if missing:
        # slots whose candidates were null: only ever the sigma = 0 cluster
        # (its u and v are unpaired), completed to full isometries
        _complete_isometry(U, missing)
        _complete_isometry(VH, missing, rows=True)
        S.index_fill_(0, torch.as_tensor(missing, dtype=torch.int64, device=dev), 0.0)
    # null right vectors of a zero cluster that the kernel returned
    # un-normalised are caught the same way (rows of VH with norm far from 1)
    res = (Array(U), Array(S), Array(VH))
    return res + (sweeps,) if return_sweeps else res


def norm(x, ord=None):
    """Frobenius / 2-norm through the deterministic dot kernel.

    Known limit: this is sqrt(<x, x>) without scaling, so it overflows to inf
    for norms above about 2^511 and underflows to 0 below about 2^-537, as
    numpy's ``norm`` (the reference's) does."""
    x = ops.asarray(x)
    if ord not in (None, "fro", 2):
        raise NotImplementedError("only the Frobenius / vector 2-norm")
    flat = ops.materialize(x).reshape(-1)
    return ops.sqrt(ops.real(ops.vdot(flat, flat)))


# matrices up to this size are "tiny projected problems" solved on the host
_EIGH_HOST_BELOW = 64


def eigh(x, host_below=None):
    """Hermitian eigendecomposition ``x = v diag(w) v^H`` (``w`` ascending,
    as numpy / the reference's ``xp.linalg.eigh``).

    Tiny problems (n <= ``host_below``, default ``_EIGH_HOST_BELOW`` = 64: Lanczos tridiagonals, DMRG's dense-Heff
    branch for prod(dims) < 800, dmrg.py:690) are host-side control logic in
    the reference too and are solved on the host.  Anything larger runs on the
    device through the one-sided Jacobi kernel: with ``sigma = |x|_F`` the
    matrix ``x + sigma I`` is positive semi-definite, so its singular value
    decomposition *is* its eigendecomposition (U = V) and
    ``w = s - sigma``; eigenvalues are accurate to ``eps * |x|_F`` like any
    backward-stable dense eigensolver.  complex128 goes through the real
    embedding, float32 / complex64 through the exact widening pass (both
    inherited from :func:`svd`).  ``sigma`` stays on the device; max|x| is
    read once on the host to decide the power-of-two scaling (and to reject
    NaN / Inf) before the SVD, which synchronises anyway."""
    x = ops.asarray(x)
    if x.ndim != 2 or x.shape[0] != x.shape[1]:
        raise ValueError(f"eigh: expected a square matrix, got shape {x.shape}")
    n = x.shape[0]
    if host_below is None:
        host_below = _EIGH_HOST_BELOW
    if n <= host_below:
        a = ops.to_numpy(x)
        w, v = np.linalg.eigh(a)
        return ops.asarray(w), ops.asarray(v)
    xm = ops.materialize(x, force=True)            # private copy (shifted in place)
    _lib.require_cuda(xm.t)
    # |x|_F squares the entries: outside [2^-200, 2^200] (the window of the
    # SVD kernel, csrc/internal.h) x is scaled by 2^-e first, like the SVD
    # scales its own input, and the eigenvalues are scaled back
    amax = float(torch.amax(torch.abs(xm.t))) if xm.t.numel() else 0.0
    if not math.isfinite(amax):
        raise ValueError("eigh: the input contains NaN or Inf")
    e = math.frexp(amax)[1] - 1 if amax > 0.0 else 0
    if abs(e) <= _DECOMP_SAFE_EXP:
        e = 0
    for f in _pow2_factors(-e):
        xm.t.mul_(f)
    sigma = norm(xm)                               # 0-d, real, on the device
    sg = sigma.t.to(_REAL_OF[xm.t.dtype])
    xm.t.diagonal().add_(sg)
    _, s, VH = svd(xm)
    w = (s.t - sg.to(s.t.dtype)).flip(0)           # ascending
    for f in _pow2_factors(e):
        w = w * f
    v = Array(VH.t.flip(0).transpose(0, 1), not VH.cj)   # v[:, i] = conj(VH[k-1-i, :])
    return Array(w), v


_DECOMP_SAFE_EXP = 200


def _pow2_factors(k):
    """2^k as at most two representable factors (|k| <= 2044)."""
    if k == 0:
        return ()
    h = k // 2
    return (math.ldexp(1.0, h), math.ldexp(1.0, k - h))


_REAL_OF = {torch.float32: torch.float32, torch.float64: torch.float64,
            torch.complex64: torch.float32, torch.complex128: torch.float64}


# ------------------------------------------------ Cholesky / pseudo-inverse --
def _scale_rows(x, d, sqrt_d=False):
    """x[i, :] *= d[i]^p in place on a contiguous matrix (``qb_scale_diag``)."""
    rows, cols = x.shape
    rc = _lib.load().qb_scale_diag(_lib.qb_dtype(x.dtype), rows, cols, x.data_ptr(),
                                   d.data_ptr(), 0, int(sqrt_d), _lib.stream_ptr())
    _lib.check(rc, "qb_scale_diag")
    return x


@_narrow
def _cholesky_lower(x):
    x = _as_matrix(x)
    n = x.shape[0]
    if x.shape[1] != n:
        raise ValueError(f"cholesky: expected a square matrix, got shape {x.shape}")
    if n == 0:
        return (x,)
    if x.t.dtype == torch.complex128:
        # chol(embed(x)) = embed(chol(x)): the embedding of the complex factor
        # is real lower triangular with a positive diagonal, and that
        # factorisation is unique
        (Le,) = _cholesky_lower(Array(_embed(x)))
        return (Array(_extract(Le.t, n, n, 2)),)
    w, v = eigh(x)
    wh = w.t.detach().cpu().numpy()
    tol = n * float(np.finfo(np.float64).eps) * float(np.abs(wh).max(initial=0.0))
    if not np.all(np.isfinite(wh)) or wh.max(initial=0.0) <= 0.0 or wh.min() < -tol:
        raise np.linalg.LinAlgError("Matrix is not positive definite")
    sq = torch.clamp(w.t, min=0.0).contiguous()
    B = ops.materialize(Array(v.t.transpose(0, 1), not v.cj), force=True).t   # V^H
    _scale_rows(B, sq, sqrt_d=True)                                           # sqrt(w) V^H
    _, R = qr(Array(B), stabilized=True, want_q=False)
    return (ops.materialize(Array(R.t.transpose(0, 1))),)


def cholesky(x, upper=False):
    """Cholesky factor of a Hermitian positive-definite matrix, ``x = L L^H``
    (``upper=True``: the factor ``L^H``), the ``xp.linalg.cholesky`` behind
    quimb's ``cholesky_regularized`` (decomp.py:2245-2322).

    No new device code: with ``x = V diag(w) V^H`` from the Jacobi ``eigh``,
    the stabilised QR ``sqrt(w) V^H = Q R`` gives ``x = R^H R`` with
    ``diag(R) > 0``, and the Cholesky factor is unique, so ``L = R^H``.  Not
    positive definite (an eigenvalue below ``-n eps |w|_max``) raises
    ``numpy.linalg.LinAlgError`` as LAPACK does; eigenvalues inside the
    rounding band around zero are treated as zero.  Off the contraction hot
    path (bond-environment gauging); ~10x the flops of a blocked potrf."""
    (L,) = _cholesky_lower(x)
    if upper:
        return ops.materialize(Array(L.t.transpose(0, 1), True))
    return L


def pinv(x, rcond=None):
    """Moore-Penrose pseudo-inverse through the device SVD (singular values
    below ``rcond * s_max`` are dropped; default ``max(m, n) * eps`` like
    ``numpy.linalg.pinv``'s ``rtol``)."""
    x = ops.asarray(x)
    U, s, VH = svd(x)
    st = s.t
    if rcond is None:
        rcond = max(x.shape) * float(torch.finfo(st.dtype).eps)
    smax = st.max() if st.numel() else st.new_zeros(())
    keep = st > rcond * smax
    sinv = torch.where(keep, 1.0 / torch.where(keep, st, torch.ones_like(st)),
                       torch.zeros_like(st)).contiguous()
    Vs = _scale_rows(ops.materialize(VH, force=True).t, sinv)        # s^-1 V^H
    left = Array(Vs.transpose(0, 1), True)                           # V s^-1
    right = Array(U.t.transpose(0, 1), not U.cj)                     # U^H
    return ops.matmul(left, right)


def inv(x):
    """Dense inverse.  Library forward (torch / cuSOLVER getrf + getri): not on
    the contraction hot path, listed in SURVEY 8(b) as forwardable."""
    return Array(torch.linalg.inv(ops.asarray(x).resolve()))


def solve(a, b):
    """``a @ out = b``.  Library forward (torch / cuSOLVER), see :func:`inv`."""
    return Array(torch.linalg.solve(ops.asarray(a).resolve(), ops.asarray(b).resolve()))


def solve_triangular(a, b, lower=False, trans=0, unit_diagonal=False, **kwargs):
    """``scipy.linalg.solve_triangular`` signature (used by quimb's
    ``qr_via_cholesky``, decomp.py:2404).  Library forward (torch / cuBLAS
    trsm), see :func:`inv`."""
    A = ops.asarray(a).resolve()
    B = ops.asarray(b).resolve()
    if trans in (1, "T"):
        A, lower = A.transpose(-2, -1), not lower
    elif trans in (2, "C"):
        A, lower = A.conj().transpose(-2, -1), not lower
    vec = B.ndim == 1
    if vec:
        B = B[:, None]
    out = torch.linalg.solve_triangular(A, B, upper=not lower, unitriangular=unit_diagonal)
    return Array(out[:, 0] if vec else out)


def eigvalsh(x):
    return eigh(x)[0]


def expm(x):
    """Matrix exponential.  Library forward (torch.linalg.matrix_exp): gate
    construction (``isometrize(method="exp")``, Trotter terms), not on the
    contraction hot path."""
    return Array(torch.linalg.matrix_exp(ops.asarray(x).resolve()))


def eig(x):
    """General (non-Hermitian) eigendecomposition ``(w, v)``.  Library forward
    (torch / cuSOLVER geev; belief-propagation gauging of quimb calls it on
    small message matrices): not on the contraction hot path."""
    w, v = torch.linalg.eig(ops.asarray(x).resolve())
    return Array(w), Array(v)


def lu(x, permute_l=False):
    """``scipy.linalg.lu`` signature: ``(P, L, U)`` or ``(P @ L, U)``.
    Library forward (torch / cuSOLVER getrf with partial pivoting)."""
    P, L, U = torch.linalg.lu(ops.asarray(x).resolve())
    if permute_l:
        return Array(P @ L), Array(U)
    return Array(P), Array(L), Array(U)


def lstsq(a, b, rcond=None):
    """``numpy.linalg.lstsq`` return convention ``(x, residuals, rank, s)``.
    Library forward (torch / cuSOLVER gels); tensor-network fitting calls it on
    small normal-equation blocks, nothing on the contraction hot path does."""
    A = ops.asarray(a).resolve()
    B = ops.asarray(b).resolve()
    vec = B.ndim == 1
    if vec:
        B = B[:, None]
    sol = torch.linalg.lstsq(A, B.to(A.dtype), rcond=rcond)
    x = sol.solution[:, 0] if vec else sol.solution
    return Array(x), Array(sol.residuals), sol.rank, Array(sol.singular_values)
