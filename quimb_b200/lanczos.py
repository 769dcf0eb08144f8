"""On-device Lanczos for the DMRG local eigensolve.

The reference solves ``eigh(Heff, k=1, which='SA', v0=..., ncv=4, tol=1e-3)``
with scipy's ARPACK (quimb/tensor/tn1d/dmrg.py:626-645 ->
quimb/linalg/scipy_linalg.py:113-128): the Krylov vectors live on the host
and every iteration calls back into ``TNLinearOperator._matvec``.  With a
device matvec that would cross PCIe twice per iteration, so the whole Krylov
process lives on the device here:

  * thick-restart Lanczos (the lowest few Ritz vectors are kept together with
    their images H x, which are known, so a restart costs no matvec and loses
    little of the Krylov space), full re-orthogonalisation by
    classical Gram-Schmidt applied twice, each pass = two fused HBM-bound
    kernels (``qb_multi_dot`` : h = V w,  ``qb_multi_axpy`` : w -= V^T h);
  * the images ``W_j = H v_j`` are kept, so the projected matrix
    ``V H V^T`` is one skinny contraction;
  * the projected matrix is assembled on the host from the Gram-Schmidt
    coefficients (small device->host reads of <= 65 doubles per step), so the
    Ritz value and the Lanczos residual estimate are monitored as the basis
    grows and a solve stops the moment it has converged; while the estimate is
    still far above the threshold up to two steps are queued before the next
    read, so the device is not idle while the host decides.  The true residual
    norm |H x - theta x| is checked once per cycle; the tiny dense
    eigenproblem is host control logic, as in ARPACK.

Convergence test as in ARPACK's dsaupd: ``resid <= tol * max(eps^(2/3),
|theta|)``.  The basis size ``ncv`` is a free parameter of the device solver:
ARPACK's 4 is memory-frugal for host vectors; on an 80 GB device a basis of
8-16 vectors (32 MiB each at chi = 1024) needs far fewer matvecs.
``eigh_arpack_host_driver`` is the parity mode (scipy ARPACK on the host
driving the device matvec).
"""

import ctypes
import math

import numpy as np
import torch

from . import _lib, ops
from .array import Array
from .contract import contract_pair
from .linalg import norm as _norm

_J, _N = 0, 1
_MD_WS = {}
_NCV_MAX = 64


def _md_ws(dev):
    """Partials of ``qb_multi_dot``, one buffer per (device, stream)."""
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
    ws = _MD_WS.get(key)
    if ws is None:
        ws = torch.empty(_lib.load().qb_multi_dot_workspace(), dtype=torch.uint8,
                         device=dev)
        _MD_WS[key] = ws
    return ws


def _norm_c(x, comm):
    """2-norm of a (possibly row-sharded) vector as a 0-d device Array."""
    if comm is None:
        return _norm(x)
    flat = ops.materialize(x).reshape(-1)
    n2 = ops.real(ops.vdot(flat, flat))
    comm.all_reduce_(n2.t)
    return ops.sqrt(n2)


_MD_MAX = 16        # rows per call of the fused Krylov kernels (csrc: MD_MAX)


# (a normalisation queued before the host has seen the norm divides by a
# device scalar; qb_scale maps an exactly zero divisor -- exact Krylov
# breakdown -- to a zero vector, and the host drops everything behind that step)


def _combine(V, m, coeffs, out, alpha=1.0):
    """out += alpha * sum_j coeffs[j] V[j]  (j < m), 16 basis rows per launch."""
    lib = _lib.load()
    n = out.numel()
    st = _lib.stream_ptr()
    for j0 in range(0, m, _MD_MAX):
        mm = min(_MD_MAX, m - j0)
        rc = lib.qb_multi_axpy(_lib.QB_F64, mm, n, V[j0].data_ptr(), V.stride(0),
                               coeffs[j0:].data_ptr(), float(alpha), out.data_ptr(), st)
        _lib.check(rc, "qb_multi_axpy")


def _orthogonalise(V, j, w, h, comm=None, keep=None):
    """Two classical Gram-Schmidt passes of w against V[0..j] (in place), each
    pass = all inner products first, then the update (16 basis rows per
    launch of the fused kernels).  With ``comm`` the vectors are row slabs:
    the dot products are summed over the ranks (one tiny all-reduce per pass).
    ``keep`` (device vector) receives the first-pass coefficients <V[i], w>:
    for w = H V[j] that is column j of the projected matrix V^T H V."""
    lib = _lib.load()
    m, n = j + 1, w.numel()
    st = _lib.stream_ptr()
    ws = _md_ws(w.device).data_ptr()
    for it in range(2):
        # the first pass writes its coefficients straight into ``keep`` (the
        # caller's column of the projected matrix): no copy kernel
        hc = keep if (it == 0 and keep is not None) else h
        for j0 in range(0, m, _MD_MAX):
            mm = min(_MD_MAX, m - j0)
            rc = lib.qb_multi_dot(_lib.QB_F64, mm, n, V[j0].data_ptr(), V.stride(0),
                                  w.data_ptr(), hc[j0:].data_ptr(), ws, st)
            _lib.check(rc, "qb_multi_dot")
        if comm is not None:
            comm.all_reduce_(hc[:m])
        _combine(V, m, hc, w, -1.0)


def eigh_lanczos(matvec, v0, which="SA", ncv=4, tol=1e-3, maxiter=None,
                 return_info=False, comm=None, min_steps=4):
    """Lowest ('SA') or highest ('LA') eigenpair of a Hermitian operator.

    Parameters
    ----------
    matvec : callable(Array[n]) -> Array[n]
        Device matvec on flat contiguous vectors.
    v0 : Array
        Start vector (any shape, flattened).
    ncv : int
        Largest Krylov basis between restarts (2 <= ncv <= 64); a cycle ends
        as soon as the Lanczos residual estimate meets ``tol``.
    min_steps : int
        Matvecs before the residual estimate may stop the solve.  ARPACK with
        ``ncv=4`` (the reference's setting) always spends 4; stopping earlier
        than that leaves the local states of a sweep visibly less converged
        than the reference's at the same ``tol``.
    comm : object with ``all_reduce_(tensor)``, optional
        Row-sharded mode (quimb_b200.dist.BondShard): ``v0`` and every vector
        handed to / returned by ``matvec`` is this rank's slab; inner products
        are summed over the ranks, all ranks take identical decisions.
    Returns ``(theta: float, x: Array[n])`` (+ info dict).
    """
    v0 = ops.materialize(ops.asarray(v0)).reshape(-1)
    if v0.t.dtype == torch.complex128:
        # A Hermitian operator on C^n is a real symmetric operator on R^2n
        # (complex storage viewed as interleaved reals); each eigenvalue is
        # doubled and every real eigenvector is the image of a complex one,
        # so the real Krylov machinery applies unchanged.
        def mv_real(vr):
            vc = Array(torch.view_as_complex(vr.t.reshape(-1, 2)))
            out = ops.materialize(matvec(vc)).t.reshape(-1)
            return Array(torch.view_as_real(out).reshape(-1))

        vr0 = Array(torch.view_as_real(v0.t).reshape(-1))
        theta, xr, info = eigh_lanczos(mv_real, vr0, which=which, ncv=ncv, tol=tol,
                                       maxiter=maxiter, return_info=True, comm=comm,
                                       min_steps=min_steps)
        x = Array(torch.view_as_complex(xr.t.reshape(-1, 2)))
        return (theta, x, info) if return_info else (theta, x)
    if v0.t.dtype in (torch.float32, torch.complex64):
        # single precision operator: the Krylov process runs in double (basis,
        # inner products, projected matrix); only the vectors handed to / taken
        # from ``matvec`` are rounded, so the operator keeps its own dtype
        # (quimb preserves the dtype end to end, test_dmrg.py:290-300)
        from .contract import convert
        narrow = v0.t.dtype
        wide = torch.float64 if narrow == torch.float32 else torch.complex128

        def mv_wide(vw):
            vn = Array(convert(ops.materialize(vw).t, narrow))
            out = ops.materialize(matvec(vn)).t.reshape(-1)
            return Array(convert(out, wide))

        # the operator itself is only accurate to single precision: a tighter
        # residual than that can never be met
        tol = max(tol, 100 * float(torch.finfo(torch.float32).eps))
        theta, xw, info = eigh_lanczos(mv_wide, Array(convert(v0.t, wide)), which=which,
                                       ncv=ncv, tol=tol, maxiter=maxiter, return_info=True,
                                       comm=comm, min_steps=min_steps)
        x = Array(convert(ops.materialize(xw).t, narrow))
        return (theta, x, info) if return_info else (theta, x)
    n = v0.size
    dt = v0.t.dtype
    if dt != torch.float64:
        raise NotImplementedError(f"eigh_lanczos: dtype {dt} is not implemented "
                                  "(float32/64, complex64/128; no fallback)")
    dev = v0.t.device
    m = max(2, min(int(ncv), n, _NCV_MAX))
    if maxiter is None:
        maxiter = 1000
    V = torch.zeros((m, n), dtype=dt, device=dev)
    W = torch.empty((m, n), dtype=dt, device=dev)
    w = torch.empty((n,), dtype=dt, device=dev)
    h = torch.zeros((_NCV_MAX,), dtype=dt, device=dev)
    eps23 = np.finfo(np.float64).eps ** (2.0 / 3.0)
    sign = 1.0 if which in ("SA", "SR") else -1.0

    # operators of this package take ``out=`` (a flat float64 basis row); the
    # real / single-precision wrappers above and foreign callables do not
    out_ok = bool(getattr(matvec, "supports_out", False))
    nrm = _norm_c(v0, comm)
    V[0].copy_(v0.t)
    ops.scale_(Array(V[0]), 1.0, div_by=nrm)
    nmv = 0
    theta, resid = None, None
    info = {"restarts": 0, "converged": False}
    x = Array(V[0])
    mmax = m
    min_steps = min(int(min_steps), n)
    colbuf = torch.zeros((mmax, _NCV_MAX + 1), dtype=dt, device=dev)
    betas = np.zeros(mmax)
    info["host_reads"] = 0
    # thick restart: the k lowest Ritz vectors (and their known images) are
    # kept, followed by the last residual direction -- close to unrestarted
    # Lanczos in matvecs at a bounded basis (Wu & Simon's TRLan scheme)
    keep_max = max(1, min(mmax // 4, 8))
    Vk = Wk = None
    jstart = 0
    best_resid, best_cycle = np.inf, 0
    Hh = np.zeros((mmax, mmax))
    for cycle in range(maxiter):
        # The projected matrix is assembled column by column on the host from
        # the Gram-Schmidt coefficients (ONE small device->host read per step),
        # so the Ritz value and the Lanczos residual estimate
        # |beta_{j+1} y_j| are known after every matvec and the cycle stops as
        # soon as it has converged: an already good v0 costs ~3 matvecs (like
        # ARPACK's ncv = 4), a hard problem uses the whole basis without
        # paying for restarts it does not need.
        m = mmax
        meff = m
        pending = jstart          # first projected-matrix column not yet on the host
        skip = 0
        est_prev = est = None
        for j in range(jstart, m):
            if out_ok:
                # the operator writes H v_j straight into its basis slot
                matvec(Array(V[j]), out=W[j])
            else:
                Wj = matvec(Array(V[j]))
                W[j].copy_(ops.materialize(Wj).t.reshape(-1))
            nmv += 1
            w.copy_(W[j])
            _orthogonalise(V, j, w, h, comm, keep=colbuf[j])
            bnorm = _norm_c(Array(w), comm)
            colbuf[j, j + 1].copy_(bnorm.t)
            if skip > 0 and j + 1 < m:
                # far from convergence (see below): keep the device busy, the
                # columns of these steps are read together with the next one
                skip -= 1
                ops.scale_into(Array(V[j + 1]), Array(w), 1.0, div_by=bnorm)
                continue
            rows = colbuf[pending:j + 1, :j + 2].cpu().numpy()
            info["host_reads"] += 1
            # the steps read now are examined in order: the first one that has
            # converged, broken down (invariant subspace: beta = 0) or filled
            # the basis ends the cycle -- steps queued behind it are dropped
            hit = None
            for jj in range(pending, j + 1):
                c = rows[jj - pending]
                Hh[:jj + 1, jj] = c[:jj + 1]
                Hh[jj, :jj + 1] = c[:jj + 1]
                betas[jj] = beta = float(c[jj + 1])
                evals, evecs = np.linalg.eigh(sign * Hh[:jj + 1, :jj + 1])
                theta = sign * evals[0]
                y = evecs[:, 0]
                est_prev, est = est, abs(beta * y[-1])
                thresh = tol * max(eps23, abs(theta))
                conv = est <= thresh and nmv - (j - jj) >= min_steps
                if (conv or jj + 1 == m or not np.isfinite(est)
                        or beta <= 1e-14 * max(1.0, abs(theta))):
                    hit = jj
                    break
            pending = j + 1
            if hit is not None:
                meff = hit + 1
                if hit < j:
                    # restore the residual direction of step `hit` for the
                    # restart: w of that step was overwritten by later ones
                    w.copy_(V[hit + 1])
                    bnorm = Array(torch.ones((), dtype=dt, device=dev))
                break
            # How many steps can run before the next look?  With the observed
            # contraction rate r the estimate reaches 10 x the threshold after
            # log(est / 10 thresh) / log(1 / r) steps; never more than 2 ahead
            # (Lanczos converges superlinearly), never while a decision --
            # convergence or breakdown -- could be near.
            skip = 0
            if est > 10.0 * thresh:
                r = 0.3 if not est_prev or est_prev <= est else max(est / est_prev, 0.05)
                if r < 1.0:
                    skip = int(min(2, math.log(est / (10.0 * thresh)) / -math.log(r)))
                if nmv + skip + 1 < min_steps:
                    skip = max(skip, min(2, min_steps - nmv - 2))
            ops.scale_into(Array(V[j + 1]), Array(w), 1.0, div_by=bnorm)
        m = meff

        def ritz(yvec, out_v, out_w):
            yd = torch.zeros(_NCV_MAX, dtype=dt)
            yd[:m] = torch.as_tensor(np.ascontiguousarray(yvec), dtype=dt)
            yd = yd.to(dev)
            out_v.zero_()
            out_w.zero_()
            _combine(V, m, yd, out_v)
            _combine(W, m, yd, out_w)

        xnew = torch.empty((n,), dtype=dt, device=dev)
        hx = torch.empty((n,), dtype=dt, device=dev)
        ritz(y, xnew, hx)
        # true residual |H x - theta x| (robust to Krylov breakdown): one more
        # host read per cycle.  `w` still holds the last residual direction,
        # so the check uses its own buffer.
        rchk = hx.clone()
        ops.axpby(-theta, Array(xnew), 1.0, Array(rchk))
        resid = float(_norm_c(Array(rchk), comm).item())
        info["restarts"] = cycle
        if resid <= tol * max(eps23, abs(theta)) or not np.isfinite(resid):
            info["converged"] = bool(np.isfinite(resid))
            x = Array(xnew)
            break
        x = Array(xnew)
        if cycle + 1 >= maxiter:
            break                      # no further cycle: skip the restart set-up
        # stagnation guard: a residual that has not improved over many matvecs
        # (>= 300 and >= 10 full bases) sits at the accuracy of the operator
        # (rounding of the matvec); return the best Ritz pair instead of
        # spinning to ``maxiter``
        if resid < 0.99 * best_resid:
            best_resid, best_cycle = resid, nmv
        elif nmv - best_cycle >= max(300, 10 * mmax):
            info["stagnated"] = True
            break
        # ---- thick restart ------------------------------------------------
        k = max(1, min(keep_max, m - 1))
        if Vk is None:
            Vk = torch.empty((keep_max, n), dtype=dt, device=dev)
            Wk = torch.empty((keep_max, n), dtype=dt, device=dev)
        ritz(y, Vk[0], Wk[0])                       # == (xnew, hx)
        for i in range(1, k):
            ritz(evecs[:, i], Vk[i], Wk[i])
        usable = beta > 1e-14 * max(1.0, abs(theta)) and np.isfinite(beta)
        V[:k].copy_(Vk[:k])
        W[:k].copy_(Wk[:k])
        Hh[:] = 0.0
        Hh[np.arange(k), np.arange(k)] = sign * evals[:k]
        if usable and k < mmax:
            # next basis vector: the residual direction shared by all Ritz pairs
            V[k].copy_(w)
            ops.scale_(Array(V[k]), 1.0, div_by=bnorm)
            jstart = k
        else:
            # invariant subspace reached without convergence of the true
            # residual (rounding): continue from the best Ritz vector alone
            k = 1
            Hh[:] = 0.0
            jstart = 0
        if jstart == 0:
            xn = _norm_c(Array(V[0]), comm)
            ops.scale_(Array(V[0]), 1.0, div_by=xn)
    # normalise the Ritz vector
    xn = _norm_c(x, comm)
    x = ops.scale_(ops.materialize(x, force=True), 1.0, div_by=xn)
    info.update(nmatvec=nmv, resid=resid, theta=theta, ncv=mmax)
    if return_info:
        return float(theta), x, info
    return float(theta), x


def eigh_arpack_host_driver(matvec, v0, which="SA", ncv=4, tol=1e-3):
    """Parity mode: the reference's own eigensolver (scipy ARPACK on the
    host) driving the device matvec; every iteration copies the vector
    host->device->host.  For validation only."""
    import scipy.sparse.linalg as spla

    v0h = ops.to_numpy(ops.asarray(v0)).reshape(-1)
    n = v0h.size
    count = [0]

    def mv(vec):
        count[0] += 1
        out = matvec(ops.asarray(np.ascontiguousarray(vec)))
        return ops.to_numpy(out).reshape(-1)

    A = spla.LinearOperator((n, n), matvec=mv, dtype=v0h.dtype)
    lk, vk = spla.eigsh(A, k=1, which=which, v0=v0h, ncv=ncv, tol=tol)
    return float(lk[0]), ops.asarray(vk[:, 0]), {"nmatvec": count[0]}
