"""Apply an MPO to an MPS on the device and compress the result by successive
sketching: successive randomized compression (SRC, arXiv:2504.06475), its
variant sampling with an MPS, and successive deterministic compression
(SDC), each alone or followed by a direct sweep.

Mirrors, at array level and for open-boundary (l, p, r) site lists,

  _do_sweep_compress_from_low_rank_left_envs   tn1d/compress.py:1115-1266
  _src_get_local_noise_tensors                  tn1d/compress.py:1269-1322
  tensor_network_1d_compress_sdc (+ oversample) tn1d/compress.py:1325-1650
  tensor_network_1d_compress_src (+ oversample) tn1d/compress.py:1653-2002
  tensor_network_1d_compress_srcmps (+ overs.)  tn1d/compress.py:2005-2339

on the ladder of ``mpo_compress``: MPS site A[a, p, b] under MPO site
W[v, u, o, p], o the output index.  Every method builds low-rank left
environments LE[x, a, v] from the left (x: the k noise samples for SRC, the
bond of the sampling MPS for 'srcmps', the kept singular directions for
SDC), then sweeps in from the right: at each site the sketch
t[(o, k), x] = LE A W RE is factored by one QR, its isometric factor Q
becomes the output site and, conjugated through the contraction's flag,
closes the next right environment.  No SVD or eigh runs in 'src' /
'srcmps'; 'sdc' truncates each left environment by SVD.

An SRC left-environment step is one ``qb_sketch_env`` launch (the sample-
batched LE . (W . Omega) product, csrc/sketch.cu) and one ``contract_pair``
GEMM; every other contraction is one ``contract_pair`` launch.  The noise is
drawn on the host by the rule of ``quimb_b200.random.array``, cast to the
ladder's dtype and uploaded once per site.
"""

import ctypes
import warnings

import numpy as np
import torch

from . import _lib, ops
from .array import Array
from .fit import random_guess_host
from .linalg import norm as _norm
from .mpo_compress import (_cp, _direct_sweep, _flip, _flip_mps, _prepare,
                           mps_gate_with_mpo)
from .split import array_split

METHODS = ("src", "src-oversample", "src-first", "srcmps", "srcmps-oversample",
           "srcmps-first", "sdc", "sdc-oversample")
_ALIAS = {"src-first": "src-oversample", "srcmps-first": "srcmps-oversample"}
NOISE_MODES = ("joint", "separable", "symmetric")


# ------------------------------------------------------------- the kernel ---
def sketch_env(LE, W, Om):
    """H[B, a, u, p] = sum_{v, o} LE[B, a, v] W[v, u, o, p] Om[B, o] through
    ``qb_sketch_env``: torch tensors of one dtype (float32, float64,
    complex64 or complex128), any strides; returns a new contiguous H."""
    if not (LE.dtype == W.dtype == Om.dtype):
        raise TypeError(f"sketch_env: dtypes {LE.dtype}, {W.dtype}, {Om.dtype} differ")
    nB, na, nv = LE.shape
    nv2, nu, no, np_ = W.shape
    if nv2 != nv or tuple(Om.shape) != (nB, no):
        raise ValueError(f"sketch_env: LE {tuple(LE.shape)}, W {tuple(W.shape)} and Omega "
                         f"{tuple(Om.shape)} do not fit")
    H = torch.empty((nB, na, nu, np_), dtype=LE.dtype, device=LE.device)
    st = [(ctypes.c_int64 * x.dim())(*x.stride()) for x in (LE, W, Om, H)]
    rc = _lib.load().qb_sketch_env(_lib.qb_dtype(LE.dtype), nB, na, nv, nu, no, np_,
                                   LE.data_ptr(), st[0], W.data_ptr(), st[1], Om.data_ptr(),
                                   st[2], H.data_ptr(), st[3], _lib.stream_ptr())
    _lib.check(rc, "qb_sketch_env")
    return H


def _plain(x):
    """The torch tensor of an Array with any lazy conjugation applied."""
    return ops.materialize(x).t if x.cj else x.t


# ------------------------------------------------------- host control logic ---
def oversample_bond(max_bond, max_bond_oversample):
    """The intermediate bond of the '-oversample' methods (compress.py:1954-
    1962): ``max(round(1.5 max_bond), max_bond + 10)`` by default, a float
    multiplies ``max_bond``, an int is taken as given."""
    if max_bond_oversample is None:
        mbo = max(round(1.5 * max_bond), max_bond + 10)
    elif isinstance(max_bond_oversample, float):
        mbo = round(max_bond * max_bond_oversample)
    else:
        mbo = int(max_bond_oversample)
    if mbo < 1:
        raise ValueError(f"mps_gate_with_mpo_successive: max_bond_oversample resolves to "
                         f"{mbo}, it must be at least 1")
    return mbo


def noise_host(rng, k, d, dist):
    """One site's SRC noise, Omega[B, o] of shape (k, d), by the rule of
    ``random.array`` (compress.py:1283: float64, drawn from ``rng``, or from
    a fresh seed of numpy's global state when ``rng`` is None)."""
    from . import _random_host
    return _random_host((k, d), dist=dist, rng=rng)


def _rng(seed):
    """``random.default_rng(seed)`` as compress.py:1766-1770: None keeps the
    global state (a fresh seed per draw)."""
    if seed is None:
        return None
    from . import random
    return random.default_rng(seed)._rng


# ------------------------------------------------------ left environments ---
def _unit(dt, device, k=1):
    """LE[B, a, v] = 1 for a chain's first site, k samples (stride 0)."""
    return ops.ones((1, 1, 1), dtype=dt, device=device).t.expand(k, 1, 1)


def _envs_src(A, W, k, rng, dist):
    """LE[i][B, b, u] for i = 1 .. L-1: site i - 1's noise drawn, in site
    order, cast and uploaded once; one sketch launch and one GEMM per site."""
    L = len(A)
    dt = A[0].dtype
    envs = [None] * L
    LE = _unit(A[0].t.dtype, A[0].t.device, k)
    for i in range(1, L):
        s = i - 1
        om = ops.asarray(noise_host(rng, k, W[s].shape[2], dist).astype(dt)).t
        H = Array(sketch_env(LE, _plain(W[s]), om))                     # [B, a, u, p]
        E = _cp(H, [0, 1, 2, 3], A[s], [1, 3, 4], [0, 4, 2])              # [B, b, u]
        envs[i] = E
        LE = E.t
    return envs


def _envs_srcmps(A, W, F):
    """LE[i][g, b, u]: the ladder closed with the sampling MPS F[f, o, g],
    not conjugated (compress.py:2138-2161)."""
    L = len(A)
    envs = [None] * L
    E = Array(_unit(A[0].t.dtype, A[0].t.device))
    for i in range(1, L):
        s = i - 1
        X = _cp(E, [0, 1, 2], A[s], [1, 3, 4], [0, 2, 3, 4])             # [f, v, p, b]
        Y = _cp(X, [0, 1, 2, 3], W[s], [1, 5, 6, 2], [0, 3, 5, 6])       # [f, b, u, o]
        E = _cp(Y, [0, 1, 2, 3], F[s], [0, 3, 7], [7, 1, 2])             # [g, b, u]
        envs[i] = E
    return envs


def _envs_sdc(A, W, copts):
    """LE[i][n, b, u] = (s VH) of the split t[(x, o), (b, u)] of the previous
    environment closed with site i - 1 (compress.py:1449-1487)."""
    L = len(A)
    envs = [None] * L
    E = Array(_unit(A[0].t.dtype, A[0].t.device))
    for i in range(L - 1):
        X = _cp(E, [0, 1, 2], A[i], [1, 3, 4], [0, 2, 3, 4])             # [x, v, p, b]
        t = _cp(X, [0, 1, 2, 3], W[i], [1, 5, 6, 2], [0, 6, 3, 5])       # [x, o, b, u]
        x, o, b, u = t.shape
        _, _, right = array_split(t.reshape(x * o, b * u), **copts)
        E = ops.materialize(right).reshape(right.shape[0], b, u)
        envs[i + 1] = E
    return envs


# ------------------------------------------------------------------ sweep ---
def _sweep(A, W, envs, popts):
    """_do_sweep_compress_from_low_rank_left_envs: from the right, the sketch
    t[o, k, x] = C[a, v, o, k] LE[x, a, v] with C = A W RE, its QR isometry
    Q[(o, k), n] the new site, and RE'[a, v, n] = C . conj(Q) (the flag, no
    conjugated copy).  Returns sites right-canonical around 0."""
    L = len(A)
    out = [None] * L
    R = ops.ones((1, 1, 1), dtype=A[0].dtype, device=A[0].device)        # R[b, u, k]
    for i in range(L - 1, -1, -1):
        T = _cp(A[i], [0, 1, 2], R, [2, 3, 4], [0, 1, 3, 4])             # [a, p, u, k]
        C = _cp(T, [0, 1, 3, 4], W[i], [5, 3, 6, 1], [0, 5, 6, 4])       # [a, v, o, k]
        if i == 0:
            la, lw, o, k = C.shape
            out[0] = C.reshape(la * lw, o, k)
            break
        t = _cp(C, [0, 1, 2, 3], envs[i], [4, 0, 1], [2, 3, 4])          # [o, k, x]
        o, k, x = t.shape
        Q, _, _ = array_split(t.reshape(o * k, x), **popts)
        n = Q.shape[1]
        Q = ops.materialize(Q).reshape(o, k, n)
        out[i] = Q.transpose(2, 0, 1)
        R = _cp(C, [0, 1, 2, 3], Q.conj(), [2, 3, 4], [0, 1, 4])         # [a, v, n]
    return out


def _src(A, W, k, rev, popts, rng, dist):
    if rev:
        A, W = _flip(A, W)
    out = _sweep(A, W, _envs_src(A, W, k, rng, dist), popts)
    return _flip_mps(out) if rev else out


def _srcmps(A, W, F, rev, popts):
    if rev:
        A, W = _flip(A, W)
        F = _flip_mps(F)
    out = _sweep(A, W, _envs_srcmps(A, W, F), popts)
    return _flip_mps(out) if rev else out


def _sdc(A, W, rev, copts, popts):
    if rev:
        A, W = _flip(A, W)
    out = _sweep(A, W, _envs_sdc(A, W, copts), popts)
    return _flip_mps(out) if rev else out


def _sampling_mps(sites, mpo, A, W, dt, tn_fit, max_bond, cutoff, seed, sweep_reverse,
                  transpose, mpo_shape):
    """The sampling MPS of 'srcmps' in natural site order (compress.py:2119-
    2135): given sites, a method (string / dict) of ``mps_gate_with_mpo``,
    or None: this project's random draw (``fit.random_guess_host``)."""
    L = len(A)
    if tn_fit is None:
        if max_bond is None:
            raise ValueError("mps_gate_with_mpo_successive: `max_bond` must be given for "
                             "the `srcmps` method")
        F = [ops.asarray(x) for x in
             random_guess_host([w.shape[2] for w in W], max_bond, dt, seed)]
    elif isinstance(tn_fit, (str, dict)):
        opts = {"method": tn_fit} if isinstance(tn_fit, str) else dict(tn_fit)
        opts.setdefault("max_bond", max_bond)
        opts.setdefault("cutoff", cutoff)
        opts.setdefault("sweep_reverse", sweep_reverse)
        opts.setdefault("transpose", transpose)
        opts.setdefault("mpo_shape", mpo_shape)
        F = mps_gate_with_mpo(sites, mpo, **opts)
    else:
        F = [ops.asarray(f) for f in tn_fit]
        if len(F) != L or any(f.ndim != 3 for f in F):
            raise ValueError("mps_gate_with_mpo_successive: `tn_fit` must be a list of "
                             f"{L} (l, p, r) sites")
        for i, f in enumerate(F):
            if f.shape[1] != W[i].shape[2] or (i and F[i - 1].shape[2] != f.shape[0]):
                raise ValueError(f"mps_gate_with_mpo_successive: `tn_fit` site {i} does not "
                                 "fit the output of the ladder")
        if F[0].shape[0] != 1 or F[-1].shape[2] != 1:
            raise ValueError("mps_gate_with_mpo_successive: `tn_fit` must have open "
                             "boundaries")
    return F


# ------------------------------------------------------------------ driver ---
def mps_gate_with_mpo_successive(sites, mpo, max_bond, method="src", cutoff=None,
                                 cutoff_mode="rsum2", max_bond_oversample=None,
                                 cutoff_oversample=0.0, noise_mode="joint",
                                 noise_dist="normal", seed=None, tn_fit=None, normalize=False,
                                 sweep_reverse=False, canonize=True, transpose=False,
                                 mpo_shape="lrud", project_opts=None, compress_opts=None,
                                 info=None, equalize_norms=False, **kwargs):
    """``MatrixProductState.gate_with_mpo(mpo, method=...)`` for the
    successive-compression methods of quimb (tn1d/compress.py:1115-2339),
    for open-boundary (l, p, r) device sites:

      'src'               successive randomized compression: left
                          environments sketched with ``max_bond`` Gaussian
                          (``noise_dist``) samples, one QR per site
      'srcmps'            the same with an MPS as the sampling noise:
                          ``tn_fit`` sites, a :func:`mps_gate_with_mpo`
                          method (string or dict), or None for a random MPS
                          of bond ``max_bond`` drawn by
                          ``fit.random_guess_host(seed)``
      'sdc'               successive deterministic compression: left
                          environments truncated by SVD (``max_bond``,
                          ``cutoff`` default 1e-10, ``cutoff_mode``,
                          ``compress_opts``; absorb='rfactor')
      '<m>-oversample'    <m> to ``max_bond_oversample`` (default
                          max(round(1.5 max_bond), max_bond + 10); a float
                          multiplies max_bond) from the other end, then one
                          direct sweep to ``max_bond`` / ``cutoff`` (default
                          1e-10) with ``compress_opts``; 'src-first' and
                          'srcmps-first' are aliases

    ``max_bond`` is required except for 'sdc' and for 'srcmps' with given
    ``tn_fit`` sites.  ``seed`` (int, Generator or None for numpy's global
    state) fixes the SRC noise, one (max_bond, d) block per site in sweep
    order; the three ``noise_mode``s draw the same noise on a ladder.
    ``project_opts`` go to every QR (default method='qr', absorb='lorthog').
    Options the reference ignores warn as it does ('src' / 'srcmps':
    ``cutoff``, ``compress_opts``; every method: ``canonize=False``); extra
    keywords join ``compress_opts`` for the methods that truncate and raise
    ``TypeError`` for 'src' / 'srcmps'.  ``mpo``, ``transpose`` and
    ``mpo_shape`` as in :func:`mps_gate_with_mpo`.

    Returns a new list of (l, p, r) device Arrays in the promoted dtype,
    right-canonical with the centre at site 0 (left-canonical at L - 1 with
    ``sweep_reverse``); ``normalize`` scales the centre to unit norm and
    ``info["cur_orthog"]`` receives it.  The caller's arrays are not
    modified."""
    if method not in METHODS:
        raise ValueError(f"mps_gate_with_mpo_successive: unknown method {method!r} "
                         f"(available: {', '.join(METHODS)})")
    method = _ALIAS.get(method, method)
    if equalize_norms:
        raise NotImplementedError("mps_gate_with_mpo_successive: equalize_norms is not "
                                  "implemented")
    if noise_mode not in NOISE_MODES:
        raise ValueError(f"Unknown noise mode {noise_mode!r}, should be one of "
                         "'separable', 'symmetric', or 'joint'.")
    base = method.split("-")[0]
    oversample = method.endswith("-oversample")
    if cutoff is None:
        cutoff = 1e-10 if (oversample or base == "sdc") else 0.0
    popts = dict(project_opts or {})
    popts.setdefault("method", "qr")
    popts.setdefault("absorb", "lorthog")
    sites, mpo = list(sites), list(mpo)
    A, W, dt = _prepare(sites, mpo, mpo_shape, transpose)
    L = len(A)

    if not canonize:
        # the reference's 'srcmps' warns with the 'src' name
        name = "src" if method == "srcmps" else method
        warnings.warn(f"`canonize=False` is ignored for the `{name}` method.")
    if base in ("src", "srcmps") and not oversample:
        if kwargs:
            raise TypeError(f"mps_gate_with_mpo_successive: method {method!r} takes no "
                            f"option(s) {sorted(kwargs)}")
        if max_bond is None and (base == "src" or tn_fit is None):
            raise ValueError(f"`max_bond` must be given for the `{method}` method.")
        _warn_src(method, cutoff, compress_opts)
        copts = None
    else:
        copts = dict(kwargs, **(compress_opts or {}))
        if oversample and max_bond is None:
            raise ValueError(f"`max_bond` must be given for the `{method}` method.")

    if oversample:
        mbo = oversample_bond(max_bond, max_bond_oversample)
        rev = not sweep_reverse
        if base == "src":
            _warn_src("src", cutoff_oversample, None)
            out = _src(A, W, mbo, rev, popts, _rng(seed), noise_dist)
        elif base == "srcmps":
            _warn_src("srcmps", cutoff_oversample, None)
            F = _sampling_mps(sites, mpo, A, W, dt, tn_fit, mbo, cutoff_oversample, seed,
                              rev, transpose, mpo_shape)
            A, W, F = _promote(A, W, F)
            out = _srcmps(A, W, F, rev, popts)
        else:
            sopts = dict(copts)
            sopts.setdefault("max_bond", mbo)
            sopts.setdefault("cutoff", cutoff_oversample)
            sopts.setdefault("cutoff_mode", cutoff_mode)
            sopts.setdefault("absorb", "rfactor")
            out = _sdc(A, W, rev, sopts, popts)
        dopts = dict(copts)
        dopts.setdefault("max_bond", max_bond)
        dopts.setdefault("cutoff", cutoff)
        dopts.setdefault("cutoff_mode", cutoff_mode)
        if sweep_reverse:
            out = _flip_mps(out)
        _direct_sweep(out, dopts)
        if sweep_reverse:
            out = _flip_mps(out)
    elif base == "src":
        out = _src(A, W, max_bond, sweep_reverse, popts, _rng(seed), noise_dist)
    elif base == "srcmps":
        F = _sampling_mps(sites, mpo, A, W, dt, tn_fit, max_bond, cutoff, seed, sweep_reverse,
                          transpose, mpo_shape)
        A, W, F = _promote(A, W, F)
        out = _srcmps(A, W, F, sweep_reverse, popts)
    else:
        copts.setdefault("max_bond", max_bond)
        copts.setdefault("cutoff", cutoff)
        copts.setdefault("cutoff_mode", cutoff_mode)
        copts.setdefault("absorb", "rfactor")
        out = _sdc(A, W, sweep_reverse, copts, popts)

    c = L - 1 if sweep_reverse else 0
    if normalize:
        x = ops.materialize(out[c], force=True)
        out[c] = ops.scale_(x, 1.0, div_by=_norm(x))
    out = [ops.materialize(x) for x in out]
    if info is not None:
        info["cur_orthog"] = (c, c)
    return out


def _promote(A, W, F):
    """One dtype for the ladder and the sampling MPS."""
    dt = np.result_type(A[0].dtype, *[f.dtype for f in F])
    return ([a.astype(dt, copy=False) for a in A], [w.astype(dt, copy=False) for w in W],
            [f.astype(dt, copy=False) for f in F])


def _warn_src(method, cutoff, compress_opts):
    if cutoff != 0.0:
        warnings.warn(f"`cutoff` is ignored for the `{method}` method, use `max_bond` "
                      "instead.")
    if compress_opts:
        warnings.warn(f"`compress_opts` is ignored for the `{method}` method, since there "
                      "is no final compression step, see `project_opts` instead.")
