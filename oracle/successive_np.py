"""numpy restatement of the successive-compression methods of
quimb_b200/successive.py ('src', 'srcmps', 'sdc' and their '-oversample'
variants; quimb/tensor/tn1d/compress.py:1115-2339) for (l, p, r) site lists
and (l, r, u, d) MPO sites.  Splits are those of oracle/decomp_np.py and
the direct sweep that of oracle/mpo_compress_np.py.

The noise is restated here: for each site in sweep order but the last, a
float64 (k, d) block drawn from ``numpy.random.default_rng(seed)`` by
``noise_dist`` -- standard normal, uniform on [-1, 1) or a choice of +-1.
"""

import numpy as np

from oracle import decomp_np as dnp
from oracle import mpo_compress_np as mnp


def noise(rng, k, d, dist):
    if dist == "normal":
        return rng.standard_normal((k, d))
    if dist == "uniform":
        return rng.uniform(-1.0, 1.0, size=(k, d))
    if dist == "rademacher":
        return rng.choice([-1.0, 1.0], size=(k, d))
    raise ValueError(dist)


def oversample_bond(max_bond, mbo):
    if mbo is None:
        return max(round(1.5 * max_bond), max_bond + 10)
    if isinstance(mbo, float):
        return round(max_bond * mbo)
    return int(mbo)


def _record(cuts, mat, kept):
    """A truncating split's singular values and kept rank."""
    if cuts is not None:
        cuts.append((np.linalg.svd(mat, compute_uv=False), kept))


# ------------------------------------------------------ left environments ---
def envs_src(A, W, k, rng, dist):
    L = len(A)
    envs = [None] * L
    E = np.ones((k, 1, 1), dtype=A[0].dtype)                         # [B, a, v]
    for i in range(1, L):
        om = noise(rng, k, W[i - 1].shape[2], dist).astype(A[0].dtype)
        E = np.einsum("Bav,apb,vuop,Bo->Bbu", E, A[i - 1], W[i - 1], om, optimize=True)
        envs[i] = E
    return envs


def envs_srcmps(A, W, F):
    L = len(A)
    envs = [None] * L
    E = np.ones((1, 1, 1), dtype=A[0].dtype)
    for i in range(1, L):
        X = np.einsum("fav,apb->fvpb", E, A[i - 1], optimize=True)
        X = np.einsum("fvpb,vuop->fbuo", X, W[i - 1], optimize=True)
        E = np.einsum("fbuo,fog->gbu", X, F[i - 1], optimize=True)
        envs[i] = E
    return envs


def envs_sdc(A, W, opts, cuts=None):
    L = len(A)
    envs = [None] * L
    E = np.ones((1, 1, 1), dtype=A[0].dtype)
    for i in range(L - 1):
        t = np.einsum("xav,apb,vuop->xobu", E, A[i], W[i], optimize=True)
        x, o, b, u = t.shape
        mat = t.reshape(x * o, b * u)
        _, _, right = mnp._split(mat, absorb="rfactor", **opts)
        _record(cuts, mat, right.shape[0])
        E = right.reshape(-1, b, u)
        envs[i + 1] = E
    return envs


# ------------------------------------------------------------------ sweep ---
def sweep(A, W, envs, sketches=None):
    """From the right: t[(o, k), x] = LE A W RE, Q of its QR the new site,
    RE' = A W RE conj(Q).  ``sketches``: a list receiving the singular
    values of every t (a rank-deficient sketch leaves Q undetermined)."""
    L = len(A)
    out = [None] * L
    R = np.ones((1, 1, 1), dtype=A[0].dtype)                         # [b, u, k]
    for i in range(L - 1, -1, -1):
        C = np.einsum("apb,buk,vuop->avok", A[i], R, W[i], optimize=True)
        if i == 0:
            out[0] = C.reshape(-1, C.shape[2], C.shape[3])
            break
        t = np.einsum("avok,xav->okx", C, envs[i], optimize=True)
        o, k, x = t.shape
        if sketches is not None:
            if isinstance(sketches, np.random.Generator):
                # a relative 1e-12 perturbation: a well-posed sketch does not
                # care, a rank-deficient one leaves Q to rounding
                t = t + 1e-12 * np.max(np.abs(t)) * sketches.standard_normal(t.shape)
            else:
                sketches.append(np.linalg.svd(t.reshape(o * k, x), compute_uv=False))
        Q, _, _ = dnp.qr_stabilized(t.reshape(o * k, x), absorb="lorthog")
        Q = Q.reshape(o, k, -1)
        out[i] = Q.transpose(2, 0, 1)
        R = np.einsum("avok,okn->avn", C, Q.conj(), optimize=True)
    return out


def _oriented(fn, A, W, rev, *extra):
    if rev:
        A, W = mnp._flip(A, W)
    out = fn(A, W, *extra)
    return mnp._flip_mps(out) if rev else out


def _direct_sweep(out, opts, cuts):
    """mpo_compress_np._direct_sweep with every cut recorded."""
    for i in range(len(out) - 1, 0, -1):
        l, d, r = out[i].shape
        mat = out[i].reshape(l, d * r)
        tc, _, nb = mnp._split(mat, **opts)
        _record(cuts, mat, nb.shape[0])
        out[i] = nb.reshape(-1, d, r)
        out[i - 1] = np.tensordot(out[i - 1], tc, axes=(2, 0))


def gate_with_mpo_successive(sites, mpo, max_bond, method="src", cutoff=None,
                             cutoff_mode="rsum2", max_bond_oversample=None,
                             cutoff_oversample=0.0, noise_dist="normal", seed=None, tn_fit=None,
                             normalize=False, sweep_reverse=False, transpose=False,
                             cuts=None, sketches=None, **_ignored):
    """Host arrays in, host arrays out.  ``seed``: an int or a numpy
    Generator (the oracle has no global-state draw); ``tn_fit``: the
    sampling MPS sites of 'srcmps'; ``cuts``: a list receiving (singular
    values, kept rank) of every truncating split."""
    method = {"src-first": "src-oversample", "srcmps-first": "srcmps-oversample"}.get(
        method, method)
    base = method.split("-")[0]
    over = method.endswith("-oversample")
    if cutoff is None:
        cutoff = 1e-10 if over or base == "sdc" else 0.0
    A, W = mnp._prepare(sites, mpo, transpose)
    if tn_fit is not None:
        dt = np.result_type(A[0].dtype, *[np.asarray(f).dtype for f in tn_fit])
        A, W = [a.astype(dt) for a in A], [w.astype(dt) for w in W]
        F = [np.asarray(f).astype(dt) for f in tn_fit]
    rng = np.random.default_rng(seed)
    k = oversample_bond(max_bond, max_bond_oversample) if over else max_bond
    rev = (not sweep_reverse) if over else sweep_reverse
    sk = sketches
    inner_cut = cutoff_oversample if over else cutoff
    if base == "src":
        if rev:
            A2, W2 = mnp._flip(A, W)
        else:
            A2, W2 = A, W
        out = sweep(A2, W2, envs_src(A2, W2, k, rng, noise_dist), sk)
        out = mnp._flip_mps(out) if rev else out
    elif base == "srcmps":
        Fo = mnp._flip_mps(F) if rev else F
        out = _oriented(lambda a, w: sweep(a, w, envs_srcmps(a, w, Fo), sk), A, W, rev)
    else:
        opts = dict(max_bond=k, cutoff=inner_cut, cutoff_mode=cutoff_mode)
        out = _oriented(lambda a, w: sweep(a, w, envs_sdc(a, w, opts, cuts), sk), A, W, rev)
    if over:
        opts = dict(max_bond=max_bond, cutoff=cutoff, cutoff_mode=cutoff_mode)
        out = mnp._flip_mps(out) if sweep_reverse else out
        _direct_sweep(out, opts, cuts)
        out = mnp._flip_mps(out) if sweep_reverse else out
    if normalize:
        c = len(out) - 1 if sweep_reverse else 0
        out[c] = out[c] / np.linalg.norm(out[c])
    return [np.ascontiguousarray(x) for x in out]


dense = mnp.dense
schmidt_values = mnp.schmidt_values
