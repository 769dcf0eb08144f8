"""numpy restatement of the variational 1D fit of quimb_b200/fit.py
(``tensor_network_1d_compress_fit``, tn1d/compress.py:2345-2966) for (l, p, r)
site lists: one- and two-site sweeps fitting an MPS to a sum of targets, each
an MPS or an MPO (l, r, u, d) applied to an MPS.  Splits and QRs are those of
oracle/decomp_np.py; the random start is ``quimb_b200.fit.random_guess_host``
(host control logic, this project's own draw)."""

import itertools

import numpy as np

from oracle import decomp_np as dnp
from oracle import mpo_compress_np as mnp
from quimb_b200.fit import bond_schedule, choose_bsz, random_guess_host


def _targets(targets, transpose):
    """[("mps", B)] / [("mpo", A, W)] with W as (l, r, o, q): o the output
    index, q the one that meets the MPS."""
    out = []
    for t in targets:
        if isinstance(t, tuple):
            W, A = t
            W = [np.asarray(w) for w in W]
            if transpose:
                W = [w.transpose(0, 1, 3, 2) for w in W]
            out.append(("mpo", [np.asarray(a) for a in A], W))
        else:
            out.append(("mps", [np.asarray(b) for b in t]))
    return out


def _ein(eq, *ops):
    """einsum as pairwise steps, left to right (no outer-product paths)."""
    ins, out = eq.split("->")
    terms = ins.split(",")
    x, tx = ops[0], terms[0]
    for k in range(1, len(ops)):
        rest = set("".join(terms[k + 1:]) + out)
        keep = "".join(c for c in dict.fromkeys(tx + terms[k]) if c in rest)
        x = np.einsum(f"{tx},{terms[k]}->{keep}", x, ops[k])
        tx = keep
    return np.einsum(f"{tx}->{out}", x)


def _left_step(E, F, tgt, i):
    if tgt[0] == "mps":
        return _ein("fa,apb,fpg->gb", E, tgt[1][i], F.conj())
    return _ein("fwa,aqb,wvoq,fog->gvb", E, tgt[1][i], tgt[2][i], F.conj())


def _right_step(R, F, tgt, i):
    if tgt[0] == "mps":
        return _ein("gb,apb,fpg->fa", R, tgt[1][i], F.conj())
    return _ein("gvb,aqb,wvoq,fog->fwa", R, tgt[1][i], tgt[2][i], F.conj())


def _local1(Lk, Rk, tgt, i):
    if tgt[0] == "mps":
        return _ein("fa,apb,gb->fpg", Lk, tgt[1][i], Rk)
    return _ein("fwa,aqb,wvoq,gvb->fog", Lk, tgt[1][i], tgt[2][i], Rk)


def _local2(Lk, Rk, tgt, i):
    if tgt[0] == "mps":
        B = tgt[1]
        return _ein("fa,apb,bsc,gc->fpsg", Lk, B[i], B[i + 1], Rk)
    A, W = tgt[1], tgt[2]
    left = _ein("fwa,aqb,wvoq->fbvo", Lk, A[i], W[i])
    right = _ein("guc,bsc,vuts->gbvt", Rk, A[i + 1], W[i + 1])
    return np.einsum("fbvo,gbvt->fotg", left, right)


def _empty(tgt, dt):
    return np.ones((1, 1) if tgt[0] == "mps" else (1, 1, 1), dtype=dt)


def _distance_normalized(x, y):
    """tensor_network_distance(normalized=True), fitting.py:9-153."""
    xx = abs(np.vdot(x, x))
    yy = abs(np.vdot(y, y))
    xy = np.vdot(x, y).real
    return abs(xx + yy - 2 * xy) ** 0.5 * 2 / (xx ** 0.5 + yy ** 0.5)


def _lq_site(F, i):
    """canonize_between(i, i - 1): LQ of site i, L absorbed into site i - 1."""
    l, d, r = F[i].shape
    Lf, _, Q = dnp.qr_stabilized(F[i].reshape(l, d * r), absorb="left")
    F[i] = Q.reshape(-1, d, r)
    F[i - 1] = np.tensordot(F[i - 1], Lf, axes=(2, 0))


def _qr_site(F, i):
    mnp._left_canonize_site(F, i)


def _expand(F, bond):
    """expand_bond_dimension_(bond) with zeros: every inner bond to at least
    ``bond``."""
    L = len(F)
    out = []
    for i, x in enumerate(F):
        l, d, r = x.shape
        nl = l if i == 0 else max(l, bond)
        nr = r if i == L - 1 else max(r, bond)
        out.append(np.pad(x, ((0, nl - l), (0, 0), (0, nr - r))))
    return out


def _sweep(F, T, bsz, bond, cutoff, envs, prepare, reverse, compute_tdiff, cutoff_mode,
           renorm, spectra):
    N, K = len(F), len(T)
    dt = F[0].dtype
    if bsz == 1 and bond is not None and max(x.shape[2] for x in F) < bond:
        F[:] = _expand(F, bond)
        prepare = True
    if prepare:
        for k in range(K):
            envs["L", 0, k] = _empty(T[k], dt)
            envs["R", N - 1, k] = _empty(T[k], dt)
        last = N - 1 if bsz == 1 else N - 2
        if not reverse:
            for i in range(N - 1, 0, -1):
                _lq_site(F, i)
            for i in range(N - 2, N - 2 - last, -1):
                for k in range(K):
                    envs["R", i, k] = _right_step(envs["R", i + 1, k], F[i + 1], T[k], i + 1)
        else:
            for i in range(N - 1):
                _qr_site(F, i)
            for i in range(1, last + 1):
                for k in range(K):
                    envs["L", i, k] = _left_step(envs["L", i - 1, k], F[i - 1], T[k], i - 1)
    max_tdiff = -1.0
    n_steps = N if bsz == 1 else N - 1
    sweep = range(n_steps)
    if reverse:
        sweep = reversed(sweep)
    for i in sweep:
        if not reverse and i > 0:
            if bsz == 1:
                _qr_site(F, i - 1)
            for k in range(K):
                envs["L", i, k] = _left_step(envs["L", i - 1, k], F[i - 1], T[k], i - 1)
        elif reverse and i < n_steps - 1:
            j = i + bsz
            if bsz == 1:
                _lq_site(F, j)
            for k in range(K):
                envs["R", j - 1, k] = _right_step(envs["R", j, k], F[j], T[k], j)
        if bsz == 1:
            G = sum(_local1(envs["L", i, k], envs["R", i, k], T[k], i) for k in range(K))
            if compute_tdiff:
                max_tdiff = max(max_tdiff, _distance_normalized(F[i], G))
            F[i] = G
            continue
        G = sum(_local2(envs["L", i, k], envs["R", i + 1, k], T[k], i) for k in range(K))
        l, d1, d2, r = G.shape
        m = G.reshape(l * d1, d2 * r)
        if spectra is not None:
            spectra.append((np.linalg.svd(m, compute_uv=False), bond, cutoff, cutoff_mode))
        opts = dnp.parse_truncation_opts(bond, cutoff, cutoff_mode, renorm)
        absorb = dnp.get_Us_VH if reverse else dnp.get_U_sVH
        left, _, right = dnp.svd_truncated(m, absorb=absorb, **opts)
        if compute_tdiff:
            old = np.tensordot(F[i], F[i + 1], axes=(2, 0))
            new = np.tensordot(left, right, axes=(1, 0)).reshape(old.shape)
            max_tdiff = max(max_tdiff, _distance_normalized(old, new))
        F[i] = left.reshape(l, d1, -1)
        F[i + 1] = right.reshape(-1, d2, r)
    return max_tdiff


def fit(targets, max_bond=None, cutoff=None, guess=None, bsz="auto", initial_bond_dim=8,
        max_iterations=10, tol=0.0, cutoff_mode="rsum2", sweep_sequence="RL", seed=None,
        normalize=False, sweep_reverse=False, transpose=False, info=None, spectra=None,
        **compress_opts):
    """tensor_network_1d_compress_fit on host arrays.  ``targets``: a list of
    (l, p, r) MPS site lists and ``(mpo, sites)`` tuples (MPO sites (l, r, u,
    d), size-1 outer bonds at the ends).  ``guess``: None (the random start of
    quimb_b200.fit), an (l, p, r) site list, or 'zipup' / a dict of
    mpo_compress_np.gate_with_mpo options (first target an MPO pair).
    ``spectra``: a list that receives, for every two-site split, the
    block's singular values and the split's (max_bond, cutoff,
    cutoff_mode).  ``info`` also receives ``tdiffs``, every sweep's
    max_tdiff."""
    targets = list(targets)
    T = _targets(targets, transpose)
    dt = np.result_type(*[x for t in T for part in t[1:] for x in part])
    T = [(t[0],) + tuple([x.astype(dt) for x in part] for part in t[1:]) for t in T]
    bsz = choose_bsz(bsz, max_bond, cutoff)
    if cutoff is None:
        cutoff = 1e-10 if bsz == 2 else 0.0
    extra = set(compress_opts) - {"cutoff_mode", "renorm"}
    if extra:
        raise TypeError(f"fit_np: split options {sorted(extra)} are not modelled")
    cutoff_mode = compress_opts.get("cutoff_mode", cutoff_mode)
    renorm = compress_opts.get("renorm")
    L = len(T[0][1])
    t0 = T[0]
    dims = [t0[1][i].shape[1] if t0[0] == "mps" else t0[2][i].shape[2] for i in range(L)]
    if guess is None or isinstance(guess, (str, dict)):
        max_bond, cur = bond_schedule(max_bond, initial_bond_dim, max_iterations, bsz,
                                      random=guess is None)
        if guess is None:
            F = [x.astype(dt) for x in random_guess_host(dims, cur, dt, seed)]
        else:
            gopts = {"method": guess} if isinstance(guess, str) else dict(guess)
            gopts.setdefault("max_bond", cur)
            gopts.setdefault("cutoff", cutoff)
            W, A = targets[0]
            F = [x.astype(dt) for x in mnp.gate_with_mpo(A, W, transpose=transpose, **gopts)]
    else:
        F = [np.array(x, dtype=dt) for x in guess]
        cur = max([x.shape[2] for x in F[:-1]], default=1)
        if max_bond is None:
            max_bond = cur
    compute_tdiff = tol != 0.0
    envs, old, tdiffs = {}, "", []
    sweeps = itertools.cycle(sweep_sequence)
    reverse, n, max_tdiff = None, 0, -1.0
    for it in range(max_iterations):
        direction = next(sweeps)
        reverse = {"R": False, "L": True}[direction] != sweep_reverse
        if cur < max_bond:
            cur = min(2 * cur, max_bond)
        max_tdiff = _sweep(F, T, bsz, None if cur == float("inf") else cur, cutoff, envs,
                           it == 0 or direction == old, reverse, compute_tdiff, cutoff_mode,
                           renorm, spectra)
        n += 1
        tdiffs.append(max_tdiff)
        if tol != 0.0 and max_tdiff < tol:
            break
        old = direction
    c = 0 if reverse else L - 1
    if normalize:
        F[c] = F[c] / np.linalg.norm(F[c])
    if info is not None:
        info.update(cur_orthog=(c, c), sweeps=n, max_tdiff=max_tdiff, tdiffs=tdiffs)
    return [np.ascontiguousarray(x) for x in F]


dense = mnp.dense
schmidt_values = mnp.schmidt_values


def target_dense(targets, transpose=False):
    """The exact sum of the targets as a dense vector."""
    v = 0
    for t in _targets(list(targets), transpose):
        sites = t[1] if t[0] == "mps" else [mnp._product(a, w) for a, w in zip(t[1], t[2])]
        v = v + dense(sites)
    return v


def fidelity(x, y):
    """|<x|y>|^2 / (<x|x> <y|y>) of two dense vectors."""
    return abs(np.vdot(x, y)) ** 2 / (np.vdot(x, x).real * np.vdot(y, y).real)


def check_svd_margin(s, max_bond, cutoff, cutoff_mode):
    """A two-site truncation (singular values ``s``, descending) is decided far
    from the device SVD's absolute noise, 1e3 eps s_0: every kept value lies
    above it, and the cut falls in a gap wider than it (max_bond) or with the
    discarded weight ('rsum2') away from the threshold by more than the noise
    of the whole tail (cutoff)."""
    assert cutoff_mode == "rsum2", cutoff_mode
    noise = 1e3 * np.finfo(np.float64).eps * s[0]
    w = s ** 2
    tail = np.cumsum(w[::-1])[::-1]
    thr = cutoff * tail[0]
    n = int(np.argmax(np.append(tail, 0.0) <= thr)) if cutoff > 0 else s.size
    n = max(1, min(n, s.size if max_bond is None else max_bond))
    assert s[n - 1] > noise, (n, s[n - 1], noise)
    if n == s.size or s[n] <= noise:
        return
    if max_bond is not None and n == max_bond and not (cutoff > 0 and tail[n] <= thr):
        assert s[n - 1] - s[n] > noise, (n, s[n - 1] - s[n], noise)
    else:
        margin = 2 * noise * s[0] * s.size
        assert abs(tail[n] - thr) > margin and abs(tail[n - 1] - thr) > margin, (n, margin)


def check_tol_margin(tdiffs, tol):
    """Each sweep's stopping decision is far from the convergence measure's
    precision (about sqrt(eps))."""
    if tol:
        for t in tdiffs:
            assert abs(t - tol) > 1e-3 * tol and abs(t - tol) > 1e-7, (t, tol)
