"""Fit an MPS to a sum of MPSs and MPO-applied MPSs on the device: the one-
and two-site variational ('DMRG-style') compression.

Mirrors, at array level and for open-boundary (l, p, r) site lists,

  tensor_network_1d_compress_fit     tn1d/compress.py:2618-2966
    _tn1d_fit_sum_sweep_1site        tn1d/compress.py:2345-2474
    _tn1d_fit_sum_sweep_2site        tn1d/compress.py:2477-2615
  mps_gate_with_mpo_fit              tn1d/compress.py:3567-3586

A target is an MPS B[a, p, b] or the ladder of ``mpo_compress``: MPS site
A[a, q, b] under MPO site W[w, v, o, q] (o the output index).  Each target k
keeps its own environments, E[f, a] or E[f, w, a] with f the fitted bond;
the fitted sites enter every contraction through the conjugation flag, so no
conjugated copy is made.  An environment step and a local tensor share their
first launches (the target site absorbed into the environment, A before W so
that nothing wider than chi^2 D_w d is formed); that partial is kept from the
local update of one step for the environment update of the next.

Every contraction is one ``contract_pair`` launch; the centre moves are the
device QR (one site) or the truncated SVD of ``split.array_split`` (two
sites).  Host arithmetic: each split's truncation rule, and the convergence
measure, read back once per sweep when ``tol > 0``.
"""

import itertools
import math

import numpy as np

from . import ops, tebd
from .array import Array
from .contract import contract_pair
from .linalg import norm as _norm
from .mpo_compress import _prepare, mps_gate_with_mpo
from .split import array_split


# ------------------------------------------------------- host control logic ---
def choose_bsz(bsz, max_bond, cutoff):
    """The block size by compress.py:2779-2797."""
    if bsz == "auto":
        if max_bond is not None:
            return 1 if cutoff is None or cutoff == 0.0 else 2
        return 1 if cutoff == 0.0 else 2
    if bsz not in (1, 2):
        raise ValueError(f"mps_fit: bsz must be 'auto', 1 or 2, not {bsz!r}")
    return bsz


def bond_schedule(max_bond, initial_bond_dim, max_iterations, bsz, random):
    """``(max_bond, current bond)`` before the first sweep when the start is
    generated, not given (compress.py:2809-2834): no larger than max_bond, and
    large enough that doubling once per sweep reaches it.  ``max_bond`` None
    (two-site only) becomes infinite."""
    if max_bond is None:
        if bsz == 1:
            raise ValueError("mps_fit: need at least one of `max_bond` or an explicit "
                             "guess when using 1-site sweeping")
        return math.inf, initial_bond_dim
    cur = min(initial_bond_dim, max_bond)
    n = 2 ** max_iterations
    cur = max(cur, max_bond // n + bool(max_bond % n))
    if random and max_iterations <= 1:
        cur = max_bond
    return max_bond, cur


def random_guess_host(dims, bond, dtype, seed):
    """This project's random start: host arrays of shape (bond, d_i, bond),
    without the outer bond at the ends (``TN_matching``'s shapes), drawn in
    site order from ``numpy.random.default_rng(seed)`` -- a standard normal
    real part, then for complex dtypes an imaginary part -- and scaled by
    1 / sqrt(l d) so that the state's norm stays of order one at any length."""
    rng = np.random.default_rng(seed)
    L = len(dims)
    cplx = np.dtype(dtype).kind == "c"
    out = []
    for i, d in enumerate(dims):
        shape = (1 if i == 0 else bond, d, 1 if i == L - 1 else bond)
        x = rng.standard_normal(shape)
        if cplx:
            x = x + 1j * rng.standard_normal(shape)
        out.append((x / math.sqrt(shape[0] * d)).astype(dtype))
    return out


def _host_read(t):
    """The one device->host read of a sweep's convergence measure."""
    return t.cpu().numpy()


def _distance_normalized(xx, yy, xy):
    """tensor_network_distance(normalized=True), fitting.py:121-153."""
    xx, yy, xy = np.abs(xx), np.abs(yy), np.real(xy)
    return np.abs(xx + yy - 2 * xy) ** 0.5 * 2 / (xx ** 0.5 + yy ** 0.5)


# ---------------------------------------------------------------- targets ---
def _is_site(x):
    return hasattr(x, "shape")


def _split_targets(targets):
    """One target or a list of them: a bare (l, p, r) site list, a tuple
    ``(mpo, sites)``, or a list of those."""
    if isinstance(targets, tuple) and len(targets) == 2 and not _is_site(targets[0]):
        return [targets]
    targets = list(targets)
    if not targets:
        raise ValueError("mps_fit: no targets")
    if _is_site(targets[0]):
        return [targets]
    return targets


def _prepare_mps(sites):
    B = [ops.asarray(b) for b in sites]
    if not B:
        raise ValueError("mps_fit: empty MPS")
    for b in B:
        if b.ndim != 3:
            raise ValueError("mps_fit: sites must be (l, p, r) arrays")
        if np.dtype(b.dtype).kind not in "fc":
            raise TypeError(f"mps_fit: unsupported dtype {b.dtype}")
    if B[0].shape[0] != 1 or B[-1].shape[2] != 1:
        raise ValueError("mps_fit: open boundaries only (first left and last right bond "
                         "of dimension 1)")
    for i in range(1, len(B)):
        if B[i - 1].shape[2] != B[i].shape[0]:
            raise ValueError(f"mps_fit: bond mismatch between sites {i - 1} and {i}")
    return B


class _Target:
    """One term of the sum: ``W`` None for an MPS.  Sites are views of the
    caller's arrays in the common dtype; ``flip`` reads the chain from the
    right, so right environments are left environments of the flipped
    chain."""

    def __init__(self, A, W):
        self.A, self.W = A, W

    def flip(self):
        A = [a.transpose(2, 1, 0) for a in reversed(self.A)]
        W = None if self.W is None else [w.transpose(1, 0, 2, 3) for w in reversed(self.W)]
        return _Target(A, W)

    def dims(self):
        return [a.shape[1] for a in self.A] if self.W is None else [w.shape[2] for w in self.W]

    def empty(self):
        shape = (1, 1) if self.W is None else (1, 1, 1)
        return Array(ops.ones(shape, dtype=self.A[0].dtype, device=self.A[0].device).t)

    def absorb(self, E, i):
        """The target's site i absorbed into the environment E left of it:
        P[f, p, b] (MPS) or P[f, b, v, o] (MPO)."""
        if self.W is None:
            return _cp(E, [0, 1], self.A[i], [1, 2, 3], [0, 2, 3])
        T = _cp(E, [0, 1, 2], self.A[i], [2, 3, 4], [0, 1, 3, 4])            # [f, w, q, b]
        return _cp(T, [0, 1, 3, 4], self.W[i], [1, 5, 6, 3], [0, 4, 5, 6])    # [f, b, v, o]

    def close_env(self, P, F):
        """The environment right of the site: P closed with the fitted site
        F[f, o, g], conjugated."""
        if self.W is None:
            return _cp(F, [0, 2, 4], P, [0, 2, 3], [4, 3], ca=True)          # [g, b]
        return _cp(P, [0, 4, 5, 6], F, [0, 6, 7], [7, 5, 4], cb=True)        # [g, v, b]

    def close1(self, P, R, out, flipped=False):
        """The one-site local tensor G[f, o, g] = P . R, added to ``out``;
        ``flipped``: P was made on the flipped chain, so G[g, o, f] is
        written."""
        if self.W is None:
            return _cp(P, [0, 2, 3], R, [4, 3], [4, 2, 0] if flipped else [0, 2, 4], out=out)
        return _cp(P, [0, 4, 5, 6], R, [7, 5, 4], [7, 6, 0] if flipped else [0, 6, 7], out=out)

    def close2(self, P, Q, out):
        """The two-site local tensor G[f, o, o', g] from the left partial P of
        site i and the right partial Q of site i + 1 (read from the right)."""
        if self.W is None:
            return _cp(P, [0, 1, 2], Q, [3, 4, 2], [0, 1, 4, 3], out=out)
        return _cp(P, [0, 1, 2, 3], Q, [4, 1, 2, 5], [0, 3, 5, 4], out=out)


def _cp(a, la, b, lb, lc, ca=False, cb=False, out=None):
    """One launch; ``out`` given: accumulate into it (beta = 1)."""
    if out is None:
        return Array(contract_pair(a.t, la, b.t, lb, lc, conj_a=a.cj != ca, conj_b=b.cj != cb))
    contract_pair(a.t, la, b.t, lb, lc, conj_a=a.cj != ca, conj_b=b.cj != cb, out=out.t,
                  beta=1.0)
    return out


def _flip_site(x):
    return x.transpose(2, 1, 0)


# ------------------------------------------------------------------ sweeps ---
class _Fit:
    """The fitted sites, the targets and their environments.  ``envs[k]``
    maps ('L', i) / ('R', i) to target k's environment left / right of site
    i, exactly the reference's ``envs`` dictionary."""

    def __init__(self, F, targets):
        self.F = F
        self.T = targets
        self.Tf = [t.flip() for t in targets]
        self.envs = [{} for _ in targets]
        self.N = len(F)

    # target site i absorbed into its environment from the left / the right
    def _left_partials(self, i):
        return [t.absorb(e["L", i], i) for t, e in zip(self.T, self.envs)]

    def _right_partials(self, i):
        N = self.N
        return [t.absorb(e["R", i], N - 1 - i) for t, e in zip(self.Tf, self.envs)]

    def _set_left(self, i, P):
        """envs[L, i] from the partials of site i - 1."""
        for t, e, p in zip(self.T, self.envs, P):
            e["L", i] = t.close_env(p, self.F[i - 1])

    def _set_right(self, i, Q):
        """envs[R, i] from the partials of site i + 1."""
        for t, e, q in zip(self.Tf, self.envs, Q):
            e["R", i] = t.close_env(q, _flip_site(self.F[i + 1]))

    def prepare(self, reverse, bsz):
        """compress.py:2384-2406 / 2499-2521: the centre to the starting end
        (the QR moves of ``canonize_around_`` on a chain), then every
        environment the sweep reads before it makes its own."""
        N = self.N
        for t, e in zip(self.T, self.envs):
            e["L", 0] = t.empty()
            e["R", N - 1] = t.empty()
        last = N - 1 if bsz == 1 else N - 2
        if not reverse:
            tebd.right_canonize(self.F)
            for i in range(N - 2, N - 2 - last, -1):
                self._set_right(i, self._right_partials(i + 1))
        else:
            tebd.left_canonize(self.F)
            for i in range(1, last + 1):
                self._set_left(i, self._left_partials(i - 1))

    def expand(self, bond):
        """expand_bond_dimension_ with zeros: every inner bond to at least
        ``bond`` (tensor_core.py:10952-11003)."""
        N = self.N
        for i, x in enumerate(self.F):
            l, d, r = x.shape
            nl = l if i == 0 else max(l, bond)
            nr = r if i == N - 1 else max(r, bond)
            if (nl, nr) != (l, r):
                self.F[i] = ops.pad(x, ((0, nl - l), (0, 0), (0, nr - r)))

    def _local(self, P, Q, bsz, flipped=False):
        """The sum over the targets, accumulated in one output."""
        G = None
        for t, p, q in zip(self.T, P, Q):
            G = t.close1(p, q, G, flipped) if bsz == 1 else t.close2(p, q, G)
        return G

    def sweep1(self, reverse, dots):
        """_tn1d_fit_sum_sweep_1site after its preparation."""
        N, F = self.N, self.F
        carry = None
        for i in (reversed(range(N)) if reverse else range(N)):
            if not reverse:
                if i > 0:
                    tebd.left_canonize_site(F, i - 1)
                    self._set_left(i, carry)
                P = self._left_partials(i)
                R = [e["R", i] for e in self.envs]
                G = self._local(P, R, 1)
                carry = P
            else:
                if i < N - 1:
                    tebd.right_canonize_site(F, i + 1)
                    self._set_right(i, carry)
                Q = self._right_partials(i)
                G = self._local(Q, [e["L", i] for e in self.envs], 1, flipped=True)
                carry = Q
            if dots is not None:
                dots += [ops.vdot(F[i], F[i]), ops.vdot(G, G), ops.vdot(F[i], G)]
            F[i] = G

    def sweep2(self, reverse, bond, cutoff, split_opts, dots):
        """_tn1d_fit_sum_sweep_2site after its preparation."""
        N, F = self.N, self.F
        carry = None
        for i in (reversed(range(N - 1)) if reverse else range(N - 1)):
            if not reverse and i > 0:
                self._set_left(i, carry)
            elif reverse and i < N - 2:
                self._set_right(i + 1, carry)
            P = self._left_partials(i)
            Q = self._right_partials(i + 1)
            carry = Q if reverse else P
            G = self._local(P, Q, 2)
            l, d1, d2, r = G.shape
            left, _, right = array_split(G.reshape(l * d1, d2 * r), max_bond=bond,
                                         cutoff=cutoff,
                                         absorb="left" if reverse else "right",
                                         **split_opts)
            k = left.shape[1]
            left = ops.materialize(left).reshape(l, d1, k)
            right = ops.materialize(right).reshape(k, d2, r)
            if dots is not None:
                old = _cp(F[i], [0, 1, 2], F[i + 1], [2, 3, 4], [0, 1, 3, 4])
                new = _cp(left, [0, 1, 2], right, [2, 3, 4], [0, 1, 3, 4])
                dots += [ops.vdot(old, old), ops.vdot(new, new), ops.vdot(old, new)]
            F[i], F[i + 1] = left, right


def _max_tdiff(dots):
    """Largest distance_normalized of one sweep from its device dot products:
    one read for the whole sweep."""
    if not dots:
        return -1.0
    import torch
    x = _host_read(torch.stack([d.t.reshape(()) for d in dots])).reshape(-1, 3)
    return float(np.max(_distance_normalized(x[:, 0], x[:, 1], x[:, 2])))


# ------------------------------------------------------------------ driver ---
def mps_fit(targets, max_bond=None, cutoff=None, guess=None, bsz="auto", initial_bond_dim=8,
            max_iterations=10, tol=0.0, cutoff_mode="rsum2", sweep_sequence="RL", seed=None,
            normalize=False, sweep_reverse=False, mpo_shape="lrud", transpose=False, info=None,
            equalize_norms=False, **compress_opts):
    """``tensor_network_1d_compress_fit`` (tn1d/compress.py:2618-2966) for
    open-boundary (l, p, r) device sites: the MPS of bond dimension at most
    ``max_bond`` closest to the sum of ``targets``, by one-site (``bsz=1``)
    or two-site (``bsz=2``) variational sweeps.

    ``targets``: one target or a list of them; a target is an (l, p, r) site
    list or a tuple ``(mpo, sites)``, the MPO (layout ``mpo_shape``, quimb's
    end tensors accepted) applied to that MPS with the conventions of
    :func:`mps_gate_with_mpo` (``transpose`` contracts the MPO's upper
    index).

    ``guess``: None (a random start, see :func:`random_guess_host`, drawn
    from ``seed``), an (l, p, r) site list used as given (``max_bond``
    defaults to its largest bond), or a method name / dict of
    :func:`mps_gate_with_mpo` options applied to the first target, which
    must then be an ``(mpo, sites)`` pair ('zipup' gives the reference's
    'fit-zipup').  ``bsz='auto'``: one-site when ``max_bond`` is given
    without a cutoff (or when ``cutoff == 0``), else two-site.  ``cutoff``
    defaults to 1e-10 for two-site and must be 0 for one-site sweeps.

    Generated starts begin at ``initial_bond_dim`` (at least max_bond /
    2^max_iterations) and the bond doubles every sweep up to ``max_bond``:
    one-site by zero-padding, two-site through the split.  ``sweep_sequence``
    ('R': left to right) is cycled, ``sweep_reverse`` flips each direction,
    and environments are rebuilt on the first sweep and when the direction
    repeats.  ``tol > 0`` stops once the largest ``distance_normalized``
    between a site's (or pair's) old and new tensor in one sweep falls below
    it.  ``compress_opts`` go to every two-site split (``cutoff_mode``
    defaults to ``cutoff_mode``); one-site sweeps take none.

    Returns a new list of (l, p, r) device Arrays in the promoted dtype of
    the targets, canonical around L - 1 after a left-to-right last sweep and
    around 0 after a right-to-left one; ``normalize`` scales that centre to
    unit norm.  ``info`` receives ``cur_orthog``, ``sweeps`` (sweeps run)
    and ``max_tdiff`` of the last sweep (-1 when not computed).  The
    caller's sites, MPOs and guess are not modified."""
    if equalize_norms:
        raise NotImplementedError("mps_fit: equalize_norms is not implemented")
    if int(max_iterations) < 1:
        raise ValueError("mps_fit: max_iterations must be at least 1")
    if tol < 0:
        raise ValueError("mps_fit: tol must be non-negative")
    if not sweep_sequence or set(sweep_sequence) - {"L", "R"}:
        raise ValueError(f"mps_fit: sweep_sequence must be made of 'L' and 'R', not "
                         f"{sweep_sequence!r}")
    bsz = choose_bsz(bsz, max_bond, cutoff)
    if bsz == 1:
        if cutoff not in (None, 0.0):
            raise ValueError("mps_fit: non-zero `cutoff` not supported for 1-site fit")
        if compress_opts:
            raise TypeError(f"mps_fit: 1-site sweeps take no split options "
                            f"({sorted(compress_opts)})")
    if cutoff is None:
        cutoff = 1e-10 if bsz == 2 else 0.0
    split_opts = dict(compress_opts)
    split_opts.setdefault("cutoff_mode", cutoff_mode)

    raw = _split_targets(targets)
    T = []
    for t in raw:
        if isinstance(t, tuple):
            if len(t) != 2:
                raise ValueError("mps_fit: an MPO target is a tuple (mpo, sites)")
            A, W, _ = _prepare(list(t[1]), list(t[0]), mpo_shape, transpose)
            T.append(_Target(A, W))
        else:
            T.append(_Target(_prepare_mps(list(t)), None))
    L, dims = len(T[0].A), T[0].dims()
    if L < 2:
        # as in the reference: a one-site chain has no bond to fit
        raise ValueError("mps_fit: the chain needs at least 2 sites")
    for t in T[1:]:
        if len(t.A) != L:
            raise ValueError(f"mps_fit: targets of {len(t.A)} and {L} sites")
        if t.dims() != dims:
            raise ValueError("mps_fit: targets with different physical dimensions")
    dt = np.result_type(*[x.dtype for t in T for x in t.A + (t.W or [])])
    for t in T:
        t.A = [a.astype(dt, copy=False) for a in t.A]
        t.W = None if t.W is None else [w.astype(dt, copy=False) for w in t.W]

    if guess is None or isinstance(guess, (str, dict)):
        max_bond, cur = bond_schedule(max_bond, initial_bond_dim, max_iterations, bsz,
                                      random=guess is None)
        if guess is None:
            if cur == math.inf:
                raise ValueError("mps_fit: a random start needs a finite bond dimension")
            F = [ops.asarray(x) for x in random_guess_host(dims, cur, dt, seed)]
        else:
            if not isinstance(raw[0], tuple):
                raise NotImplementedError("mps_fit: a generated guess compresses the first "
                                          "target, which must be an (mpo, sites) pair")
            gopts = {"method": guess} if isinstance(guess, str) else dict(guess)
            gopts.setdefault("max_bond", cur)
            gopts.setdefault("cutoff", cutoff)
            gopts.setdefault("mpo_shape", mpo_shape)
            gopts.setdefault("transpose", transpose)
            F = mps_gate_with_mpo(list(raw[0][1]), list(raw[0][0]), **gopts)
    else:
        F = _prepare_mps(list(guess))
        if len(F) != L or [f.shape[1] for f in F] != dims:
            raise ValueError("mps_fit: the guess does not match the targets' sites")
        cur = max(f.shape[2] for f in F[:-1])
        if max_bond is None:
            max_bond = cur
    F = [f.astype(dt, copy=False) for f in F]

    fit = _Fit(F, T)
    compute_tdiff = tol != 0.0
    sweeps = itertools.cycle(sweep_sequence)
    old, n, max_tdiff, reverse = "", 0, -1.0, False
    for it in range(int(max_iterations)):
        direction = next(sweeps)
        reverse = (direction == "L") != bool(sweep_reverse)
        if cur < max_bond:
            cur = min(2 * cur, max_bond)
        prepare = it == 0 or direction == old
        if bsz == 1 and max(f.shape[2] for f in F[:-1]) < cur:
            fit.expand(cur)
            prepare = True
        if prepare:
            fit.prepare(reverse, bsz)
        dots = [] if compute_tdiff else None
        if bsz == 1:
            fit.sweep1(reverse, dots)
        else:
            fit.sweep2(reverse, None if cur == math.inf else cur, cutoff, split_opts, dots)
        n += 1
        if compute_tdiff:
            max_tdiff = _max_tdiff(dots)
            if max_tdiff < tol:
                break
        old = direction

    c = 0 if reverse else L - 1
    # forced copies: a site no sweep replaced may still be the caller's array
    out = [ops.materialize(f, force=True) for f in F]
    if normalize:
        out[c] = ops.scale_(out[c], 1.0, div_by=_norm(out[c]))
    if info is not None:
        info["cur_orthog"] = (c, c)
        info["sweeps"] = n
        info["max_tdiff"] = max_tdiff
    return out


def mps_gate_with_mpo_fit(sites, mpo, max_bond, **kwargs):
    """``mps_gate_with_mpo_fit`` (tn1d/compress.py:3567-3586): the MPO applied
    to the MPS by :func:`mps_fit`; ``guess='zipup'`` is the reference's
    'fit-zipup'."""
    return mps_fit([(mpo, sites)], max_bond, **kwargs)
