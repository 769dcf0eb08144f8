"""Two-site DMRG on the device: the host-side mirror of quimb's ``DMRG2``
for open-boundary MPOs (quimb/tensor/tn1d/dmrg.py).

What is mirrored, with the reference line it follows:

  DMRG2(ham, bond_dims, cutoffs, p0)      :501-601, :1161-1185
  opts (local_eig_tol/ncv, cutoff mode)   :19-102 (get_default_opts)
  sweep(direction, canonize, ...)         :885-998
  MovingEnvironment (right/left envs)     :105-443 -> env_*_step below
  _update_local_state_2site               :803-870
       Heff as a linear operator          :681-732 (TNLinearOperator)
       v0 = old two-site tensor           :832
       local eigensolve k=1               :626-645  -> eigh_lanczos (device)
       SVD split, absorb = direction      :842-848  -> svd_truncated (device)
       total energy = local network       :868
  solve(tol, max_sweeps, sweep_sequence)  :1032-1131

Every contraction is a launch of the pairwise kernel on whatever strides the
operands have; nothing is transposed in memory and nothing runs on the host
except control logic (tiny ncv x ncv eigenproblems, the truncation rule).

Layouts: MPS sites are held as (l, p, r) arrays, MPO sites as (l, r, u, d)
with u the ket-side index (quimb's 'lrud').  ``DMRG2.from_quimb_layout``
accepts quimb's own 'lrp' site arrays.
"""

import itertools

import numpy as np
import torch

from . import ops
from .array import Array
from .contract import contract_pair
from .lanczos import eigh_arpack_host_driver, eigh_lanczos
from .mps import (L_, LB_, P_, PB_, R_, RB_, W_, WN_, env_left_step,
                  env_right_step, mpo_lrud, mps_norm2, site_lpr)
from .split import get_U_sVH, get_Us_VH, qr_stabilized, svd_truncated

# extra labels for the two-site problem
S_, T_, SB_, TB_, W1_, W2_ = 10, 11, 12, 13, 14, 15


def get_default_opts():
    """The OBC subset of quimb's defaults (dmrg.py:84-102)."""
    return {
        "default_sweep_sequence": "R",
        "bond_compress_method": "svd",
        "bond_compress_cutoff_mode": "sum2",
        "local_eig_tol": 1e-3,
        "local_eig_ncv": 4,          # ARPACK's basis size in parity mode
        "device_eig_ncv": 32,        # max basis size of the device Lanczos
        "device_eig_min_steps": 4,   # like ARPACK's ncv=4: >= 4 matvecs per solve
        "local_eig_backend": None,   # None: device Lanczos; 'SCIPY': parity mode
        "local_eig_maxiter": None,
        "bond_expand_rand_strength": 1e-6,
    }


class EffHam2:
    """Two-site effective Hamiltonian  L - W_i - W_{i+1} - R  as a device
    linear operator (the role of TNLinearOperator, tensor_core.py:12297+).

    matvec order  L.x -> .W_i -> .W_{i+1} -> .R :
        2 w d^2 chi^3 + 2 w^2 d^3 chi^2 (x2) + 2 w d^2 chi^3 flops.
    """

    def __init__(self, Lenv, W1, W2, Renv, dims):
        self.L, self.W1, self.W2, self.R = Lenv, W1, W2, Renv
        self.dims = tuple(dims)  # (a, s, t, b)
        self.nmatvec = 0
        # W12[w, s, t, w2, s', t'] = sum_w1 W1[w, w1, s, s'] W2[w1, w2, t, t']:
        # the two bandwidth-bound MPO steps become one pass over the
        # (chi, w, d, d, chi) intermediate
        self.W12 = contract_pair(W1.t, [W_, W1_, S_, SB_], W2.t, [W1_, W2_, T_, TB_],
                                 [W_, S_, T_, W2_, SB_, TB_], conj_a=W1.cj,
                                 conj_b=W2.cj)

    supports_out = True      # matvec(v, out=flat tensor) writes the result in place

    def _out_view(self, out, rows):
        a, s, t, b = self.dims
        return None if out is None else out.view(rows, s, t, self.R.shape[0])

    def matvec(self, v, out=None):
        self.nmatvec += 1
        x = v.reshape(self.dims)
        # T1[a', w, s, t, b] = L[a', w, a] x[a, s, t, b]
        T = contract_pair(self.L.t, [LB_, W_, L_], x.t, [L_, S_, T_, R_],
                          [LB_, W_, S_, T_, R_], conj_a=self.L.cj, conj_b=x.cj)
        # T3[a', s', t', w2, b] = T1[a', w, s, t, b] W12[w, s, t, w2, s', t']
        T = contract_pair(T, [LB_, W_, S_, T_, R_], self.W12,
                          [W_, S_, T_, W2_, SB_, TB_], [LB_, SB_, TB_, W2_, R_])
        # y[a', s', t', b'] = T3 R[b', w2, b]
        y = contract_pair(T, [LB_, SB_, TB_, W2_, R_], self.R.t,
                          [RB_, W2_, R_], [LB_, SB_, TB_, RB_], conj_b=self.R.cj,
                          out=self._out_view(out, self.L.shape[0]))
        return Array(y).reshape(-1)

    __call__ = matvec

    def flops(self):
        a, s, t, b = self.dims
        w0, w1 = self.W1.shape[0], self.W1.shape[1]
        w2 = self.W2.shape[1]
        bp = self.R.shape[0]
        ap = self.L.shape[0]
        return 2 * (ap * w0 * a * s * t * b + ap * t * b * w0 * s * w1 * s
                    + ap * s * b * w1 * t * w2 * t + ap * s * t * b * w2 * bp)


class ShardedEffHam2(EffHam2):
    """Bond-sharded matvec (SURVEY.md 8e): this rank holds the rows
    a' in [lo, hi) of L[a', w, a] and of the vector.  One all-gather of the
    input vector per matvec; the three contraction steps are local in a'."""

    def __init__(self, Lenv, W1, W2, Renv, dims, shard):
        super().__init__(Lenv, W1, W2, Renv, dims)
        self.shard = shard
        self.lo, self.hi = shard.slab(dims[0])
        self.Ls = Array(self.L.t[self.lo:self.hi], self.L.cj)
        self.cols = dims[1] * dims[2] * dims[3]

    def local_slab(self, v):
        """Rows [lo, hi) of a full vector, as a flat contiguous Array."""
        x = ops.materialize(v).reshape(self.dims[0], self.cols)
        return Array(x.t[self.lo:self.hi].contiguous()).reshape(-1)

    def gather(self, v_local, transient=False):
        x = ops.materialize(v_local).t.reshape(self.hi - self.lo, self.cols)
        return Array(self.shard.all_gather_rows(x, self.dims[0],
                                                transient=transient)).reshape(-1)

    def matvec(self, v_local, out=None):
        self.nmatvec += 1
        # the gathered vector is consumed by the first contraction below: the
        # peer-memory exchange may hand out its own buffer (no copy)
        x = self.gather(v_local, transient=True).reshape(self.dims)
        T = contract_pair(self.Ls.t, [LB_, W_, L_], x.t, [L_, S_, T_, R_],
                          [LB_, W_, S_, T_, R_], conj_a=self.Ls.cj, conj_b=x.cj)
        T = contract_pair(T, [LB_, W_, S_, T_, R_], self.W12,
                          [W_, S_, T_, W2_, SB_, TB_], [LB_, SB_, TB_, W2_, R_])
        y = contract_pair(T, [LB_, SB_, TB_, W2_, R_], self.R.t,
                          [RB_, W2_, R_], [LB_, SB_, TB_, RB_], conj_b=self.R.cj,
                          out=self._out_view(out, self.hi - self.lo))
        return Array(y).reshape(-1)

    __call__ = matvec


class DMRG2:
    """Two-site DMRG for an open-boundary MPO, on the device.

    ``shard`` (a ``quimb_b200.dist.BondShard``): run the local eigensolves
    row-sharded over the ranks of the process group (every rank constructs the
    same DMRG2 with the same inputs and seed; the rest of the sweep is
    replicated and bit-identical on all ranks)."""

    def __init__(self, ham, bond_dims, cutoffs=1e-8, which="SA", p0=None,
                 mpo_shape="lrud", mps_shape="lpr", seed=None, dtype=None, shard=None):
        self.shard = shard if (shard is not None and shard.active) else None
        self.shard_min_bond = 64
        self.L = len(ham)
        n = self.L
        self.which = which
        self.ham = [mpo_lrud(w, mpo_shape, i, n) for i, w in enumerate(ham)]
        dt = np.dtype(dtype) if dtype is not None else self.ham[0].dtype
        self.phys_dim = self.ham[0].shape[2]
        self._set_bond_dim_seq(bond_dims)
        self._set_cutoff_seq(cutoffs)
        if p0 is None:
            p0 = _rand_mps(n, self._bond_dim0, self.phys_dim, dt, seed)
            mps_shape = "lpr"
        self._k = [ops.materialize(site_lpr(a, mps_shape, i, n), force=True)
                   for i, a in enumerate(p0)]
        if self._k[0].dtype != self.ham[0].dtype:
            # the network runs in the dtype of the state (quimb preserves the
            # dtype end to end: test_dmrg.py:290-300)
            self.ham = [w.astype(self._k[0].dtype) for w in self.ham]
        # quimb's DMRG starts from a normalised state (MPS_rand_state
        # normalises; a user p0 is used as given)
        self.energies, self.local_energies, self.total_energies = [], [], []
        self.nmatvecs = []
        self.opts = get_default_opts()
        self.timings = {}

    @classmethod
    def from_quimb_layout(cls, ham_arrays, bond_dims, cutoffs=1e-8, p0_arrays=None,
                          **kw):
        return cls(ham_arrays, bond_dims, cutoffs, p0=p0_arrays,
                   mpo_shape="lrud", mps_shape="lrp", **kw)

    def _set_bond_dim_seq(self, bond_dims):
        bds = (bond_dims,) if isinstance(bond_dims, int) else tuple(bond_dims)
        self._bond_dim0 = bds[0]
        self._bond_dims = itertools.chain(bds, itertools.repeat(bds[-1]))

    def _set_cutoff_seq(self, cutoffs):
        bds = (cutoffs,) if isinstance(cutoffs, float) else tuple(cutoffs)
        self._cutoffs = itertools.chain(bds, itertools.repeat(bds[-1]))

    @property
    def energy(self):
        return self.energies[-1]

    @property
    def state(self):
        """Site arrays in (l, p, r) layout."""
        return [Array(a.t.clone()) for a in self._k]

    def max_bond(self):
        return max(a.shape[2] for a in self._k[:-1]) if self.L > 1 else 1

    # ---- canonisation (tn1d/core.py:824-990 via tensor_canonize_bond) ------
    def right_canonize(self):
        k = self._k
        for i in range(self.L - 1, 0, -1):
            A = k[i]
            l, d, r = A.shape
            Lf, _, Q = qr_stabilized(A.reshape(l, d * r), absorb=get_Us_VH)
            kk = Q.shape[0]
            k[i] = ops.materialize(Q).reshape(kk, d, r)
            k[i - 1] = Array(contract_pair(k[i - 1].t, [0, 1, 2], Lf.t, [2, 3],
                                           [0, 1, 3], conj_a=k[i - 1].cj,
                                           conj_b=Lf.cj))

    def left_canonize(self):
        k = self._k
        for i in range(self.L - 1):
            A = k[i]
            l, d, r = A.shape
            Q, _, Rf = qr_stabilized(A.reshape(l * d, r), absorb=get_U_sVH)
            kk = Q.shape[1]
            k[i] = Q.reshape(l, d, kk)
            k[i + 1] = Array(contract_pair(Rf.t, [0, 1], k[i + 1].t, [1, 2, 3],
                                           [0, 2, 3], conj_a=Rf.cj,
                                           conj_b=k[i + 1].cj))

    # ---- environments (MovingEnvironment.init_segment, dmrg.py:281-322) -----
    def _ones_env(self):
        A = self._k[0]
        return ops.ones((1, 1, 1), dtype=A.dtype, device=A.device)

    bsz = 2     # sites optimised at once (DMRG1 overrides)

    def _init_right_envs(self):
        """renv[j]: everything to the right of site j."""
        self.renv = {self.L - 1: self._ones_env()}
        for i in range(self.L - 1, self.bsz - 1, -1):
            self.renv[i - 1] = env_right_step(self.renv[i], self._k[i], self.ham[i])

    def _init_left_envs(self):
        """lenv[i]: everything to the left of site i."""
        self.lenv = {0: self._ones_env()}
        for i in range(0, self.L - self.bsz):
            self.lenv[i + 1] = env_left_step(self.lenv[i], self._k[i], self.ham[i])

    def _update_local_state(self, i, direction, **update_opts):
        return self._update_local_state_2site(i, direction, **update_opts)

    # ---- local update (dmrg.py:803-870) --------------------------------------
    def _eigs(self, Heff, v0, comm=None):
        backend = self.opts["local_eig_backend"]
        if backend == "SCIPY":
            return eigh_arpack_host_driver(Heff, v0, which=self.which,
                                           ncv=self.opts["local_eig_ncv"],
                                           tol=self.opts["local_eig_tol"])
        n = v0.size if comm is None else Heff.dims[0] * Heff.cols
        ncv = self.opts["device_eig_ncv"]
        tol = self.opts["local_eig_tol"]
        if n < 800:
            # the reference diagonalises small effective Hamiltonians densely
            # (dmrg.py:690); here: the largest Krylov space, tight tolerance
            ncv, tol = min(n, 16), 1e-12
        return eigh_lanczos(Heff, v0, which=self.which, ncv=ncv, tol=tol,
                            maxiter=self.opts["local_eig_maxiter"],
                            return_info=True, comm=comm,
                            min_steps=self.opts["device_eig_min_steps"])

    def _update_local_state_2site(self, i, direction, max_bond=None,
                                  cutoff=1e-10, cutoff_mode="sum2",
                                  method="svd"):
        A, B = self._k[i], self._k[i + 1]
        a, s, _ = A.shape
        _, t, b = B.shape
        dims = (a, s, t, b)
        Heff = EffHam2(self.lenv[i], self.ham[i], self.ham[i + 1],
                       self.renv[i + 1], dims)
        # old two-site tensor as the initial guess (dmrg.py:832)
        v0 = Array(contract_pair(A.t, [L_, S_, 9], B.t, [9, T_, R_],
                                 [L_, S_, T_, R_], conj_a=A.cj, conj_b=B.cj))
        if (self.shard is not None and self.opts["local_eig_backend"] is None
                and a >= self.shard_min_bond * self.shard.world_size):
            Hs = ShardedEffHam2(self.lenv[i], self.ham[i], self.ham[i + 1],
                                self.renv[i + 1], dims, self.shard)
            loc_en, gs_local, info = self._eigs(Hs, Hs.local_slab(v0), comm=self.shard)
            loc_gs = Hs.gather(gs_local)
            self.shard.check()
            Heff.nmatvec = Hs.nmatvec
        else:
            loc_en, loc_gs, info = self._eigs(Heff, v0)
        self.nmatvecs.append(Heff.nmatvec)
        mat = loc_gs.reshape(a * s, t * b)
        absorb = get_U_sVH if direction == "right" else get_Us_VH
        if method not in ("svd", "svd:eig", "svd:rand"):
            raise ValueError("quimb_b200.DMRG2: bond_compress_method must be "
                             "'svd', 'svd:eig' or 'svd:rand'")
        from .split import array_split
        sinfo = {"error": None}
        extra = {}
        if method == "svd:rand":
            # static truncation to max_bond by a randomized range finder
            # (GEMM-bound: ~2.5x cheaper than the full Jacobi SVD at chi = 1024,
            # approximate near the cut); reproducible per (sweep, site)
            extra["seed"] = 7919 * len(self.local_energies) + i
            sinfo = None
        left, _, right = array_split(mat, method=method, absorb=absorb,
                                     max_bond=max_bond, cutoff=cutoff,
                                     cutoff_mode=cutoff_mode, info=sinfo, **extra)
        sinfo = sinfo or {"error": None}
        kdim = left.shape[1]
        self._k[i] = ops.materialize(left).reshape(a, s, kdim)
        self._k[i + 1] = ops.materialize(right).reshape(kdim, t, b)
        # total energy: the local network with the new tensors (dmrg.py:868)
        x = Array(contract_pair(self._k[i].t, [L_, S_, 9], self._k[i + 1].t,
                                [9, T_, R_], [L_, S_, T_, R_])).reshape(-1)
        Hx = Heff.matvec(x)
        tot_en = ops.vdot(x, Hx).item()
        self.last_trunc = sinfo
        return loc_en, float(np.real(tot_en))

    # ---- sweeps (dmrg.py:885-998) --------------------------------------------
    def sweep(self, direction, canonize=True, verbosity=0, **update_opts):
        L = self.L
        loc, tot = [], []
        if direction == "R":
            if canonize:
                self.right_canonize()
            self._init_right_envs()
            self.lenv = {0: self._ones_env()}
            for i in range(L - self.bsz + 1):
                if i > 0:
                    self.lenv[i] = env_left_step(self.lenv[i - 1], self._k[i - 1],
                                                 self.ham[i - 1])
                    self.lenv.pop(i - 1, None)
                le, te = self._update_local_state(i, "right", **update_opts)
                self.renv.pop(i + self.bsz - 1, None)
                loc.append(le); tot.append(te)
        elif direction == "L":
            if canonize:
                self.left_canonize()
            self._init_left_envs()
            self.renv = {L - 1: self._ones_env()}
            b = self.bsz
            for i in range(L - b, -1, -1):
                if i < L - b:
                    self.renv[i + b - 1] = env_right_step(self.renv[i + b],
                                                          self._k[i + b], self.ham[i + b])
                    self.renv.pop(i + b, None)
                le, te = self._update_local_state(i, "left", **update_opts)
                self.lenv.pop(i, None)
                loc.append(le); tot.append(te)
        else:
            raise ValueError("direction must be 'R' or 'L'")
        self.local_energies.append(tuple(loc))
        self.total_energies.append(tuple(tot))
        return tot[-1]

    def sweep_right(self, canonize=True, verbosity=0, **update_opts):
        return self.sweep("R", canonize=canonize, verbosity=verbosity, **update_opts)

    def sweep_left(self, canonize=True, verbosity=0, **update_opts):
        return self.sweep("L", canonize=canonize, verbosity=verbosity, **update_opts)

    def _compute_post_sweep(self):
        """Per-sweep work after the energy is recorded (dmrg.py:1129); DMRG-X
        records the variance here."""

    def _check_convergence(self, tol):
        if len(self.energies) < 2:
            return False
        return abs(self.energies[-2] - self.energies[-1]) < tol

    def solve(self, tol=1e-4, bond_dims=None, cutoffs=None, sweep_sequence=None,
              max_sweeps=10, verbosity=0):
        if bond_dims is not None:
            self._set_bond_dim_seq(bond_dims)
        if cutoffs is not None:
            self._set_cutoff_seq(cutoffs)
        if sweep_sequence is None:
            sweep_sequence = self.opts["default_sweep_sequence"]
        directions = itertools.cycle(sweep_sequence)
        previous = "0"
        converged = False
        for _ in range(max_sweeps):
            direction, max_bond, cutoff = (next(directions), next(self._bond_dims),
                                           next(self._cutoffs))
            canonize = not (direction + previous in {"LR", "RL"})
            if self.bsz == 1:
                # one-site updates cannot grow a bond (dmrg.py:1100-1106)
                self.expand_bond_dimension(
                    max_bond, rand_strength=self.opts["bond_expand_rand_strength"])
            energy = self.sweep(direction, canonize=canonize, max_bond=max_bond,
                                cutoff=cutoff,
                                cutoff_mode=self.opts["bond_compress_cutoff_mode"],
                                method=self.opts["bond_compress_method"])
            self.energies.append(energy)
            self._compute_post_sweep()
            if verbosity:
                print(f"sweep {len(self.energies)} {direction} max_bond={max_bond} "
                      f"E={energy}", flush=True)
            converged = self._check_convergence(tol)
            if converged:
                break
            previous = direction
        return converged


class EffHam1:
    """One-site effective Hamiltonian L - W - R (dmrg.py:756-801 through
    ``form_local_ops``): three launches of the contraction kernel,
    2 w d chi^3 + 2 w^2 d^2 chi^2 + 2 w d chi^3 flops."""

    def __init__(self, Lenv, W, Renv, dims):
        self.L, self.W, self.R = Lenv, W, Renv
        self.dims = tuple(dims)      # (a, s, b)
        self.nmatvec = 0

    def matvec(self, v):
        self.nmatvec += 1
        x = v.reshape(self.dims)
        T = contract_pair(self.L.t, [LB_, W_, L_], x.t, [L_, S_, R_], [LB_, W_, S_, R_],
                          conj_a=self.L.cj, conj_b=x.cj)
        T = contract_pair(T, [LB_, W_, S_, R_], self.W.t, [W_, W1_, S_, SB_],
                          [LB_, SB_, W1_, R_], conj_b=self.W.cj)
        y = contract_pair(T, [LB_, SB_, W1_, R_], self.R.t, [RB_, W1_, R_],
                          [LB_, SB_, RB_], conj_b=self.R.cj)
        return Array(y).reshape(-1)

    __call__ = matvec


class DMRG1(DMRG2):
    """One-site DMRG (quimb's ``DMRG1`` = ``DMRG(bsz=1)``, dmrg.py:1137-1156;
    local update :756-801): the bond dimension is raised before every sweep
    by padding the bonds with small noise (``expand_bond_dimension``,
    tn1d/core.py:1523-1569; tensor_core.py:2369-2440), each site is solved with
    the device Lanczos and the orthogonality centre moves on by a stabilised
    QR / LQ (``_canonize_after_1site_update`` :617-624)."""

    bsz = 1

    def __init__(self, ham, bond_dims=None, cutoffs=1e-8, which="SA", p0=None, **kw):
        if bond_dims is None:
            bond_dims = range(10, 1001, 10)
        self._expand_seed = kw.get("seed", None)
        super().__init__(ham, bond_dims, cutoffs, which=which, p0=p0, **kw)
        self._expand_calls = 0

    def expand_bond_dimension(self, new_bond_dim, rand_strength=0.0):
        """Pad every bond to at least ``new_bond_dim`` (zeros, or gaussian noise
        of strength ``rand_strength``), in place."""
        k = self._k
        gen = None
        for i in range(self.L - 1):
            cur = k[i].shape[2]
            if cur >= new_bond_dim:
                continue
            extra = new_bond_dim - cur
            for which in (i, i + 1):
                A = k[which].resolve()
                shape = list(A.shape)
                shape[2 if which == i else 0] = extra
                if rand_strength:
                    if gen is None:
                        gen = torch.Generator(device=A.device)
                        seed = 0 if self._expand_seed is None else int(self._expand_seed)
                        gen.manual_seed(1000003 * (seed + 1) + self._expand_calls)
                    rdt = A.real.dtype if A.dtype.is_complex else A.dtype
                    pad = torch.randn(shape, generator=gen, dtype=rdt, device=A.device)
                    pad = (pad * rand_strength).to(A.dtype)
                else:
                    pad = torch.zeros(shape, dtype=A.dtype, device=A.device)
                k[which] = Array(torch.cat([A, pad], dim=2 if which == i else 0))
        self._expand_calls += 1

    def _update_local_state(self, i, direction, **update_opts):
        return self._update_local_state_1site(i, direction, **update_opts)

    def _update_local_state_1site(self, i, direction, **compress_opts):
        from .tebd import left_canonize_site, right_canonize_site
        A = self._k[i]
        dims = A.shape
        Heff = EffHam1(self.lenv[i], self.ham[i], self.renv[i], dims)
        loc_en, loc_gs, info = self._eigs(Heff, ops.materialize(A, force=True))
        x = ops.materialize(loc_gs).reshape(-1)
        self._k[i] = x.reshape(*dims)
        Hx = Heff.matvec(x)
        tot_en = ops.vdot(x, Hx).item()
        self.nmatvecs.append(Heff.nmatvec)
        if direction == "right" and i < self.L - 1:
            left_canonize_site(self._k, i)
        elif direction == "left" and i > 0:
            right_canonize_site(self._k, i)
        return loc_en, float(np.real(tot_en))


def _rand_mps(n, bond_dim, d, dtype, seed):
    """Random normalised OBC MPS in (l, p, r) layout (the role of
    ham.rand_state / MPS_rand_state, tensor_builder.py:4166-4244)."""
    rng = np.random.default_rng(seed)
    bonds = [1]
    for i in range(1, n):
        e = min(i, n - i)
        cap = d ** e if e < 40 else bond_dim
        bonds.append(int(min(cap, bond_dim)))
    bonds.append(1)
    sites = []
    for i in range(n):
        shape = (bonds[i], d, bonds[i + 1])
        x = rng.standard_normal(shape)
        if np.dtype(dtype).kind == "c":
            x = (x + 1j * rng.standard_normal(shape)) / np.sqrt(2)
        nd = sum(1 for q in shape if q > 1) or 1
        x = x / np.linalg.norm(x) ** (1.5 / nd)
        sites.append(ops.asarray(x.astype(np.dtype(dtype))))
    nrm = float(np.sqrt(abs(mps_norm2(sites, "lpr").item())))
    sites[0] = sites[0] / nrm
    return sites
