"""DMRG-X on the device: one highly excited eigenstate of an open-boundary
MPO, the host-side mirror of quimb's ``DMRGX`` (quimb/tensor/tn1d/dmrg.py).

Each local step diagonalises the one-site effective Hamiltonian densely and
keeps the eigenvector that overlaps most with the state of the previous
sweep; among near-ties (overlap above ``overlap_thresh`` times the best) the
one of least local energy variance wins.  Started from a product state, the
sweeps converge to the eigenstate it is perturbatively close to -- the
standard tool for many-body-localised chains.

What is mirrored, with the reference line it follows:

  DMRGX(ham, p0, bond_dims, cutoffs, bsz)     :1214-1239
      energies[0] = <H>(p0), variances[0]     :1226-1228  (mps_expec, mps_expec2)
  sweep(direction, canonize)                  :1402-1447
      old ket as the bra of the overlap net   :1416-1417
      <H>, <H^2>, <old|new> environments      :1430-1432  -> env_*_step,
                                                              env2_*_step, norm_step*
  _update_local_state_1site_dmrgx             :1254-1358
      dense Heff                              :1245-1252  -> two contractions
      full eigh / partial eigh near target    :1270-1286  -> linalg.eigh (Jacobi)
      overlaps with the previous state        :1304
      selection by overlap, then variance     :1306-1346
      canonise after the update               :617-624
  _compute_post_sweep (variance)              :1449-1451
  _check_convergence (variance < tol)         :1465-1466

Divergence: above ``local_eig_partial_cutoff`` the reference runs a
shift-invert Lanczos around the current target energy for k eigenpairs to a
tolerance of 0.1; here the dense spectrum is still computed in full and the
k eigenpairs nearest the target are kept -- the set shift-invert converges
to, exactly.  Local problems are limited to ``MAX_LOCAL_DIM`` = 8192.

Host reads per site are the reference's own control reads: the eigenvalues,
the overlaps and, when several candidates survive the threshold, their
<H^2>.  The total energies of a sweep are read once when it ends.
"""

import numpy as np
import torch

from . import ops
from .array import Array
from .contract import contract_pair
from .dmrg import DMRG1
from .linalg import eigh
from .mps import (L_, LB_, M_, P_, PB_, R_, RB_, W2_, W_, WN2_, WN_, env2_left_step,
                  env2_right_step, env_left_step, env_right_step, mps_expec, mps_expec2,
                  norm_step, norm_step_right)

# largest local dimension D = chi_l d chi_r: the complex embedding (2D rows)
# of the dense Heff then still fits the Jacobi kernel without the blocked-QR
# preconditioning (linalg._QR_MAX_ROWS = 16384)
MAX_LOCAL_DIM = 8192

# labels of the flattened local index and of the eigenvector / candidate index
X_, K_ = 11, 12


def get_default_opts():
    """The reference's DMRGX options (dmrg.py:1230-1239)."""
    return {
        "local_eig_partial_cutoff": 2**11,
        "local_eig_partial_k": 0.02,
        "local_eig_tol": 1e-1,
        "overlap_thresh": 2 / 3,
        "bond_compress_method": "svd",
        "bond_compress_cutoff_mode": "sum2",
        "default_sweep_sequence": "RRLL",
        "bond_expand_rand_strength": 1e-9,
    }


def _columns(V, idx):
    """Columns ``idx`` of a (D, n) Array as a contiguous (D, len(idx)) Array."""
    ix = torch.as_tensor(np.asarray(idx, dtype=np.int64), device=V.t.device)
    return Array(V.t.index_select(1, ix), V.cj)


class DMRGX(DMRG1):
    """DMRG-X (Khemani, Pollmann & Sondhi, PRL 116, 247204 (2016)) for an
    open-boundary MPO, on the device.

    ``p0`` is the initial state (e.g. a computational basis state) as site
    arrays in ``mps_shape`` layout; the bond dimension is raised before every
    sweep of :meth:`solve` by ``expand_bond_dimension``.  ``energies`` holds
    <H> of ``p0`` and then the energy after every sweep, ``variances`` the
    matching <H^2> - <H>^2 (the convergence measure of :meth:`solve`)."""

    def __init__(self, ham, p0, bond_dims, cutoffs=1e-8, bsz=1, mpo_shape="lrud",
                 mps_shape="lpr", seed=None, dtype=None):
        if bsz != 1:
            raise NotImplementedError(
                f"quimb_b200.DMRGX: bsz={bsz}; only one-site updates exist (the "
                "reference has no two-site DMRG-X either)")
        if p0 is None:
            raise ValueError("quimb_b200.DMRGX: an initial state p0 is required")
        super().__init__(ham, bond_dims, cutoffs, p0=p0, mpo_shape=mpo_shape,
                         mps_shape=mps_shape, seed=seed, dtype=dtype)
        if self.ham[0].shape[0] != 1 or self.ham[-1].shape[1] != 1:
            raise NotImplementedError(
                "quimb_b200.DMRGX: open-boundary MPOs only (the end sites have "
                f"outer bonds {self.ham[0].shape[0]} and {self.ham[-1].shape[1]})")
        if dtype is not None and self._k[0].dtype != np.dtype(dtype):
            self._k = [ops.materialize(a.astype(dtype)) for a in self._k]
            self.ham = [w.astype(dtype) for w in self.ham]
        self.opts = get_default_opts()
        en = float(np.real(mps_expec(self._k, self.ham, shape="lpr").item()))
        en2 = float(np.real(mps_expec2(self._k, self.ham, shape="lpr").item()))
        self.energies.append(en)
        self.variances = [en2 - en ** 2]
        self._target_energy = en

    @classmethod
    def from_quimb_layout(cls, ham_arrays, p0_arrays, bond_dims, cutoffs=1e-8, **kw):
        return cls(ham_arrays, p0_arrays, bond_dims, cutoffs, mpo_shape="lrud",
                   mps_shape="lrp", **kw)

    @property
    def variance(self):
        return self.variances[-1]

    # ---- local operators (dmrg.py:1245-1252) ---------------------------------
    def dense_heff(self, i):
        """Heff[(a', s', b'), (a, s, b)] = L[a', w, a] W[w, w', s, s'] R[b', w', b]
        as a (D, D) device Array, rows on the bra side (``to_dense(lix, uix)``):
        two launches, the output ordered so that the reshape is free."""
        Lenv, W, Renv = self.lenv[i], self.ham[i], self.renv[i]
        a, s, b = self._k[i].shape
        T = contract_pair(Lenv.t, [LB_, W_, L_], W.t, [W_, WN_, P_, PB_],
                          [LB_, PB_, WN_, L_, P_], conj_a=Lenv.cj, conj_b=W.cj)
        H = contract_pair(T, [LB_, PB_, WN_, L_, P_], Renv.t, [RB_, WN_, R_],
                          [LB_, PB_, RB_, L_, P_, R_], conj_b=Renv.cj)
        D = a * s * b
        return Array(H.view(D, D))

    def _overlaps(self, i, V):
        """o[k] = sum_x V[x, k] g[x] with g the previous state's site ``i``
        between the overlap environments (conjugated): <old|new> with site i
        of the new state replaced by column k (dmrg.py:1296-1304)."""
        B, OL, OR = self._old[i], self.lovl[i], self.rovl[i]
        T = contract_pair(OL.t, [LB_, L_], B.t, [LB_, P_, RB_], [L_, P_, RB_],
                          conj_a=OL.cj, conj_b=not B.cj)
        g = contract_pair(T, [L_, P_, RB_], OR.t, [RB_, R_], [L_, P_, R_],
                          conj_b=OR.cj)
        return Array(contract_pair(V.t, [X_, K_], g.reshape(-1), [X_], [K_],
                                   conj_a=V.cj))

    def _candidate_en2(self, i, C):
        """en2[c] = <C_c| H^2_eff |C_c> for every candidate column at once
        (dmrg.py:1319-1343): the two-layer environments applied to the
        (D, c) block with c a free label, then the column-wise dot with c as a
        batch label."""
        a, s, b = self._k[i].shape
        X = C.reshape(a, s, b, C.shape[1])
        L2, W, R2 = self.lenv2[i], self.ham[i], self.renv2[i]
        T = contract_pair(L2.t, [LB_, W_, W2_, L_], X.t, [L_, P_, R_, K_],
                          [LB_, W_, W2_, P_, R_, K_], conj_a=L2.cj, conj_b=X.cj)
        T = contract_pair(T, [LB_, W_, W2_, P_, R_, K_], W.t, [W_, WN_, P_, M_],
                          [LB_, M_, WN_, W2_, R_, K_], conj_b=W.cj)
        T = contract_pair(T, [LB_, M_, WN_, W2_, R_, K_], W.t, [W2_, WN2_, M_, PB_],
                          [LB_, PB_, WN_, WN2_, R_, K_], conj_b=W.cj)
        T = contract_pair(T, [LB_, PB_, WN_, WN2_, R_, K_], R2.t, [RB_, WN_, WN2_, R_],
                          [LB_, PB_, RB_, K_], conj_b=R2.cj)
        return Array(contract_pair(X.t, [LB_, PB_, RB_, K_], T, [LB_, PB_, RB_, K_],
                                   [K_], conj_a=not X.cj))

    # ---- local update (dmrg.py:1254-1358) ------------------------------------
    def _update_local_state(self, i, direction, **compress_opts):
        return self._update_local_state_1site_dmrgx(i, direction)

    def _local_eigh(self, Heff, D):
        """Eigenpairs of the dense Heff as (host eigenvalues, device columns):
        all of them, or above ``local_eig_partial_cutoff`` the k nearest the
        target energy in ascending order (dmrg.py:1270-1286)."""
        evals, evecs = eigh(Heff)
        w = ops.to_numpy(evals)
        if D <= self.opts["local_eig_partial_cutoff"]:
            return w, evecs
        k = self.opts["local_eig_partial_k"]
        k = int(k * D) if isinstance(k, float) else int(k)
        keep = np.sort(np.argsort(np.abs(w - self._target_energy), kind="stable")[:k])
        return w[keep], _columns(evecs, keep)

    def _update_local_state_1site_dmrgx(self, i, direction):
        from .tebd import left_canonize_site, right_canonize_site
        a, s, b = self._k[i].shape
        D = a * s * b
        if D > MAX_LOCAL_DIM:
            raise NotImplementedError(
                f"quimb_b200.DMRGX: the local problem at site {i} has dimension "
                f"D = {a}*{s}*{b} = {D}; dense local eigensolves stop at "
                f"{MAX_LOCAL_DIM}")
        Heff = self.dense_heff(i)
        w, V = self._local_eigh(Heff, D)
        ov = np.abs(ops.to_numpy(self._overlaps(i, V)))
        thresh = self.opts["overlap_thresh"]
        if thresh == 1:
            best = int(np.argmax(ov))
        else:
            (cand,) = np.where(ov > np.max(ov) * thresh)
            if len(cand) == 1:
                best = int(cand[0])
            else:
                en2 = np.real(ops.to_numpy(self._candidate_en2(i, _columns(V, cand))))
                best = int(cand[np.argmin(en2 - w[cand] ** 2)])
        x = ops.materialize(Array(V.t[:, best], V.cj), force=True)
        self._k[i] = x.reshape(a, s, b)
        self._target_energy = float(w[best])
        # total energy <x|Heff|x>, left on the device until the sweep ends
        Hx = contract_pair(Heff.t, [LB_, L_], x.t, [L_], [LB_])
        tot_en = ops.vdot(x, Array(Hx))
        if direction == "right" and i < self.L - 1:
            left_canonize_site(self._k, i)
        elif direction == "left" and i > 0:
            right_canonize_site(self._k, i)
        return float(w[best]), tot_en

    # ---- sweeps (dmrg.py:1402-1447) ------------------------------------------
    def _ones(self, rank):
        A = self._k[0]
        return ops.ones((1,) * rank, dtype=A.dtype, device=A.device)

    def sweep(self, direction, canonize=True, verbosity=0, **update_opts):
        if direction not in ("R", "L"):
            raise ValueError("direction must be 'R' or 'L'")
        # the state before this sweep is the bra of the overlap network; site
        # updates replace list entries, never the arrays themselves
        self._old = list(self._k)
        if canonize:
            (self.right_canonize if direction == "R" else self.left_canonize)()
        k, W, old, L = self._k, self.ham, self._old, self.L
        one = (self._ones(3), self._ones(4), self._ones(2))
        loc, tot = [], []
        if direction == "R":
            self.renv, self.renv2, self.rovl = ({L - 1: e} for e in one)
            for i in range(L - 1, 0, -1):
                self.renv[i - 1] = env_right_step(self.renv[i], k[i], W[i])
                self.renv2[i - 1] = env2_right_step(self.renv2[i], k[i], W[i])
                self.rovl[i - 1] = norm_step_right(self.rovl[i], k[i], old[i])
            self.lenv, self.lenv2, self.lovl = ({0: e} for e in one)
            for i in range(L):
                if i > 0:
                    self.lenv[i] = env_left_step(self.lenv.pop(i - 1), k[i - 1], W[i - 1])
                    self.lenv2[i] = env2_left_step(self.lenv2.pop(i - 1), k[i - 1],
                                                   W[i - 1])
                    self.lovl[i] = norm_step(self.lovl.pop(i - 1), k[i - 1], old[i - 1])
                le, te = self._update_local_state(i, "right")
                for env in (self.renv, self.renv2, self.rovl):
                    env.pop(i, None)
                loc.append(le)
                tot.append(te)
        else:
            self.lenv, self.lenv2, self.lovl = ({0: e} for e in one)
            for i in range(L - 1):
                self.lenv[i + 1] = env_left_step(self.lenv[i], k[i], W[i])
                self.lenv2[i + 1] = env2_left_step(self.lenv2[i], k[i], W[i])
                self.lovl[i + 1] = norm_step(self.lovl[i], k[i], old[i])
            self.renv, self.renv2, self.rovl = ({L - 1: e} for e in one)
            for i in range(L - 1, -1, -1):
                if i < L - 1:
                    self.renv[i] = env_right_step(self.renv.pop(i + 1), k[i + 1], W[i + 1])
                    self.renv2[i] = env2_right_step(self.renv2.pop(i + 1), k[i + 1],
                                                    W[i + 1])
                    self.rovl[i] = norm_step_right(self.rovl.pop(i + 1), k[i + 1],
                                                   old[i + 1])
                le, te = self._update_local_state(i, "left")
                for env in (self.lenv, self.lenv2, self.lovl):
                    env.pop(i, None)
                loc.append(le)
                tot.append(te)
        self._old = None
        tot = tuple(float(e) for e in np.real(torch.stack([t.t for t in tot]).cpu().numpy()))
        self.local_energies.append(tuple(loc))
        self.total_energies.append(tot)
        return tot[-1]

    # ---- solve hooks (dmrg.py:1449-1466) -------------------------------------
    def _compute_post_sweep(self):
        en2 = float(np.real(mps_expec2(self._k, self.ham, shape="lpr").item()))
        self.variances.append(en2 - self.energies[-1] ** 2)

    def _check_convergence(self, tol):
        return self.variance < tol
