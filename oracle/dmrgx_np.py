"""Numpy restatement of DMRG-X (quimb/tensor/tn1d/dmrg.py:1185-1466), the
oracle of ``quimb_b200.dmrgx``.  Never imports the product package.

Layouts as in the product: MPS sites (l, p, r), MPO sites (l, r, u, d) with u
the ket-side index.  Every local step diagonalises the dense one-site Heff
with ``np.linalg.eigh``; above ``local_eig_partial_cutoff`` it keeps the k
eigenpairs nearest the target energy (the product's rule, see DESIGN.md),
selects by overlap with the previous sweep's state and, among candidates,
by least <H^2> - E^2.
"""

import itertools

import numpy as np

SX = np.array([[0, 0.5], [0.5, 0]])
ISY = np.array([[0, 0.5], [-0.5, 0]])
SZ = np.array([[0.5, 0], [0, -0.5]])


# -------------------------------------------------------------- operators ---
def mpo_mbl(fields, j=1.0):
    """H = j sum_i S_i.S_{i+1} + sum_i h_i S^z_i (spin-1/2, open chain) as
    (l, r, u, d) arrays of bond dimension 5 (real form: S^y S^y = -(iS^y)(iS^y))."""
    L = len(fields)
    out = []
    for i, h in enumerate(fields):
        W = np.zeros((5, 5, 2, 2))
        W[0, 0] = W[4, 4] = np.eye(2)
        W[4, 1], W[1, 0] = SX, j * SX
        W[4, 2], W[2, 0] = ISY, -j * ISY
        W[4, 3], W[3, 0] = SZ, j * SZ
        W[4, 0] = h * SZ
        # (l, r, d, u) -> (l, r, u, d): the operators are real symmetric up
        # to iS^y, whose transpose flips both its occurrences' signs
        W = W.transpose(0, 1, 3, 2)
        w = W[4:5] if i == 0 else (W[:, 0:1] if i == L - 1 else W)
        out.append(np.ascontiguousarray(w))
    return out


def mpo_fields(mpo):
    """h_i = Tr(H S^z_i) / 2^(L-2): the field part of an MBL MPO."""
    L = len(mpo)
    out = []
    for i in range(L):
        E = np.ones(1)
        for k, W in enumerate(mpo):
            op = SZ if k == i else np.eye(2)
            E = np.einsum("w,wvud,du->v", E, W, op)
        out.append(float(E.item().real) / 2.0 ** (L - 2))
    return out


def mpo_dist2(A, B):
    """|A - B|_F^2 of two MPOs through transfer matrices."""
    def tr(X, Y):
        E = np.ones((1, 1))
        for x, y in zip(X, Y):
            E = np.einsum("ab,acud,bedu->ce", E, x, y)
        return E.item()
    return (tr(A, A) - 2 * tr(A, B) + tr(B, B)).real


def mpo_dense(mpo):
    """(ket-side rows u... , bra-side cols d...) -> H[d, u] as a matrix acting
    on kets: <d|H|u>."""
    T = mpo[0][0]
    for W in mpo[1:]:
        T = np.einsum("a...,abud->b...ud", T, W)
    T = T[0]
    L = len(mpo)
    # axes: u0 d0 u1 d1 ...
    perm = [2 * i + 1 for i in range(L)] + [2 * i for i in range(L)]
    n = 2 ** L
    return T.transpose(perm).reshape(n, n)


def mps_dense(sites):
    T = sites[0][0]
    for A in sites[1:]:
        T = np.tensordot(T, A, axes=([-1], [0]))
    return T[..., 0].reshape(-1)


# ------------------------------------------------------------ environments ---
def env_left(E, A, W):
    return np.einsum("xwa,apb,wvpq,xqy->yvb", E, A, W, A.conj(), optimize=True)


def env_right(E, A, W):
    return np.einsum("apb,yvb,wvpq,xqy->xwa", A, E, W, A.conj(), optimize=True)


def env2_left(E, A, W):
    return np.einsum("xwza,apb,wvpm,zumq,xqy->yvub", E, A, W, W, A.conj(), optimize=True)


def env2_right(E, A, W):
    return np.einsum("apb,yvub,wvpm,zumq,xqy->xwza", A, E, W, W, A.conj(), optimize=True)


def ovl_left(E, A, B):
    """E'[b', b] = sum E[a', a] conj(B)[a', p, b'] A[a, p, b]"""
    return np.einsum("xa,apb,xpy->yb", E, A, B.conj(), optimize=True)


def ovl_right(E, A, B):
    return np.einsum("apb,yb,xpy->xa", A, E, B.conj(), optimize=True)


def mps_expec(sites, mpo):
    E = np.ones((1, 1, 1))
    for A, W in zip(sites, mpo):
        E = env_left(E, A, W.astype(A.dtype))
    return E.item()


def mps_expec2(sites, mpo):
    E = np.ones((1, 1, 1, 1))
    for A, W in zip(sites, mpo):
        E = env2_left(E, A, W.astype(A.dtype))
    return E.item()


def dense_heff(Lenv, W, Renv):
    a, s, b = Lenv.shape[2], W.shape[2], Renv.shape[2]
    H = np.einsum("xwa,wvpq,yvb->xqyapb", Lenv, W, Renv, optimize=True)
    return H.reshape(a * s * b, a * s * b)


# ------------------------------------------------------------ canonisation ---
def left_canonize_site(sites, i):
    A = sites[i]
    l, d, r = A.shape
    Q, R = np.linalg.qr(A.reshape(l * d, r))
    sites[i] = Q.reshape(l, d, -1)
    sites[i + 1] = np.tensordot(R, sites[i + 1], axes=([1], [0]))


def right_canonize_site(sites, i):
    A = sites[i]
    l, d, r = A.shape
    Q, R = np.linalg.qr(A.reshape(l, d * r).T)
    sites[i] = Q.T.reshape(-1, d, r)
    sites[i - 1] = np.tensordot(sites[i - 1], R.T, axes=([2], [0]))


def left_canonize(sites):
    for i in range(len(sites) - 1):
        left_canonize_site(sites, i)


def right_canonize(sites):
    for i in range(len(sites) - 1, 0, -1):
        right_canonize_site(sites, i)


def expand_bond_dimension(sites, new_bond_dim, rand_strength, rng):
    """Pad every bond to ``new_bond_dim`` with gaussian noise (core.py:1523-1569)."""
    for i in range(len(sites) - 1):
        cur = sites[i].shape[2]
        if cur >= new_bond_dim:
            continue
        extra = new_bond_dim - cur
        for which, ax in ((i, 2), (i + 1, 0)):
            A = sites[which]
            shape = list(A.shape)
            shape[ax] = extra
            pad = rand_strength * rng.standard_normal(shape)
            sites[which] = np.concatenate([A, pad.astype(A.dtype)], axis=ax)


# --------------------------------------------------------------- DMRG-X -----
def default_opts():
    return {
        "local_eig_partial_cutoff": 2**11,
        "local_eig_partial_k": 0.02,
        "overlap_thresh": 2 / 3,
        "default_sweep_sequence": "RRLL",
        "bond_expand_rand_strength": 1e-9,
    }


class DMRGX:
    """Mirror of the reference's DMRGX (bsz = 1, open chain).  ``decisions``
    records every selection: (site, n_candidates, threshold margin, winner gap)."""

    def __init__(self, mpo, p0, bond_dims, seed=0):
        self.mpo = [np.asarray(w) for w in mpo]
        self.k = [np.array(a) for a in p0]
        self.mpo = [w.astype(self.k[0].dtype) for w in self.mpo]
        self.L = len(mpo)
        bds = (bond_dims,) if isinstance(bond_dims, int) else tuple(bond_dims)
        self._bond_dims = itertools.chain(bds, itertools.repeat(bds[-1]))
        self.opts = default_opts()
        self.rng = np.random.default_rng(seed)
        en = float(np.real(mps_expec(self.k, self.mpo)))
        self.energies = [en]
        self.variances = [float(np.real(mps_expec2(self.k, self.mpo))) - en ** 2]
        self.target = en
        self.local_energies, self.total_energies, self.decisions = [], [], []

    @property
    def energy(self):
        return self.energies[-1]

    @property
    def variance(self):
        return self.variances[-1]

    def _update(self, i, direction):
        A = self.k[i]
        a, s, b = A.shape
        D = a * s * b
        H = dense_heff(self.lenv[i], self.mpo[i], self.renv[i])
        w, V = np.linalg.eigh(H)
        if D > self.opts["local_eig_partial_cutoff"]:
            kk = self.opts["local_eig_partial_k"]
            kk = int(kk * D) if isinstance(kk, float) else int(kk)
            keep = np.sort(np.argsort(np.abs(w - self.target), kind="stable")[:kk])
            w, V = w[keep], V[:, keep]
        g = np.einsum("xa,xpy,yb->apb", self.lovl[i], self.old[i].conj(), self.rovl[i])
        ov = np.abs(g.reshape(-1) @ V)
        thresh = self.opts["overlap_thresh"]
        order = np.sort(ov)[::-1]
        if thresh == 1:
            best = int(np.argmax(ov))
            self.decisions.append((i, 1, np.inf, (order[0] - order[1]) / order[0]
                                   if len(order) > 1 else np.inf))
        else:
            cut = np.max(ov) * thresh
            (cand,) = np.where(ov > cut)
            margin = np.min(np.abs(ov - cut)) / np.max(ov)
            if len(cand) == 1:
                best = int(cand[0])
                self.decisions.append((i, 1, margin, np.inf))
            else:
                C = V[:, cand].reshape(a, s, b, -1)
                en2 = np.real(np.einsum("xwza,apbc,wvpm,zumq,yvub,xqyc->c",
                                        self.lenv2[i], C, self.mpo[i], self.mpo[i],
                                        self.renv2[i], C.conj(), optimize=True))
                var = en2 - w[cand] ** 2
                best = int(cand[np.argmin(var)])
                vs = np.sort(var)
                self.decisions.append((i, len(cand), margin,
                                       (vs[1] - vs[0]) / max(abs(vs[0]), abs(vs[1]))))
        x = V[:, best]
        self.k[i] = x.reshape(a, s, b)
        self.target = float(w[best])
        tot = float(np.real(x.conj() @ H @ x))
        if direction == "right" and i < self.L - 1:
            left_canonize_site(self.k, i)
        elif direction == "left" and i > 0:
            right_canonize_site(self.k, i)
        return float(w[best]), tot

    def sweep(self, direction, canonize=True):
        self.old = list(self.k)
        if canonize:
            (right_canonize if direction == "R" else left_canonize)(self.k)
        k, W, old, L = self.k, self.mpo, self.old, self.L
        dt = k[0].dtype
        o3, o4, o2 = np.ones((1, 1, 1), dt), np.ones((1, 1, 1, 1), dt), np.ones((1, 1), dt)
        loc, tot = [], []
        if direction == "R":
            self.renv, self.renv2, self.rovl = {L - 1: o3}, {L - 1: o4}, {L - 1: o2}
            for i in range(L - 1, 0, -1):
                self.renv[i - 1] = env_right(self.renv[i], k[i], W[i])
                self.renv2[i - 1] = env2_right(self.renv2[i], k[i], W[i])
                self.rovl[i - 1] = ovl_right(self.rovl[i], k[i], old[i])
            self.lenv, self.lenv2, self.lovl = {0: o3}, {0: o4}, {0: o2}
            for i in range(L):
                if i > 0:
                    self.lenv[i] = env_left(self.lenv[i - 1], k[i - 1], W[i - 1])
                    self.lenv2[i] = env2_left(self.lenv2[i - 1], k[i - 1], W[i - 1])
                    self.lovl[i] = ovl_left(self.lovl[i - 1], k[i - 1], old[i - 1])
                le, te = self._update(i, "right")
                loc.append(le)
                tot.append(te)
        else:
            self.lenv, self.lenv2, self.lovl = {0: o3}, {0: o4}, {0: o2}
            for i in range(L - 1):
                self.lenv[i + 1] = env_left(self.lenv[i], k[i], W[i])
                self.lenv2[i + 1] = env2_left(self.lenv2[i], k[i], W[i])
                self.lovl[i + 1] = ovl_left(self.lovl[i], k[i], old[i])
            self.renv, self.renv2, self.rovl = {L - 1: o3}, {L - 1: o4}, {L - 1: o2}
            for i in range(L - 1, -1, -1):
                if i < L - 1:
                    self.renv[i] = env_right(self.renv[i + 1], k[i + 1], W[i + 1])
                    self.renv2[i] = env2_right(self.renv2[i + 1], k[i + 1], W[i + 1])
                    self.rovl[i] = ovl_right(self.rovl[i + 1], k[i + 1], old[i + 1])
                le, te = self._update(i, "left")
                loc.append(le)
                tot.append(te)
        self.local_energies.append(tuple(loc))
        self.total_energies.append(tuple(tot))
        return tot[-1]

    def solve(self, tol=1e-4, sweep_sequence=None, max_sweeps=10):
        seq = itertools.cycle(sweep_sequence or self.opts["default_sweep_sequence"])
        previous, converged = "0", False
        for _ in range(max_sweeps):
            direction, max_bond = next(seq), next(self._bond_dims)
            canonize = not (direction + previous in {"LR", "RL"})
            expand_bond_dimension(self.k, max_bond, self.opts["bond_expand_rand_strength"],
                                  self.rng)
            self.energies.append(self.sweep(direction, canonize=canonize))
            self.variances.append(float(np.real(mps_expec2(self.k, self.mpo)))
                                  - self.energies[-1] ** 2)
            converged = self.variance < tol
            if converged:
                break
            previous = direction
        return converged
