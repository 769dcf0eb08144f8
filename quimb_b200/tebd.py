"""MPS gate application and TEBD on the device: the two-site
contract-then-split primitive either side of the hot path (SURVEY.md 8f-4).

Mirrors, at array level and for open boundaries,

  gate_split                     quimb/tensor/tn1d/core.py:2219-2247
      -> eager 'split' path      quimb/tensor/gating.py:86-123
  left/right_canonize_site       tn1d/core.py:824-905 (tensor_canonize_bond)
  LocalHam1D (nearest neighbour) tn1d/tebd.py:12-96, tnag/tebd.py:180-392
  trotter_schedule               tnag/tebd.py:78-126
  TEBD.sweep / step / update_to  tn1d/tebd.py:221-553
  MatrixProductState.sample      tn1d/core.py:3871-3990 (all samples at once)

MPS sites are (l, p, r) device arrays.  One gate application is a 3-tensor
contraction (two launches of the pairwise kernel, gate indices folded into
the second) plus one truncated split (device Jacobi SVD); the only host
arithmetic is the d^2 x d^2 matrix exponential of a local term (control
logic, cached per (bond, step fraction) exactly as the reference caches it).
"""

import numpy as np

from . import ops
from .array import Array
from .contract import contract_pair
from .linalg import norm as _norm
from .mps import site_lpr
from .split import qr_stabilized, tensor_split, get_U_sVH, get_Us_VH


def set_default_compress_mode(opts, cyclic=False):
    opts.setdefault("cutoff_mode", "rel" if cyclic else "rsum2")


# ------------------------------------------------------------ canonization ---
def left_canonize_site(sites, i):
    """QR site i, absorb R into site i + 1 (tn1d/core.py:824-847), in place."""
    A = sites[i]
    l, d, r = A.shape
    Q, _, R = qr_stabilized(A.reshape(l * d, r), absorb=get_U_sVH)
    k = Q.shape[1]
    sites[i] = Q.reshape(l, d, k)
    B = sites[i + 1]
    sites[i + 1] = Array(contract_pair(R.t, [0, 1], B.t, [1, 2, 3], [0, 2, 3],
                                       conj_a=R.cj, conj_b=B.cj))


def right_canonize_site(sites, i):
    """LQ site i, absorb L into site i - 1 (tn1d/core.py:849-872), in place."""
    A = sites[i]
    l, d, r = A.shape
    Lf, _, Q = qr_stabilized(A.reshape(l, d * r), absorb=get_Us_VH)
    k = Q.shape[0]
    sites[i] = ops.materialize(Q).reshape(k, d, r)
    B = sites[i - 1]
    sites[i - 1] = Array(contract_pair(B.t, [0, 1, 2], Lf.t, [2, 3], [0, 1, 3],
                                       conj_a=B.cj, conj_b=Lf.cj))


def left_canonize(sites, start=None, stop=None):
    """tn1d/core.py:874-925: sites start .. stop-1 become left isometries."""
    start = 0 if start is None else start
    stop = len(sites) - 1 if stop is None else stop
    for i in range(start, stop):
        left_canonize_site(sites, i)


def right_canonize(sites, start=None, stop=None):
    """tn1d/core.py:937-988: sites start .. stop+1 become right isometries."""
    start = len(sites) - 1 if start is None else start
    stop = 0 if stop is None else stop
    for i in range(start, stop, -1):
        right_canonize_site(sites, i)


def canonicalize(sites, where):
    """Orthogonality centre at site(s) ``where`` (int or (imin, imax))."""
    imin, imax = (where, where) if isinstance(where, int) else (min(where), max(where))
    left_canonize(sites, 0, imin)
    right_canonize(sites, len(sites) - 1, imax)


# --------------------------------------------------------------- gate_split ---
def gate_split(sites, G, where, **compress_opts):
    """Apply the two-site gate ``G`` (d^2 x d^2 or (d, d, d, d), index order
    (out_i, out_j, in_i, in_j)) to adjacent sites ``where = (i, j)`` and split
    the result back into MPS form, in place (gate_split, tn1d/core.py:2219;
    the eager contract + ``tensor_split`` of gating.py:86-123).  Defaults as
    the reference: method 'svd', cutoff 1e-10, cutoff_mode 'rsum2',
    absorb 'both'."""
    set_default_compress_mode(compress_opts)
    i, j = where
    if abs(i - j) != 1:
        raise ValueError("gate_split: sites must be adjacent "
                         "(use gate_with_auto_swap for distant sites)")
    A, B = sites[min(i, j)], sites[max(i, j)]
    d1, d2 = A.shape[1], B.shape[1]
    G = ops.asarray(G)
    if G.ndim == 2:
        G = G.reshape(*((d1, d2, d1, d2) if i < j else (d2, d1, d2, d1)))
    if i > j:
        G = G.transpose(1, 0, 3, 2)          # gate given for (j, i): relabel
    # theta[l, p', q', r] = sum A[l, p, m] B[m, q, r] G[p', q', p, q]
    if A.dtype != G.dtype or B.dtype != G.dtype:
        dt = np.result_type(A.dtype, B.dtype, G.dtype)
        A, B, G = (x.astype(dt, copy=False) for x in (A, B, G))
    T = contract_pair(A.t, [0, 1, 2], B.t, [2, 3, 4], [0, 1, 3, 4],
                      conj_a=A.cj, conj_b=B.cj)
    T = Array(contract_pair(G.t, [5, 6, 1, 3], T, [0, 1, 3, 4], [0, 5, 6, 4],
                            conj_a=G.cj))
    info = compress_opts.pop("info", None)
    parts = tensor_split(T, "lpqr", "lp", "qr", info=info, **compress_opts)
    left, right = parts[0], parts[-1]
    sites[min(i, j)] = ops.materialize(left)
    sites[max(i, j)] = ops.materialize(right)
    return parts[1] if len(parts) == 3 else None


def swap_sites_with_compress(sites, i, j, **compress_opts):
    """Swap adjacent sites by a SWAP 'gate' + split (tn1d/core.py
    swap_sites_with_compress): theta[l, q, p, r] split back."""
    i, j = min(i, j), max(i, j)
    if j != i + 1:
        raise ValueError("swap_sites_with_compress: sites must be adjacent")
    set_default_compress_mode(compress_opts)
    A, B = sites[i], sites[j]
    T = Array(contract_pair(A.t, [0, 1, 2], B.t, [2, 3, 4], [0, 3, 1, 4],
                            conj_a=A.cj, conj_b=B.cj))
    left, right = tensor_split(T, "lqpr", "lq", "pr", **compress_opts)
    sites[i], sites[j] = ops.materialize(left), ops.materialize(right)


def gate_with_auto_swap(sites, G, where, swap_back=True, **compress_opts):
    """Two-site gate on non-adjacent sites by swapping j next to i, gating,
    and swapping back (tn1d/core.py:2251-2322)."""
    i, j = where
    if i > j:
        i, j = j, i
        final_where, absorb = (i + 1, i), "left"
    else:
        final_where, absorb = (i, i + 1), "right"
    need = i + 1 != j
    if need:
        for k in range(j, i + 1, -1):
            canonicalize(sites, (k - 1, k))
            swap_sites_with_compress(sites, k - 1, k, absorb="left", **compress_opts)
    canonicalize(sites, (i, i + 1))
    gate_split(sites, G, final_where, absorb=absorb, **compress_opts)
    if need and swap_back:
        for k in range(i + 1, j):
            canonicalize(sites, (k, k + 1))
            swap_sites_with_compress(sites, k, k + 1, absorb="right", **compress_opts)


# -------------------------------------------------------------- LocalHam1D ---
def trotter_schedule(nlayers, order=2):
    """tnag/tebd.py:78-126."""
    if order == 1:
        return [(k, 1.0) for k in range(nlayers)]
    if order == 2:
        if nlayers == 0:
            return []
        return [*((k, 0.5) for k in range(nlayers - 1)), (nlayers - 1, 1.0),
                *((k, 0.5) for k in reversed(range(nlayers - 1)))]
    if order == 4:
        s = 1 / (4 - 4 ** (1 / 3))
        order2 = trotter_schedule(nlayers, order=2)
        return [(k, frac * f) for f in (s, s, 1 - 4 * s, s, s) for k, frac in order2]
    raise ValueError(f"Unknown Trotter order {order}, valid options are 1, 2, 4.")


class LocalHam1D:
    """Nearest-neighbour Hamiltonian as a dict of two-site terms
    (tn1d/tebd.py:12-96); single-site terms are split evenly over the bonds
    covering the site (tnag/tebd.py:244-273).  Terms live on the host (they are
    d^2 x d^2); exponentiated gates are uploaded once and cached."""

    def __init__(self, L, H2, H1=None, cyclic=False):
        if cyclic:
            raise NotImplementedError("quimb_b200.LocalHam1D: open boundaries only")
        self.L = int(L)
        self.cyclic = False
        if hasattr(H2, "shape"):
            H2 = {None: np.asarray(H2)}
        else:
            H2 = {k: np.asarray(v) for k, v in dict(H2).items()}
        default = H2.pop(None, None)
        self.terms = {}
        for (a, b), h in H2.items():
            if a > b:
                d = int(round(h.shape[0] ** 0.5))
                h = h.reshape(d, d, d, d).transpose(1, 0, 3, 2).reshape(d * d, d * d)
                a, b = b, a
            self.terms[a, b] = h
        if default is not None:
            for i in range(self.L - 1):
                self.terms.setdefault((i, i + 1), default)
        if H1 is not None:
            if hasattr(H1, "shape"):
                H1 = {None: np.asarray(H1)}
            else:
                H1 = {k: np.asarray(v) for k, v in dict(H1).items()}
            d1 = H1.pop(None, None)
            if d1 is not None:
                for site in range(self.L):
                    H1.setdefault(site, d1)
            for site, h in H1.items():
                pairs = [p for p in self.terms if site in p]
                if not pairs:
                    raise ValueError("There are no two site terms to add this single "
                                     f"site term to - site {site} is not coupled to "
                                     "anything.")
                Id = np.eye(h.shape[0], dtype=h.dtype)
                tens = (np.kron(h, Id), np.kron(Id, h))
                for p in pairs:
                    self.terms[p] = self.terms[p] + tens[p.index(site)] / len(pairs)
        self._expm = {}

    def mean_norm(self):
        return sum(np.linalg.norm(h) for h in self.terms.values()) / len(self.terms)

    def get_gate(self, where):
        return self.terms[tuple(sorted(where))]

    def get_gate_expm(self, where, x):
        key = (tuple(sorted(where)), complex(x))
        U = self._expm.get(key)
        if U is None:
            import scipy.linalg as sla
            U = ops.asarray(np.ascontiguousarray(sla.expm(self.get_gate(where) * x)))
            self._expm[key] = U
        return U


# --------------------------------------------------------------------- TEBD ---
class TEBD:
    """Time evolving block decimation of an open-boundary MPS (tn1d/tebd.py:
    221-553).  ``p0``: site arrays (layout ``mps_shape``); ``H``: a
    :class:`LocalHam1D` or a two-site d^2 x d^2 array."""

    TARGET_TOL = 1e-13

    def __init__(self, p0, H, dt=None, tol=None, t0=0.0, split_opts=None,
                 imag=False, mps_shape="lpr"):
        n = len(p0)
        self._pt = [ops.materialize(site_lpr(a, mps_shape, i, n), force=True)
                    for i, a in enumerate(p0)]
        self.L = n
        if not isinstance(H, LocalHam1D):
            H = LocalHam1D(self.L, H2=np.asarray(H))
        self.H = H
        if not imag and not np.issubdtype(self._pt[0].dtype, np.complexfloating):
            # real-time gates are complex: the state is complex from the start
            self._pt = [a.astype(np.result_type(a.dtype, np.complex64)) for a in self._pt]
        canonicalize(self._pt, 0)
        self._ham_norm = H.mean_norm()
        self._err = 0.0
        self.t0 = self.t = t0
        if dt and tol:
            raise ValueError("Can't set default for both ``dt`` and ``tol``.")
        self.dt = self._dt = dt
        self.tol = tol
        self.imag = imag
        self.split_opts = dict(split_opts or {})
        self._queued_sweep = None

    @property
    def pt(self):
        return [a.copy() for a in self._pt]

    @property
    def err(self):
        return self._err

    def choose_time_step(self, tol, T, order):
        return (tol / (T * self._ham_norm)) ** (1 / order)

    def _get_gate_from_ham(self, dt_frac, sites):
        imag_factor = 1.0 if self.imag else 1.0j
        return self.H.get_gate_expm(sites, -imag_factor * self._dt * dt_frac)

    def sweep(self, direction, dt_frac, dt=None, queue=False):
        """tn1d/tebd.py:323-436 (open boundaries)."""
        if dt is not None:
            dt_frac *= dt / self._dt
        if queue:
            if self._queued_sweep:
                if direction == self._queued_sweep[0]:
                    self._queued_sweep[1] += dt_frac
                    return
                new_queued = [direction, dt_frac]
                direction, dt_frac = self._queued_sweep
                self._queued_sweep = new_queued
            else:
                self._queued_sweep = [direction, dt_frac]
                return
        elif self._queued_sweep:
            qd, qf = self._queued_sweep
            self._queued_sweep = None
            self.sweep(qd, qf, queue=False)
        pt = self._pt
        if direction == "right":
            final_site_ind = self.L - 1
            for i in range(0, final_site_ind, 2):
                U = self._get_gate_from_ham(dt_frac, (i, i + 1))
                left_canonize(pt, start=max(0, i - 1), stop=i)
                gate_split(pt, U, (i, i + 1), absorb="right", **self.split_opts)
            if self.L % 2 == 1:
                left_canonize_site(pt, self.L - 2)
        elif direction == "left":
            final_site_ind = 1
            for i in reversed(range(final_site_ind, self.L - 1, 2)):
                U = self._get_gate_from_ham(dt_frac, (i, i + 1))
                right_canonize(pt, start=min(self.L - 1, i + 2), stop=i + 1)
                gate_split(pt, U, (i, i + 1), absorb="left", **self.split_opts)
            right_canonize_site(pt, 1)
        else:
            raise ValueError("direction must be 'right' or 'left'")
        if self.imag:
            x = pt[final_site_ind]
            pt[final_site_ind] = ops.scale_(ops.materialize(x, force=True), 1.0,
                                            div_by=_norm(x))

    def step(self, order=2, dt=None, **sweep_opts):
        directions = ("right", "left")
        for k, frac in trotter_schedule(2, order=order):
            self.sweep(directions[k], frac, dt=dt, **sweep_opts)
        dt = self._dt if dt is None else dt
        self.t += dt
        self._err += self._ham_norm * dt ** (order + 1)

    def _compute_sweep_dt_tol(self, T, dt, tol, order):
        dt = self.dt if dt is None else dt
        tol = self.tol if tol is None else tol
        if not (dt or tol):
            raise ValueError("Must set one of ``dt`` and ``tol``.")
        if dt and tol:
            raise ValueError("Can't set both ``dt`` and ``tol``.")
        self._dt = self.choose_time_step(tol, T - self.t, order) if dt is None else dt
        return self._dt

    def update_to(self, T, dt=None, tol=None, order=4):
        if T < self.t - self.TARGET_TOL:
            raise NotImplementedError
        self._compute_sweep_dt_tol(T, dt, tol, order)
        while self.t < T - self._dt:
            self.step(order=order, dt=None, queue=True)
        self.step(order=order, dt=T - self.t, queue=False)

    def at_times(self, ts, dt=None, tol=None, order=4):
        for t in ts:
            self.update_to(t, dt=dt, tol=tol, order=order)
            yield self.pt


# ------------------------------------------------------- MPS circuit driver ---
def gate_single(sites, G, i):
    """Apply a one-site gate G[out, in] to site i (MatrixProductState.gate with
    contract=True, tn1d/core.py:2132-2217): one launch, isometries preserved
    for unitary G."""
    A = sites[i]
    G = ops.asarray(G)
    if A.dtype != G.dtype:
        dt = np.result_type(A.dtype, G.dtype)
        A, G = A.astype(dt, copy=False), G.astype(dt, copy=False)
    sites[i] = Array(contract_pair(A.t, [0, 1, 2], G.t, [3, 1], [0, 3, 2],
                                   conj_a=A.cj, conj_b=G.cj))


def mps_zero_state(n, d=2, dtype="complex128"):
    """|00...0> as bond-dimension-1 (l, p, r) site arrays on the device."""
    out = []
    for _ in range(n):
        x = np.zeros((1, d, 1), dtype=dtype)
        x[0, 0, 0] = 1.0
        out.append(ops.asarray(x))
    return out


def apply_circuit(sites, gates, contract="swap+split", **compress_opts):
    """Run a gate list on an MPS in place, the way quimb's ``CircuitMPS`` does
    (quimb/tensor/circuit/mps.py): one-qubit gates are contracted into their
    site, two-qubit gates go through ``gate_with_auto_swap`` (swap to
    adjacency, canonicalise, contract + truncated split, swap back).

    ``gates``: iterable of ``(G, (i,))`` or ``(G, (i, j))`` with ``G`` a
    (2, 2) / (4, 4) or (2, 2, 2, 2) array, index order (out..., in...).

    ``contract`` chooses how gates on several sites are applied, as
    ``gate_contract`` does (tn1d/core.py:214-246):

      'swap+split'  (default) two-site gates only, by ``gate_with_auto_swap``
      'auto-mps'    two-site gates by ``gate_with_auto_swap``, wider ones by
                    ``nonlocal_gates.mps_gate_nonlocal``
      'nonlocal'    every gate on two or more sites by ``mps_gate_nonlocal``

    Under 'auto-mps' and 'nonlocal' an entry may also be
    ``(G, qubits, controls)``, applied by ``nonlocal_gates.mps_gate_controlled``,
    and ``compress_opts`` (``max_bond``, ``cutoff`` ...) go to every gate;
    ``method`` names the sub-MPO compression ('direct', 'dm', 'zipup') and
    goes to the sub-MPO gates only.  One ``info`` dict (``compress_opts["info"]``, or a new one)
    carries the orthogonality centre from gate to gate, so a gate whose span
    already holds the centre skips canonicalisation."""
    compress_opts.setdefault("cutoff", 1e-10)
    if contract not in ("swap+split", "auto-mps", "nonlocal"):
        raise ValueError(f"apply_circuit: unknown contract mode {contract!r}")
    if contract == "swap+split":
        for entry in gates:
            if len(entry) != 2:
                raise ValueError("apply_circuit: controlled gates need contract='auto-mps' "
                                 "or 'nonlocal'")
            G, where = entry
            where = tuple(where)
            if len(where) == 1:
                gate_single(sites, G, where[0])
            elif len(where) == 2:
                gate_with_auto_swap(sites, G, where, **compress_opts)
            else:
                raise ValueError("apply_circuit: only one- and two-qubit gates")
        return sites
    from . import nonlocal_gates as nl
    info = compress_opts.pop("info", None)
    if info is None:
        info = {}
    swap_opts = {k: v for k, v in compress_opts.items() if k != "method"}
    for entry in gates:
        G, where = entry[0], tuple(int(w) for w in entry[1])
        controls = tuple(entry[2]) if len(entry) > 2 else ()
        if controls:
            sites[:] = nl.mps_gate_controlled(sites, G, where, controls, info=info,
                                              **compress_opts)
        elif len(where) == 1:
            gate_single(sites, G, where[0])
            # a non-unitary gate leaves its site no longer an isometry
            cur = info.get("cur_orthog")
            if isinstance(cur, tuple):
                info["cur_orthog"] = (min(cur[0], where[0]), max(cur[1], where[0]))
        elif len(where) == 2 and contract == "auto-mps":
            gate_with_auto_swap(sites, G, where, **swap_opts)
            # every site outside the gate's span is an isometry afterwards
            info["cur_orthog"] = (min(where), max(where))
        else:
            sites[:] = nl.mps_gate_nonlocal(sites, G, where, info=info, **compress_opts)
    return sites


def mps_amplitude(sites, bits):
    """<bits|psi>: the chain of selected (chi x chi) matrices, left to right."""
    v = None
    for A, b in zip(sites, bits):
        M = Array(A.t[:, int(b), :], A.cj)
        v = M if v is None else ops.tensordot(v, M, axes=((v.ndim - 1,), (0,)))
    return v.reshape(()).item()


# ---------------------------------------------------------------- sampling ---
# Byte budget of one chunk's W = V . A_i (C_chunk x d x r): samples are drawn
# in chunks small enough for W to stay below it.
SAMPLE_CHUNK_BYTES = 1 << 30


def _sample_rng(seed):
    """numpy Generator of ``seed``: an int / None seeds a new one, a Generator
    (or a ``quimb_b200.random.default_rng`` wrapper of one) is used as is."""
    if hasattr(seed, "_rng"):
        seed = seed._rng
    return np.random.default_rng(seed)


def _sample_prepare(sites):
    """Right-canonical, unit-norm fp64 / c128 copy of an open-boundary MPS
    (the caller's list and arrays are not touched) and the norm factor taken
    off its first site, a 0-d device array."""
    sites = [ops.asarray(a) for a in sites]
    if not sites:
        raise ValueError("mps_sample: empty MPS")
    for a in sites:
        if a.ndim != 3:
            raise ValueError("mps_sample: sites must be (l, p, r) arrays")
        if np.dtype(a.dtype).kind not in "fc":
            raise TypeError(f"mps_sample: unsupported dtype {a.dtype}")
    if sites[0].shape[0] != 1 or sites[-1].shape[2] != 1:
        raise ValueError("mps_sample: open boundaries only (first left and last "
                         "right bond of dimension 1)")
    from .contract import _WIDE, convert
    cplx = any(np.dtype(a.dtype).kind == "c" for a in sites)
    psi = []
    for a in sites:
        if cplx and np.dtype(a.dtype).kind == "f":
            a = a.astype(np.complex128 if a.dtype == np.float64 else np.complex64)
        if a.t.dtype in _WIDE:
            # single precision: widen once, sample in double precision
            a = Array(convert(ops.materialize(a).t, _WIDE[a.t.dtype]))
        psi.append(a)
    canonicalize(psi, 0)
    # the centre to unit norm through an LQ of the 1 x (d r) site: the QR
    # kernel rescales by a power of two, so norms of 1e+-200 neither overflow
    # nor underflow; L (1 x 1) is the norm
    A = psi[0]
    _, d, r = A.shape
    Lf, _, Q = qr_stabilized(A.reshape(1, d * r), absorb=get_Us_VH)
    psi[0] = ops.materialize(Q).reshape(1, d, r)
    return psi, Lf.reshape(())


def _sample_chunks(psi, u, configs, omegas, events=None):
    """The sampling loop on the device: for every chunk of samples and every
    site, W = V . A_i on the contraction engine, then ``qb_sample_select``
    (two launches per site per chunk).  ``u`` (C x L, fp64), ``configs``
    (C x L, int64) and ``omegas`` (C, fp64, ones) are contiguous device
    tensors; returns the number of chunks.  ``events``: a list that receives
    one (rows, site, start, after-contraction, after-selection) tuple of
    recorded CUDA events per step (benchmarks)."""
    import torch
    from . import _lib
    C, L = u.shape
    dt = psi[0].t.dtype
    row_bytes = max(a.shape[1] * a.shape[2] for a in psi) * psi[0].t.element_size()
    chunk = max(1, min(C, SAMPLE_CHUNK_BYTES // row_bytes))
    code = _lib.qb_dtype(dt)
    lib = _lib.load()
    n_chunks = 0
    for c0 in range(0, C, chunk):
        cc = min(chunk, C - c0)
        V = torch.ones((cc, 1), dtype=dt, device=u.device)
        for i, A in enumerate(psi):
            _, d, r = A.shape
            if events is not None:
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                ev[0].record()
            W = contract_pair(V, [0, 1], A.t, [1, 2, 3], [0, 2, 3], conj_b=A.cj)
            if events is not None:
                ev[1].record()
            V = torch.empty((cc, r), dtype=dt, device=u.device)
            rc = lib.qb_sample_select(
                code, cc, d, r, W.data_ptr(), u.data_ptr() + 8 * (c0 * L + i), L,
                configs.data_ptr() + 8 * (c0 * L + i), L, omegas.data_ptr() + 8 * c0,
                V.data_ptr(), _lib.stream_ptr())
            _lib.check(rc, "qb_sample_select")
            if events is not None:
                ev[2].record()
                events.append((cc, i, *ev))
        n_chunks += 1
    return n_chunks


def mps_sample(sites, C, seed=None):
    """``C`` configurations drawn from |psi|^2 of an open-boundary MPS, with
    their probabilities: ``MatrixProductState.sample(C, seed)``
    (tn1d/core.py:3943-3990) for (l, p, r) device arrays, all samples at once.

    Returns ``(configs, omegas)``: int64 (C, L) and float64 (C,) numpy arrays;
    ``zip(configs.tolist(), omegas)`` is the reference's sequence of
    ``(config, omega)``.  The uniforms are ``rng.random((C, L))`` of
    ``rng = np.random.default_rng(seed)`` (a Generator, or a
    ``quimb_b200.random.default_rng`` one, is used and advanced by C * L
    doubles), the very draws the reference makes one ``rng.choice`` at a time,
    so the configurations agree sample for sample.  Unlike the reference, the
    selected row is renormalised at every site (no underflow of long chains);
    the distribution and the probabilities are the same.

    float32 / complex64 states are widened once; the caller's sites are left
    untouched.  Raises ``ValueError`` when a probability vector is not finite
    or sums to zero (as ``rng.choice`` does)."""
    import torch
    C = int(C)
    if C < 0:
        raise ValueError("mps_sample: C must be >= 0")
    L = len(sites)
    if C == 0:
        return np.empty((0, L), dtype=np.int64), np.empty((0,), dtype=np.float64)
    rng = _sample_rng(seed)
    psi, nrm = _sample_prepare(sites)
    dev = psi[0].t.device
    u = torch.from_numpy(rng.random((C, L))).to(dev)
    configs = torch.empty((C, L), dtype=torch.int64, device=dev)
    omegas = torch.ones((C,), dtype=torch.float64, device=dev)
    _sample_chunks(psi, u, configs, omegas)
    configs, omegas, nrm = configs.cpu().numpy(), omegas.cpu().numpy(), complex(nrm.item())
    if not (np.isfinite(nrm) and nrm != 0) or (configs < 0).any():
        raise ValueError("mps_sample: probabilities contain NaN or sum to zero")
    return configs, omegas


def mps_sample_configuration(sites, seed=None):
    """One configuration and its probability,
    ``MatrixProductState.sample_configuration(seed)`` (tn1d/core.py:
    3871-3941): ``(list of int, float)``, the first draw of
    :func:`mps_sample` with the same seed."""
    configs, omegas = mps_sample(sites, 1, seed=seed)
    return configs[0].tolist(), float(omegas[0])


# ------------------------------------------------------ MPS compression etc. ---
def left_compress_site(sites, i, **compress_opts):
    """Truncate the bond (i, i+1) leaving site i left-isometric
    (tn1d/core.py:1194-1224: tensor_compress_bond with absorb='right',
    reduced='left'), in place."""
    from .split import tensor_compress_bond
    set_default_compress_mode(compress_opts)
    compress_opts.setdefault("absorb", "right")
    compress_opts.setdefault("reduced", "left")
    sites[i], sites[i + 1] = tensor_compress_bond(
        sites[i], ("l", "p", "x"), sites[i + 1], ("x", "q", "r"), **compress_opts)


def right_compress_site(sites, i, **compress_opts):
    """Truncate the bond (i-1, i) leaving site i right-isometric
    (tn1d/core.py:1226-1256), in place."""
    from .split import tensor_compress_bond
    set_default_compress_mode(compress_opts)
    compress_opts.setdefault("absorb", "left")
    compress_opts.setdefault("reduced", "right")
    sites[i - 1], sites[i] = tensor_compress_bond(
        sites[i - 1], ("l", "p", "x"), sites[i], ("x", "q", "r"), **compress_opts)


def left_compress(sites, start=None, stop=None, **compress_opts):
    start = 0 if start is None else start
    stop = len(sites) - 1 if stop is None else stop
    for i in range(start, stop):
        left_compress_site(sites, i, **compress_opts)


def right_compress(sites, start=None, stop=None, **compress_opts):
    start = len(sites) - 1 if start is None else start
    stop = 0 if stop is None else stop
    for i in range(start, stop, -1):
        right_compress_site(sites, i, **compress_opts)


def mps_compress(sites, form=None, **compress_opts):
    """``MatrixProductState.compress`` (tn1d/core.py:1330-1390): canonise one
    way, sweep truncated SVDs back the other way.  ``form``: 'right' (default,
    centre at site 0), 'left', an integer centre, or 'flat'."""
    import numbers
    n = len(sites)
    if form is None:
        form = "right"
    if isinstance(form, numbers.Integral):
        if form < n // 2:
            left_canonize(sites)
            right_compress(sites, **compress_opts)
            left_canonize(sites, stop=form)
        else:
            right_canonize(sites)
            left_compress(sites, **compress_opts)
            right_canonize(sites, stop=form)
    elif form == "left":
        right_canonize(sites)
        left_compress(sites, **compress_opts)
    elif form == "right":
        left_canonize(sites)
        right_compress(sites, **compress_opts)
    elif form == "flat":
        compress_opts["absorb"] = "both"
        right_compress(sites, stop=n // 2, **compress_opts)
        left_compress(sites, stop=n // 2, **compress_opts)
    else:
        raise ValueError(f"Form specifier {form} not understood, should be either "
                         "'left', 'right', 'flat' or an int specifiying a new orthog "
                         "center.")
    return sites


def mps_overlap(bra, ket):
    """<bra|ket> of two (l, p, r) MPS with matching physical dimensions: two
    launches per site, the bra conjugated on load."""
    return mps_overlap_array(bra, ket).item()


def mps_overlap_array(bra, ket):
    """:func:`mps_overlap` as a 0-d device Array (nothing read back)."""
    E = None
    for A, B in zip(bra, ket):
        if E is None:
            E = ops.ones((A.shape[0], B.shape[0]), dtype=np.result_type(A.dtype, B.dtype),
                         device=B.device)
        if A.dtype != B.dtype or E.dtype != B.dtype:
            dt = np.result_type(A.dtype, B.dtype, E.dtype)
            A, B, E = A.astype(dt, copy=False), B.astype(dt, copy=False), E.astype(dt, copy=False)
        T = contract_pair(E.t, [0, 1], B.t, [1, 2, 3], [0, 2, 3], conj_a=E.cj, conj_b=B.cj)
        E = Array(contract_pair(A.t, [0, 2, 4], T, [0, 2, 3], [4, 3], conj_a=not A.cj))
    return E.reshape(())


def mps_add(a, b):
    """|a> + |b> as an MPS with bond dimensions added (block-diagonal bonds;
    MatrixProductState.add_MPS, tn1d/core.py): pure data placement."""
    import torch
    n = len(a)
    out = []
    for i, (x, y) in enumerate(zip(a, b)):
        xt, yt = x.resolve(), y.resolve()
        if xt.dtype != yt.dtype:
            dt = torch.promote_types(xt.dtype, yt.dtype)
            xt, yt = xt.to(dt), yt.to(dt)
        if n == 1:
            out.append(Array(xt + yt))
        elif i == 0:
            out.append(Array(torch.cat([xt, yt], dim=2)))          # row vector of blocks
        elif i == n - 1:
            out.append(Array(torch.cat([xt, yt], dim=0)))          # column vector
        else:
            (l1, d, r1), (l2, _, r2) = xt.shape, yt.shape
            z = torch.zeros((l1 + l2, d, r1 + r2), dtype=xt.dtype, device=xt.device)
            z[:l1, :, :r1] = xt
            z[l1:, :, r1:] = yt
            out.append(Array(z))
    return out


def mpo_apply(mpo, sites, mpo_shape="lrud", compress=False, **compress_opts):
    """H|psi> as an MPS: new_site[(l, wl), d, (r, wr)] = sum_u A[l, u, r]
    W[wl, wr, u, d] (one launch per site; bond dimensions multiply), optionally
    followed by :func:`mps_compress` (MatrixProductOperator.apply,
    tn1d/core.py)."""
    from .mps import mpo_lrud
    n = len(sites)
    out = []
    for i, A in enumerate(sites):
        W = mpo_lrud(mpo[i], mpo_shape, i, n)
        if W.dtype != A.dtype:
            dt = np.result_type(W.dtype, A.dtype)
            W, A = W.astype(dt, copy=False), A.astype(dt, copy=False)
        T = Array(contract_pair(A.t, [0, 1, 2], W.t, [3, 4, 1, 5], [0, 3, 5, 2, 4],
                                conj_a=A.cj, conj_b=W.cj))
        l, wl, d, r, wr = T.shape
        out.append(T.reshape(l * wl, d, r * wr))
    if compress:
        mps_compress(out, **compress_opts)
    return out
