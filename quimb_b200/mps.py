"""1D structured contractions on the device: the callers either side of the
pairwise kernel for BASELINE config 2 (MPS norm / expectation) and for the
DMRG environments.

Mirrors (numerically, not structurally) quimb's
``TensorNetwork1D.contract_structured`` / ``expec_TN_1D``
(quimb/tensor/tn1d/core.py:55-95, 502-557) and ``TensorNetwork.norm``
(quimb/tensor/tensor_core.py:4879-4918): the network is swept left to right
carrying a (chi, chi) [or (chi, w, chi)] environment.  Each site costs
4 d chi^3 flops in two launches of the contraction kernel; the bra is never
materialised -- conjugation is a load flag of the kernel -- and site arrays
are consumed in whatever layout they come in (strided views, no copies).

Layouts: every function takes the index order of the site arrays as a string
over {l, r, p} (quimb's default is 'lrp', tn1d/core.py:1801) and of MPO sites
over {l, r, u, d} (quimb's 'lrud': u = ket-side 'k' index, d = bra-side 'b'
index).  End sites may omit their dangling bond, as quimb's do.
"""

from . import ops
from .array import Array
from .contract import contract_pair

# integer mode labels handed to the kernel
L_, P_, R_, LB_, PB_, RB_, W_, WN_ = range(8)


def site_lpr(x, shape, i, n):
    """Free (l, p, r) view of site ``i`` of ``n`` given its layout string."""
    x = ops.asarray(x)
    lay = shape
    if x.ndim == len(shape) - 1:
        if i == 0 and "l" in lay:
            lay = lay.replace("l", "")
        elif i == n - 1 and "r" in lay:
            lay = lay.replace("r", "")
    if x.ndim != len(lay):
        raise ValueError(f"site {i}: rank {x.ndim} does not fit layout {shape!r}")
    t = x.t
    for c in "lpr":
        if c not in lay:
            t = t.unsqueeze(-1)
            lay = lay + c
    return Array(t.permute(lay.index("l"), lay.index("p"), lay.index("r")), x.cj)


def mpo_lrud(w, shape, i, n):
    """Free (l, r, u, d) view of MPO site ``i`` of ``n``."""
    w = ops.asarray(w)
    lay = shape
    if w.ndim == len(shape) - 1:
        if i == 0 and "l" in lay:
            lay = lay.replace("l", "")
        elif i == n - 1 and "r" in lay:
            lay = lay.replace("r", "")
    if w.ndim != len(lay):
        raise ValueError(f"MPO site {i}: rank {w.ndim} does not fit {shape!r}")
    t = w.t
    for c in "lrud":
        if c not in lay:
            t = t.unsqueeze(-1)
            lay = lay + c
    return Array(t.permute(*(lay.index(c) for c in "lrud")), w.cj)


def norm_step(E, A, B=None):
    """E'[b', b] = sum_{a', a, p} E[a', a] conj(B)[a', p, b'] A[a, p, b]

    ``B`` (the bra site, default ``A``) may have other bonds than ``A``: the
    overlap <phi|psi> of two states carries a (chi_phi, chi_psi) environment."""
    B = A if B is None else B
    T = contract_pair(E.t, [LB_, L_], A.t, [L_, P_, R_], [LB_, P_, R_],
                      conj_a=E.cj, conj_b=A.cj)
    return Array(contract_pair(B.t, [LB_, P_, RB_], T, [LB_, P_, R_],
                               [RB_, R_], conj_a=not B.cj))


def _is_host(x):
    import numpy as np
    import torch
    if isinstance(x, np.ndarray):
        return True
    return isinstance(x, torch.Tensor) and x.device.type == "cpu"


_STAGE_RING = {}


def stream_sites(sites, copy_stream=None, depth=3):
    """Iterate over site arrays, staging host-resident sites to the device
    ``depth`` sites ahead on a side stream so the H2D copies overlap the
    contraction of the previous sites (pinned host memory makes the copies
    truly asynchronous).

    Host sites land in a fixed RING of ``depth + 1`` device staging buffers
    (allocated once per device / dtype / size, reused across calls): no
    allocator traffic on the path, and a buffer is overwritten only after the
    main stream has passed the work that consumed it (event recorded when the
    consumer asks for the next site).  The yielded device tensors are therefore
    TRANSIENT views: valid until ``depth`` further sites have been requested.
    A consumer that stops early closes the generator: that orders the main
    stream after the copies still in flight into the ring."""
    import torch
    if not any(_is_host(s) for s in sites):
        yield from sites
        return
    dev = ops.default_device()
    main = torch.cuda.current_stream(dev)
    side = copy_stream or torch.cuda.Stream(device=dev)
    side.wait_stream(main)
    nbuf = depth + 1

    def as_tensor(s):
        return s if isinstance(s, torch.Tensor) else torch.from_numpy(s)

    hosts = [as_tensor(s) if _is_host(s) else None for s in sites]
    need = {}
    for h in hosts:
        if h is not None:
            need[h.dtype] = max(need.get(h.dtype, 0), h.numel())
    rings = {}
    for dt, n in need.items():
        key = (dev.index, dt, nbuf)
        ring = _STAGE_RING.get(key)
        if ring is None or ring[0].numel() < n:
            ring = [torch.empty(n, dtype=dt, device=dev) for _ in range(nbuf)]
            _STAGE_RING[key] = ring
        rings[dt] = ring
    consumed = {dt: [None] * nbuf for dt in need}     # main-stream events per slot
    count = {dt: 0 for dt in need}
    pending = []

    def issue(i):
        h = hosts[i]
        if h is None:
            return (sites[i], None, None)
        dt = h.dtype
        slot = count[dt] % nbuf
        count[dt] += 1
        buf = rings[dt][slot][:h.numel()].view(h.shape)
        with torch.cuda.stream(side):
            if consumed[dt][slot] is not None:
                side.wait_event(consumed[dt][slot])
            buf.copy_(h, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(side)
        return (buf, ev, (dt, slot))

    n = len(sites)
    nxt = 0
    try:
        while nxt < n and len(pending) < depth:
            pending.append(issue(nxt))
            nxt += 1
        prev = None
        while pending:
            d, ev, where = pending.pop(0)
            if prev is not None:
                # everything the consumer enqueued for the previous site is on
                # the main stream by now: its staging slot may be refilled after
                main_done = torch.cuda.Event()
                main_done.record(main)
                consumed[prev[0]][prev[1]] = main_done
            if nxt < n:
                pending.append(issue(nxt))
                nxt += 1
            if ev is not None:
                main.wait_event(ev)
            prev = where
            yield d
    finally:
        # a consumer that stops early leaves copies into the shared ring in
        # flight: order the main stream after them, so the next call (whose
        # side stream starts behind the main stream) cannot race them
        main.wait_stream(side)


def mps_norm2(sites, shape="lrp", copy_stream=None):
    """<psi|psi> of an MPS given as device arrays, or as host arrays (numpy /
    pinned torch tensors) that are streamed to the device while contracting;
    returns a 0-d device Array."""
    n = len(sites)
    E = None
    staged = stream_sites(sites, copy_stream)
    try:
        for i, s in enumerate(staged):
            A = site_lpr(s, shape, i, n)
            if E is None:
                E = ops.ones((A.shape[0], A.shape[0]), dtype=A.dtype, device=A.device)
                if A.shape[0] != 1:
                    E = ops.eye(A.shape[0], dtype=A.dtype, device=A.device)
            E = norm_step(E, A)
    finally:
        staged.close()           # an error midway: settle the staging copies now
    if E.shape != (1, 1):
        return ops.trace(E)
    return E.reshape(())


def mps_norm(sites, shape="lrp"):
    return ops.sqrt(ops.real(mps_norm2(sites, shape)))


def env_left_step(E, A, W):
    """E'[b', w', b] = sum E[a', w, a] A[a, p, b] W[w, w', p, q] conj(A)[a', q, b']

    Order E.A -> .W -> .conj(A): 2 d w chi^3 + 2 w^2 d^2 chi^2 + 2 d w chi^3
    flops (the MovingEnvironment update, quimb/tensor/tn1d/dmrg.py:383-405)."""
    T = contract_pair(E.t, [LB_, W_, L_], A.t, [L_, P_, R_], [LB_, W_, P_, R_],
                      conj_a=E.cj, conj_b=A.cj)
    T = contract_pair(T, [LB_, W_, P_, R_], W.t, [W_, WN_, P_, PB_],
                      [LB_, PB_, WN_, R_], conj_b=W.cj)
    return Array(contract_pair(A.t, [LB_, PB_, RB_], T, [LB_, PB_, WN_, R_],
                               [RB_, WN_, R_], conj_a=not A.cj))


def env_right_step(E, A, W):
    """E'[a', w, a] = sum A[a, p, b] E[b', w', b] W[w, w', p, q] conj(A)[a', q, b']"""
    T = contract_pair(A.t, [L_, P_, R_], E.t, [RB_, WN_, R_], [L_, P_, WN_, RB_],
                      conj_a=A.cj, conj_b=E.cj)
    T = contract_pair(W.t, [W_, WN_, P_, PB_], T, [L_, P_, WN_, RB_],
                      [W_, L_, PB_, RB_], conj_a=W.cj)
    return Array(contract_pair(A.t, [LB_, PB_, RB_], T, [W_, L_, PB_, RB_],
                               [LB_, W_, L_], conj_a=not A.cj))


def mps_expec(sites, mpo, shape="lrp", mpo_shape="lrud"):
    """<psi|H|psi> (quimb's expec_TN_1D(bra, mpo, ket)); 0-d Array."""
    n = len(sites)
    E = None
    for i in range(n):
        A = site_lpr(sites[i], shape, i, n)
        W = mpo_lrud(mpo[i], mpo_shape, i, n)
        if W.dtype != A.dtype:
            W = W.astype(A.dtype)
        if E is None:
            E = ops.ones((1, 1, 1), dtype=A.dtype, device=A.device)
        E = env_left_step(E, A, W)
    return E.reshape(())


# labels of the second MPO layer of <psi|H.H|psi>: its bonds and the
# physical index between the two layers
W2_, WN2_, M_ = 8, 9, 10


def env2_left_step(E, A, W):
    """Two-layer step of <psi|H.H|psi>, ket-side layer first (the reference's
    ``TN_energy2``, tn1d/dmrg.py:1219-1225):

    E'[b', w1', w2', b] = sum E[a', w1, w2, a] A[a, p, b] W[w1, w1', p, m]
                              W[w2, w2', m, q] conj(A)[a', q, b']

    Four launches of the contraction kernel, 2 d w^2 chi^3 (x2) +
    2 d^2 w^3 chi^2 (x2) flops."""
    T = contract_pair(E.t, [LB_, W_, W2_, L_], A.t, [L_, P_, R_],
                      [LB_, W_, W2_, P_, R_], conj_a=E.cj, conj_b=A.cj)
    T = contract_pair(T, [LB_, W_, W2_, P_, R_], W.t, [W_, WN_, P_, M_],
                      [LB_, M_, WN_, W2_, R_], conj_b=W.cj)
    T = contract_pair(T, [LB_, M_, WN_, W2_, R_], W.t, [W2_, WN2_, M_, PB_],
                      [LB_, PB_, WN_, WN2_, R_], conj_b=W.cj)
    return Array(contract_pair(A.t, [LB_, PB_, RB_], T, [LB_, PB_, WN_, WN2_, R_],
                               [RB_, WN_, WN2_, R_], conj_a=not A.cj))


def env2_right_step(E, A, W):
    """E'[a', w1, w2, a] = sum A[a, p, b] E[b', w1', w2', b] W[w1, w1', p, m]
    W[w2, w2', m, q] conj(A)[a', q, b']  (mirror of :func:`env2_left_step`)"""
    T = contract_pair(A.t, [L_, P_, R_], E.t, [RB_, WN_, WN2_, R_],
                      [L_, P_, WN_, WN2_, RB_], conj_a=A.cj, conj_b=E.cj)
    T = contract_pair(W.t, [W_, WN_, P_, M_], T, [L_, P_, WN_, WN2_, RB_],
                      [W_, L_, M_, WN2_, RB_], conj_a=W.cj)
    T = contract_pair(W.t, [W2_, WN2_, M_, PB_], T, [W_, L_, M_, WN2_, RB_],
                      [W_, W2_, L_, PB_, RB_], conj_a=W.cj)
    return Array(contract_pair(A.t, [LB_, PB_, RB_], T, [W_, W2_, L_, PB_, RB_],
                               [LB_, W_, W2_, L_], conj_a=not A.cj))


def mps_expec2(sites, mpo, shape="lrp", mpo_shape="lrud"):
    """<psi|H.H|psi> (the reference's ``TN_energy2 ^ ...``,
    tn1d/dmrg.py:1219-1227): with :func:`mps_expec`, the energy variance
    <H^2> - <H>^2 that certifies an eigenstate; 0-d Array."""
    n = len(sites)
    E = None
    for i in range(n):
        A = site_lpr(sites[i], shape, i, n)
        W = mpo_lrud(mpo[i], mpo_shape, i, n)
        if W.dtype != A.dtype:
            W = W.astype(A.dtype)
        if E is None:
            E = ops.ones((1, 1, 1, 1), dtype=A.dtype, device=A.device)
        E = env2_left_step(E, A, W)
    return E.reshape(())


# ------------------------------------------------------------ environments ---
def compute_left_environments(sites, mpo=None, shape="lrp", mpo_shape="lrud"):
    """Left environments of <psi|psi> (``mpo=None``: (chi, chi) arrays) or
    <psi|H|psi> ((chi, w, chi) arrays), indexed by the site they are to the
    left of: keys 1 .. L-1 (tn1d/core.py:559-580).  All environments stay
    resident on the device (40 MiB each at chi = 1024, w = 5)."""
    n = len(sites)
    envs, E = {}, None
    for i in range(n - 1):
        A = site_lpr(sites[i], shape, i, n)
        if mpo is None:
            if E is None:
                E = ops.eye(A.shape[0], dtype=A.dtype, device=A.device)
            E = norm_step(E, A)
        else:
            W = mpo_lrud(mpo[i], mpo_shape, i, n)
            if W.dtype != A.dtype:
                W = W.astype(A.dtype)
            if E is None:
                E = ops.ones((1, 1, 1), dtype=A.dtype, device=A.device)
            E = env_left_step(E, A, W)
        envs[i + 1] = E
    return envs


def norm_step_right(E, A, B=None):
    """E'[a', a] = sum_{b', b, p} conj(B)[a', p, b'] A[a, p, b] E[b', b]
    (``B``: the bra site, default ``A``)"""
    B = A if B is None else B
    T = contract_pair(A.t, [L_, P_, R_], E.t, [RB_, R_], [L_, P_, RB_],
                      conj_a=A.cj, conj_b=E.cj)
    return Array(contract_pair(B.t, [LB_, P_, RB_], T, [L_, P_, RB_],
                               [LB_, L_], conj_a=not B.cj))


def compute_right_environments(sites, mpo=None, shape="lrp", mpo_shape="lrud"):
    """Right environments, indexed by the site they are to the right of: keys
    0 .. L-2 (tn1d/core.py:582-605)."""
    n = len(sites)
    envs, E = {}, None
    for i in range(n - 1, 0, -1):
        A = site_lpr(sites[i], shape, i, n)
        if mpo is None:
            if E is None:
                E = ops.eye(A.shape[2], dtype=A.dtype, device=A.device)
            E = norm_step_right(E, A)
        else:
            W = mpo_lrud(mpo[i], mpo_shape, i, n)
            if W.dtype != A.dtype:
                W = W.astype(A.dtype)
            if E is None:
                E = ops.ones((1, 1, 1), dtype=A.dtype, device=A.device)
            E = env_right_step(E, A, W)
        envs[i - 1] = E
    return envs


class MovingEnvironment:
    """Left / right environments of <psi|H|psi> around a moving window of
    ``bsz`` sites (quimb/tensor/tn1d/dmrg.py:105-443, open boundaries): all
    environments on the far side are built once (``init_segment`` :281-322),
    moving the window by one site contracts the site left behind into the near
    environment (:383-425).  ``sites`` is the live list of (l, p, r) arrays the
    caller keeps updating.

    ``envs`` maps a window start ``i`` to ``(L_i, R_i)`` with L_i the
    contraction of sites < i and R_i of sites >= i + bsz.  Like the reference,
    environments of visited positions stay cached (40 MiB each at chi = 1024,
    w = 5: 4 GB for L = 100 out of an 80 GB device) and are overwritten when the window
    comes back after the sites changed."""

    def __init__(self, sites, mpo, begin="left", bsz=2):
        if begin not in ("left", "right"):
            raise ValueError("begin must be 'left' or 'right'")
        self.sites, self.mpo = sites, mpo
        self.L, self.bsz, self.begin = len(sites), int(bsz), begin
        self.lenv, self.renv = {}, {}
        A = sites[0]
        one = ops.ones((1, 1, 1), dtype=A.dtype, device=A.device)
        last = self.L - self.bsz
        if begin == "left":
            self.pos = 0
            self.lenv[0] = one
            self.renv[last] = one
            for i in range(last, 0, -1):
                k = i + self.bsz - 1
                self.renv[i - 1] = env_right_step(self.renv[i], sites[k], mpo[k])
        else:
            self.pos = last
            self.renv[last] = one
            self.lenv[0] = one
            for i in range(0, last):
                self.lenv[i + 1] = env_left_step(self.lenv[i], sites[i], mpo[i])

    def move_right(self):
        i = self.pos
        if i + 1 > self.L - self.bsz:
            raise ValueError("window already at the right end")
        self.lenv[i + 1] = env_left_step(self.lenv[i], self.sites[i], self.mpo[i])
        self.pos = i + 1

    def move_left(self):
        i = self.pos
        if i - 1 < 0:
            raise ValueError("window already at the left end")
        k = i + self.bsz - 1
        self.renv[i - 1] = env_right_step(self.renv[i], self.sites[k], self.mpo[k])
        self.pos = i - 1

    def move_to(self, i):
        """dmrg.py:427-443: step until the window starts at site ``i``."""
        while self.pos < i:
            self.move_right()
        while self.pos > i:
            self.move_left()

    def __call__(self):
        return self.lenv[self.pos], self.renv[self.pos]


def mpo_ham_heis(L, j=1.0, bz=0.0, dtype="float64"):
    """Host arrays of the open Heisenberg chain MPO, H = sum_i j S_i.S_{i+1}
    - bz sum_i S^z_i, bond dimension 5 (one row / column per two-site term
    plus identity / finish), the same operator as quimb's ``MPO_ham_heis``
    (tensor_builder.py:5501 through ``spin_ham_mpo_tensor`` :4856-4947).
    Sites are (l, r, d, u) arrays ('lrdu'; the real form uses i S^y, which is
    antisymmetric), end sites keep a size-1 outer bond.  Synthetic-input
    builder for the benchmarks and examples -- the drop-in route takes quimb's
    own MPO tensors."""
    import numpy as np
    sx = np.array([[0, 0.5], [0.5, 0]])
    isy = np.array([[0, 0.5], [-0.5, 0]])
    sz = np.array([[0.5, 0], [0, -0.5]])
    W = np.zeros((5, 5, 2, 2))
    W[0, 0] = W[4, 4] = np.eye(2)
    W[4, 1], W[1, 0] = sx, j * sx
    W[4, 2], W[2, 0] = isy, -j * isy
    W[4, 3], W[3, 0] = sz, j * sz
    W[4, 0] = -bz * sz
    sites = []
    for i in range(L):
        w = W[4:5] if i == 0 else (W[:, 0:1] if i == L - 1 else W)
        sites.append(np.ascontiguousarray(w.astype(dtype)))
    return sites


class ChainPlan:
    """A structured chain contraction captured ONCE into a CUDA graph and
    replayed: the device-resident plan for ``contract_structured`` /
    ``compute_left/right_environments`` / ``MovingEnvironment.init_segment``
    (quimb/tensor/tn1d/core.py:502-607, tn1d/dmrg.py:281-322; SURVEY 8f rank 2).

    ``kind``: 'norm' (<psi|psi>), 'expec' (<psi|H|psi>), 'left_envs' /
    'right_envs' (all environments, of the norm network when ``mpo`` is None).
    The site (and MPO) arrays are copied into static device buffers owned by
    the plan; ``update(i, array)`` / ``update_all(sites)`` refresh them in place
    and ``__call__`` replays the whole chain -- hundreds of launches of the
    contraction kernel, their workspaces and intermediates -- with one graph
    launch and no host work per site.  Outputs are the plan's own buffers
    (clone to keep across replays); so is the contraction scratch the graph
    uses (``contract.capture_graph``), so plans may be replayed in any order
    and on different streams at once."""

    def __init__(self, sites, mpo=None, shape="lrp", mpo_shape="lrud", kind="norm"):
        from .contract import capture_graph
        if kind not in ("norm", "expec", "left_envs", "right_envs"):
            raise ValueError(f"unknown plan kind {kind!r}")
        if kind == "expec" and mpo is None:
            raise ValueError("kind='expec' needs an MPO")
        self.kind, self.shape, self.mpo_shape = kind, shape, mpo_shape
        self.sites = [ops.materialize(ops.asarray(s), force=True) for s in sites]
        self.mpo = None if mpo is None else [ops.materialize(ops.asarray(w), force=True)
                                             for w in mpo]
        self.graph, self.out, self._scratch = capture_graph(self._run)
        self.replays = 0

    def _run(self):
        if self.kind == "norm":
            return mps_norm2(self.sites, self.shape)
        if self.kind == "expec":
            return mps_expec(self.sites, self.mpo, self.shape, self.mpo_shape)
        fn = compute_left_environments if self.kind == "left_envs" else compute_right_environments
        return fn(self.sites, self.mpo, self.shape, self.mpo_shape)

    def update(self, i, array):
        a = ops.asarray(array)
        if tuple(a.shape) != tuple(self.sites[i].shape):
            raise ValueError("shape mismatch with the captured plan")
        self.sites[i].t.copy_(a.resolve())

    def update_all(self, sites):
        if len(sites) != len(self.sites):
            raise ValueError("wrong number of sites")
        for i, s in enumerate(sites):
            self.update(i, s)

    def __call__(self, sites=None):
        if sites is not None:
            self.update_all(sites)
        self.graph.replay()
        self.replays += 1
        return self.out
