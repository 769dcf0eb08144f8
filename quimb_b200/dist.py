"""Multi-GPU sharding of the contraction path (SURVEY.md section 8e).

One process per GPU (torchrun); ``torch.distributed`` (NCCL over NVLink on
the GPUs, gloo in the CPU tests) is plumbing only.  What shards naturally on
this path are *independent units with a single exchange at the end*:

  * slices of a contraction tree: cotengra fixes the values of a few indices,
    every assignment is a complete independent contraction and the results
    are summed (quimb/tensor/tensor_core.py:255-259).  Units are dealt
    round-robin to the ranks, summed locally on the device and combined by
    ONE all-reduce of the (small) output -- no collective on the data path;
  * independent networks (many MPS norms / amplitudes): pure replicas.

The DMRG chain itself is sequential (each environment depends on the
previous one, dmrg.py:297-301), but its dominant cost -- the Lanczos matvecs
of the two-site eigensolve -- shards over the left bond with ONE exchange
step per matvec (``BondShard``): rank r owns the row slab a' in [lo_r, hi_r)
of the left environment L[a', w, a] and of every Krylov vector, all-gathers
the input vector (32 MiB at chi = 1024) and all-reduces the handful of inner
products of the re-orthogonalisation.  Everything else of the sweep (SVD,
environment updates) is replicated deterministically on every rank.
"""

import itertools

import torch
import torch.distributed as dist


def world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_units(n_units, rank=None, world_size=None):
    """Round-robin assignment of ``n_units`` independent units."""
    if rank is None or world_size is None:
        rank, world_size = world()
    return list(range(rank, n_units, world_size))


def all_reduce_sum(t):
    """In-place sum over ranks of a torch tensor (no-op without a group)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


def slice_assignments(sliced_inds, size_dict):
    """All value assignments of the sliced indices, in a fixed order."""
    ranges = [range(size_dict[ix]) for ix in sliced_inds]
    return list(itertools.product(*ranges))


def contract_sliced(arrays, inputs, output, sliced_inds=None, optimize="auto",
                    contract_fn=None, rank=None, world_size=None, reduce=True,
                    target_width=None, min_slices=None):
    """Slice-parallel contraction: sum over all assignments of ``sliced_inds``
    of the contraction with those indices fixed; assignments are sharded over
    the ranks and combined with one all-reduce.

    ``sliced_inds=None`` picks the indices with :func:`quimb_b200.tree.
    find_slices` (at least one slice per rank, intermediates of at most
    ``2**target_width`` elements).
    ``contract_fn(arrays, inputs, output, optimize)`` defaults to the device
    tree executor; the CPU tests inject a stand-in to exercise the sharding
    and the collective without a GPU.
    """
    if contract_fn is None:
        from .tree import array_contract as contract_fn
    inputs = [tuple(t) for t in inputs]
    if sliced_inds is None:
        # choose the slices from the tree: enough of them to feed every rank
        # and narrow enough to fit ``target_width`` (log2 elements)
        from .tree import find_slices, find_tree
        sd = {}
        for t, x in zip(inputs, arrays):
            for ix, d in zip(t, x.shape):
                sd[ix] = int(d)
        if min_slices is None:
            min_slices = world()[1] if world_size is None else world_size
        if optimize == "auto-hq" and target_width is not None:
            # tree and slices searched together (tree of the sliced network)
            from .tree import find_sliced_tree
            optimize, sliced_inds = find_sliced_tree(inputs, tuple(output), sd,
                                                     target_width, min_slices)
        else:
            full_tree = find_tree(inputs, tuple(output), sd, optimize)
            sliced_inds = find_slices(full_tree, target_width, min_slices)[0]
    if (rank is None and world_size is None and torch.distributed.is_available()
            and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1):
        # every rank searched for itself (deterministically: tree.py canonicalises
        # index names); rank 0's choice is nevertheless the one all ranks use
        from .tree import Tree
        steps = [(i, j) for i, j, _, _ in optimize.steps] if isinstance(optimize, Tree) else None
        box = [(tuple(sliced_inds), steps)]
        torch.distributed.broadcast_object_list(box, src=0)
        sliced_inds, steps0 = box[0]
        if steps0 is not None and isinstance(optimize, Tree) and steps0 != steps:
            red = [tuple(ix for ix in t if ix not in set(sliced_inds)) for t in inputs]
            optimize = Tree(red, tuple(output), optimize.size_dict, steps0)
    sliced = tuple(sliced_inds)
    if any(ix in output for ix in sliced):
        raise ValueError("cannot slice an output index")
    size_dict = {}
    for t, x in zip(inputs, arrays):
        for ix, d in zip(t, x.shape):
            size_dict[ix] = int(d)
    units = slice_assignments(sliced, size_dict)
    mine = shard_units(len(units), rank, world_size)
    red_inputs = [tuple(ix for ix in t if ix not in sliced) for t in inputs]
    if contract_fn.__module__.endswith("tree") and isinstance(optimize, (str, type(None))):
        # every slice has the same structure: find the tree once
        from .tree import find_tree
        optimize = find_tree(red_inputs, tuple(output), size_dict, optimize)
    total = None
    for u in mine:
        vals = dict(zip(sliced, units[u]))
        sub = []
        for t, x in zip(inputs, arrays):
            idx = tuple(vals[ix] if ix in vals else slice(None) for ix in t)
            sub.append(x[idx])
        part = contract_fn(sub, red_inputs, tuple(output), optimize)
        total = part if total is None else total + part
    if not reduce:
        return total, mine
    return _finish(total, arrays, inputs, output, size_dict), mine


def _finish(total, arrays, inputs, output, size_dict):
    from .array import Array
    t = total.t if isinstance(total, Array) else total
    if t is None:
        # this rank had no unit: contribute zeros of the output shape
        ref = arrays[0]
        rt = ref.t if isinstance(ref, Array) else ref
        shape = [size_dict[ix] for ix in output]
        t = torch.zeros(shape, dtype=rt.dtype if isinstance(rt, torch.Tensor) else torch.float64,
                        device=rt.device if isinstance(rt, torch.Tensor) else "cpu")
    elif not isinstance(t, torch.Tensor):
        t = torch.as_tensor(t)
    t = t.contiguous()
    all_reduce_sum(t)
    return t


class _DevView:
    """Zero-copy torch view of raw device memory (CUDA array interface)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1",
                                         "data": (int(ptr), False), "version": 2}


class PeerExchange:
    """Symmetric peer-memory block of the fused exchange kernels
    (csrc/p2p.cu): allocated by the library with cudaMalloc, exported to the
    peers of the process group through CUDA IPC (handles travel over
    ``all_gather_object``), after which the all-gather of a Krylov vector and
    the all-reduce of a handful of inner products are ONE kernel each that
    stores straight into the peers' HBM over NVLink and spins on flag words
    -- no NCCL call on the data path.  Raises if IPC / peer access is not
    available; ``BondShard(exchange='auto')`` then stays on NCCL."""

    def __init__(self, gather_bytes, group, rank, world_size, device):
        import ctypes
        from . import _lib
        self.lib = lib = _lib.load()
        self.rank, self.world, self.group = rank, world_size, group
        self.gather_bytes = int(gather_bytes)
        self.device = device
        total = lib.qb_p2p_block_bytes(self.gather_bytes)
        ptr = ctypes.c_void_p()
        _lib.check(lib.qb_p2p_alloc(total, ctypes.byref(ptr)), "qb_p2p_alloc")
        self.local = ptr.value
        self.total = total
        handle = (ctypes.c_ubyte * 64)()
        _lib.check(lib.qb_p2p_export(ctypes.c_void_p(self.local), handle), "qb_p2p_export")
        handles = [None] * world_size
        dist.all_gather_object(handles, bytes(handle), group=group)
        self.peers, self._imported = [], []
        ok = 1
        for r, h in enumerate(handles):
            if r == rank:
                self.peers.append(self.local)
                continue
            pp = ctypes.c_void_p()
            buf = (ctypes.c_ubyte * 64).from_buffer_copy(h)
            rc = lib.qb_p2p_import(buf, ctypes.byref(pp))
            if rc != 0:
                ok = 0
                self.peers.append(0)
            else:
                self.peers.append(pp.value)
                self._imported.append(pp.value)
        staged = dist.get_backend(group) != "nccl"
        flag = torch.tensor([ok], dtype=torch.int32, device="cpu" if staged else device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        if int(flag.item()) != 1:
            self.close()
            raise RuntimeError("CUDA IPC peer mapping failed on at least one rank: "
                               + _lib.last_error())
        self.peer_arr = (ctypes.c_void_p * world_size)(*self.peers)
        self.scratch = torch.zeros(2, dtype=torch.int32, device=device)
        self.g_epoch = 0
        self.r_epoch = 0
        self._bytes = torch.as_tensor(_DevView(self.local, total), device=device)
        dist.barrier(group=group)

    def data_view(self, parity, dtype, numel):
        off = self.lib.qb_p2p_data_offset(self.gather_bytes, parity)
        return self._bytes[off:off + numel * dtype.itemsize].view(dtype)

    def all_gather(self, local, dst_off_bytes):
        """Enqueue the push of ``local`` (contiguous) into every rank's gather
        buffer; returns the parity of the buffer that holds the gathered vector
        once the kernel has completed (stream order)."""
        import ctypes
        from . import _lib
        self.g_epoch += 1
        rc = self.lib.qb_p2p_allgather(self.peer_arr, self.world, self.rank,
                                       ctypes.c_void_p(local.data_ptr()),
                                       local.numel() * local.element_size(), int(dst_off_bytes),
                                       self.gather_bytes, self.g_epoch,
                                       ctypes.c_void_p(self.scratch.data_ptr()),
                                       _lib.stream_ptr())
        _lib.check(rc, "qb_p2p_allgather")
        return self.g_epoch & 1

    def all_reduce_small_(self, t):
        import ctypes
        from . import _lib
        self.r_epoch += 1
        rc = self.lib.qb_p2p_allreduce_small(self.peer_arr, self.world, self.rank,
                                             ctypes.c_void_p(t.data_ptr()), t.numel(),
                                             self.r_epoch,
                                             ctypes.c_void_p(self.scratch.data_ptr()),
                                             _lib.stream_ptr())
        _lib.check(rc, "qb_p2p_allreduce_small")
        return t

    def check(self):
        """Raise if a kernel gave up waiting for a peer (bounded spin)."""
        if int(self.scratch[1].item()) != 0:
            raise RuntimeError("quimb_b200 peer exchange: timed out waiting for a peer's flag")

    def close(self, collective=True):
        """Unmap the peers' blocks, then free our own.  Collective by default:
        an exporter must not free its block while a peer still has it mapped
        (CUDA IPC), so all ranks pass a barrier between the two steps."""
        for p in self._imported:
            self.lib.qb_p2p_unimport(p)
        self._imported = []
        if collective and dist.is_available() and dist.is_initialized():
            try:
                dist.barrier(group=self.group)
            except Exception:  # noqa: BLE001  (process group already torn down)
                pass
        if getattr(self, "local", None):
            self.lib.qb_p2p_free(self.local)
            self.local = None


class BondShard:
    """Row-slab sharding of a bond of size ``n`` over the ranks of a process
    group: the exchange layer of the sharded two-site eigensolve.

    ``exchange``: 'p2p' = the fused peer-memory kernels of csrc/p2p.cu (one
    launch per all-gather / small all-reduce, stores over NVLink into the
    peers' HBM), 'nccl' = ``torch.distributed`` collectives, 'auto' = p2p when
    the group runs on NCCL (one GPU per rank) and the IPC mapping succeeds,
    else NCCL.  With the gloo backend (CPU tests, or several ranks sharing one
    GPU in the single-GPU test) the collectives are staged through host memory.
    """

    def __init__(self, group=None, rank=None, world_size=None, exchange="auto"):
        self.group = group
        if rank is None or world_size is None:
            rank, world_size = world()
        self.rank, self.world_size = int(rank), int(world_size)
        self.active = (dist.is_available() and dist.is_initialized()
                       and self.world_size > 1)
        self._stage = self.active and dist.get_backend(group) != "nccl"
        self.bytes_gathered = 0
        if exchange not in ("auto", "p2p", "nccl"):
            raise ValueError("exchange must be 'auto', 'p2p' or 'nccl'")
        self._want = exchange
        self._px = None
        self._px_failed = None
        self.exchange_name = "nccl" if self.active else "none"
        if self._stage:
            self.exchange_name = "gloo (host staged)"

    def _peer_exchange(self, nbytes, device):
        """The PeerExchange for vectors of ``nbytes`` (built on first use; all
        ranks take the same decision)."""
        if not self.active or self._want == "nccl" or self._px_failed:
            return None
        if self._stage and self._want != "p2p":
            return None
        if self._px is not None and self._px.gather_bytes >= nbytes:
            return self._px
        if self._px is not None:
            self._px.close()
            self._px = None
        try:
            self._px = PeerExchange(nbytes, self.group, self.rank, self.world_size, device)
            self.exchange_name = "p2p (fused peer-memory kernels over NVLink, CUDA IPC)"
        except Exception as e:  # noqa: BLE001
            if self._want == "p2p":
                raise
            self._px_failed = str(e)
            self.exchange_name = f"nccl (p2p unavailable: {self._px_failed[:80]})"
        return self._px

    def slab(self, n, rank=None):
        """[lo, hi) of this rank's rows of a bond of size ``n`` (balanced)."""
        r = self.rank if rank is None else rank
        return (n * r) // self.world_size, (n * (r + 1)) // self.world_size

    def all_reduce_(self, t):
        if not self.active:
            return t
        if (self._px is not None and t.dtype == torch.float64 and t.numel() <= 64
                and t.is_contiguous() and t.device.type == "cuda"):
            return self._px.all_reduce_small_(t)
        if self._stage and t.device.type != "cpu":
            h = t.cpu()
            dist.all_reduce(h, op=dist.ReduceOp.SUM, group=self.group)
            t.copy_(h)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t

    def all_gather_rows(self, local, n, transient=False):
        """Concatenate the row slabs ``local`` (rows_r, cols) of all ranks into
        the full (n, cols) matrix, identical on every rank.  ``transient``: the
        caller consumes the result before the next gather is enqueued on this
        stream, so the p2p path may return a view of its gather buffer instead
        of a copy.  (Once this rank's next gather has run, a peer may start the
        one after it, whose push overwrites the buffer of the view.)"""
        cols = local.shape[1]
        if not self.active:
            return local
        nbytes = n * cols * local.element_size()
        self.bytes_gathered += nbytes
        even = n % self.world_size == 0
        px = None
        if even and local.dtype == torch.float64 and (nbytes // self.world_size) % 16 == 0:
            px = self._peer_exchange(nbytes, local.device)
        if px is not None:
            lo, _ = self.slab(n)
            src = local.contiguous()
            parity = px.all_gather(src, lo * cols * local.element_size())
            full = px.data_view(parity, local.dtype, n * cols).view(n, cols)
            return full if transient else full.clone()
        full = torch.empty((n, cols), dtype=local.dtype, device=local.device)
        if even and not self._stage:
            dist.all_gather_into_tensor(full, local.contiguous(), group=self.group)
            return full
        # ragged slabs / staged backend: pad every slab to the largest one
        rows = max(self.slab(n, r)[1] - self.slab(n, r)[0] for r in range(self.world_size))
        src = local.cpu() if self._stage else local
        pad = torch.zeros((rows, cols), dtype=src.dtype, device=src.device)
        pad[: src.shape[0]].copy_(src)
        parts = [torch.empty_like(pad) for _ in range(self.world_size)]
        dist.all_gather(parts, pad, group=self.group)
        for r, part in enumerate(parts):
            lo, hi = self.slab(n, r)
            full[lo:hi].copy_(part[: hi - lo])
        return full

    def check(self):
        if self._px is not None:
            self._px.check()

    def close(self):
        if self._px is not None:
            self._px.close()
            self._px = None


def mps_norm2_two_ended(sites, shape="lrp", group=None):
    """<psi|psi> with the chain contracted from both ends at once (SURVEY.md
    8e, cfg2): rank 0 carries the (chi, chi) environment in from the left over
    the first half of the sites, rank 1 from the right over the second half;
    ONE broadcast of the 8 MiB right environment (chi = 1024) and one
    (chi x chi) . (chi x chi) trace join them.  Each rank needs only its half
    of the site tensors resident (pass ``None`` for the others).  Beyond two
    ranks the chain does not shard this way (replicas only); without a process
    group both halves run locally.  Returns a 0-d device Array (identical on
    all ranks)."""
    from . import ops
    from .array import Array
    from .contract import contract_pair
    from .mps import norm_step, norm_step_right, site_lpr
    n = len(sites)
    if n < 2:
        from .mps import mps_norm2
        return mps_norm2(sites, shape)
    half = n // 2
    active = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
    rank = dist.get_rank(group) if active else 0

    def left():
        E = None
        for i in range(half):
            A = site_lpr(sites[i], shape, i, n)
            if E is None:
                E = ops.eye(A.shape[0], dtype=A.dtype, device=A.device)
            E = norm_step(E, A)
        return E

    def right():
        E = None
        for i in range(n - 1, half - 1, -1):
            A = site_lpr(sites[i], shape, i, n)
            if E is None:
                E = ops.eye(A.shape[2], dtype=A.dtype, device=A.device)
            E = norm_step_right(E, A)
        return E

    if not active:
        EL, ER = left(), right()
    else:
        EL = left() if rank == 0 else None
        ER = right() if rank == 1 else None
        stage = dist.get_backend(group) != "nccl"
        out = []
        for src, E in ((0, EL), (1, ER)):
            meta = [None]
            if rank == src:
                meta[0] = (tuple(E.shape), str(E.t.dtype))
            dist.broadcast_object_list(meta, src=src, group=group)
            shp, dt = meta[0]
            if rank == src:
                buf = ops.materialize(E, force=True).t
            else:
                buf = torch.empty(shp, dtype=getattr(torch, dt.split(".")[-1]),
                                  device=ops.default_device())
            wire = torch.view_as_real(buf) if buf.dtype.is_complex else buf
            if stage and wire.device.type != "cpu":
                host = wire.cpu()
                dist.broadcast(host, src=src, group=group)
                wire.copy_(host)
            else:
                dist.broadcast(wire, src=src, group=group)
            out.append(Array(buf))
        EL, ER = out
    # <psi|psi> = sum_{a', a} EL[a', a] ER[a', a]
    return Array(contract_pair(EL.t, [0, 1], ER.t, [0, 1], [], conj_a=EL.cj, conj_b=ER.cj))
