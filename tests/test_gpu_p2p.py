"""GPU tier: the peer-memory exchange kernels of csrc/p2p.cu against exact
oracles.

Virtual ranks in one process: every rank owns a block from qb_p2p_alloc, the
peer array is simply the list of those device pointers (no IPC), and each rank
issues its calls on its own stream.  Kernels of different streams run
concurrently, so the ranks really wait on each other's flags.  Every byte of
every block is compared with a model image after each pass:
  * the all-gather is a bitwise copy: the gather buffer of parity e & 1 holds
    the concatenated slabs, everything else keeps its sentinel or the previous
    epoch, flag word r holds the epoch for r < world and 0 above;
  * the all-reduce is the sequential IEEE sum in rank order starting from rank
    0's partial, bit-identical on every rank, and the identity on one rank.
The module also runs two processes sharing one GPU through CUDA IPC
(tests/p2p_worker.py) and provides the process-group runner that every GPU
test spawning processes uses.

Skipped under CUDA_LAUNCH_BLOCKING=1: serialised launches cannot overlap two
ranks, and a rank would wait out the kernels' 4 s bound.  No test depends on
reaching that bound.
"""

import ctypes
import os
import signal
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from quimb_b200 import _lib
from quimb_b200.dist import _DevView

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(os.environ.get("CUDA_LAUNCH_BLOCKING") == "1",
                       reason="serialised launches cannot overlap the virtual ranks"),
]

# layout of a symmetric block (csrc/p2p.cu)
GFLAG, RFLAG, RSLOT, DATA = 0, 4096, 8192, 65536
MAX_RANKS, RMAX = 16, 64
SENT = 0xA5        # sentinel of the blocks' data, slot and padding bytes
XSENT = 0x5A       # sentinel past every slab in the callers' x buffers


# ------------------------------------------------------------ process groups
def run_process_group(cmd, timeout, cwd=ROOT, env=None):
    """Run ``cmd`` as the leader of a new process group and return
    ``(returncode, stdout, stderr)``.  On a timeout, a failure or an
    interruption the whole group is killed, so that workers a launcher
    started (``torch.distributed.run``) do not outlive it holding the GPU;
    the launcher itself is always reaped."""
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                            cwd=cwd, env=env, start_new_session=True)
    try:
        out, err = proc.communicate(timeout=timeout)
    except BaseException:
        _kill_group(proc.pid)
        out, err = proc.communicate()
        if proc.returncode is None:
            proc.wait()
        raise
    if proc.returncode != 0:
        _kill_group(proc.pid)
    return proc.returncode, out, err


def _kill_group(pgid):
    try:
        os.killpg(pgid, signal.SIGKILL)
    except ProcessLookupError:
        pass


def free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def torchrun_cmd(script, nproc, *args):
    return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
            "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
            "--master-port", str(free_port()), os.path.join(ROOT, "tests", script), *args]


# ------------------------------------------------------------- virtual ranks
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bytes(a):
    """uint8 device tensor of a numpy array's bytes."""
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


class VirtualRanks:
    """``world`` symmetric blocks in this process, one stream and one zeroed
    scratch per rank, and the model image every block must equal."""

    def __init__(self, world, gather_bytes):
        self.lib = _lib.load()
        self.world, self.gather = world, int(gather_bytes)
        self.g = (self.gather + 255) // 256 * 256
        self.total = int(self.lib.qb_p2p_block_bytes(self.gather))
        self.ptrs = []

    def __enter__(self):
        try:
            for _ in range(self.world):
                p = ctypes.c_void_p()
                _lib.check(self.lib.qb_p2p_alloc(self.total, ctypes.byref(p)), "qb_p2p_alloc")
                self.ptrs.append(p.value)
            self.peers = (ctypes.c_void_p * self.world)(*self.ptrs)
            self.blocks = [torch.as_tensor(_DevView(p, self.total), device="cuda")
                           for p in self.ptrs]
            self.streams = [torch.cuda.Stream() for _ in range(self.world)]
            self.scratch = [torch.zeros(2, dtype=torch.int32, device="cuda")
                            for _ in range(self.world)]
            # everything but the flag words carries the sentinel; the flags
            # stay 0 because they must be monotone
            self.image = torch.full((self.total,), SENT, dtype=torch.uint8, device="cuda")
            self.image[GFLAG:GFLAG + 8 * MAX_RANKS] = 0
            self.image[RFLAG:RFLAG + 8 * MAX_RANKS] = 0
            for b in self.blocks:
                b.copy_(self.image)
            torch.cuda.synchronize()
        except BaseException:
            self.__exit__()
            raise
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.blocks = None
        for p in self.ptrs:
            self.lib.qb_p2p_free(ctypes.c_void_p(p))
        self.ptrs = []

    # -- calls
    def allgather(self, r, x, nbytes, dst_off, epoch):
        with torch.cuda.stream(self.streams[r]):
            rc = self.lib.qb_p2p_allgather(
                self.peers, self.world, r, ctypes.c_void_p(x), nbytes, dst_off, self.gather,
                epoch, ctypes.c_void_p(self.scratch[r].data_ptr()),
                ctypes.c_void_p(self.streams[r].cuda_stream))
        assert rc == 0, _lib.last_error()

    def allreduce(self, r, x, m, epoch):
        with torch.cuda.stream(self.streams[r]):
            rc = self.lib.qb_p2p_allreduce_small(
                self.peers, self.world, r, ctypes.c_void_p(x), m, epoch,
                ctypes.c_void_p(self.scratch[r].data_ptr()),
                ctypes.c_void_p(self.streams[r].cuda_stream))
        assert rc == 0, _lib.last_error()

    def parity_view(self, r, epoch):
        off = DATA + (epoch & 1) * self.g
        return self.blocks[r][off:off + self.gather]

    # -- model
    def model_gather(self, epoch, full):
        self.image[GFLAG:GFLAG + 8 * self.world].view(torch.int64).fill_(epoch)
        if self.gather:
            off = DATA + (epoch & 1) * self.g
            self.image[off:off + self.gather] = full

    def model_reduce(self, epoch, partials):
        self.image[RFLAG:RFLAG + 8 * self.world].view(torch.int64).fill_(epoch)
        m = partials.shape[1]
        slot = RSLOT + (epoch & 1) * MAX_RANKS * RMAX * 8
        for r in range(self.world):
            if m:
                self.image[slot + r * RMAX * 8:slot + r * RMAX * 8 + 8 * m] = _bytes(partials[r])

    # -- checks
    def check(self, what):
        torch.cuda.synchronize()
        words = torch.stack(self.scratch).cpu().tolist()
        assert all(w == [0, 0] for w in words), f"{what}: (counter, error) per rank {words}"
        for r, b in enumerate(self.blocks):
            if not torch.equal(b, self.image):
                bad = (b != self.image).nonzero().flatten()
                first = int(bad[0])
                raise AssertionError(
                    f"{what}: rank {r}: {bad.numel()} bytes differ from the model, first at "
                    f"{first} ({self.region(first)}): got {b[first:first + 8].tolist()}, "
                    f"want {self.image[first:first + 8].tolist()}")

    def region(self, off):
        if off < RFLAG:
            return "gather flags" if off < 8 * MAX_RANKS else "gather flag padding"
        if off < RSLOT:
            return "reduce flags" if off < RFLAG + 8 * MAX_RANKS else "reduce flag padding"
        if off < DATA:
            return "reduce slots / padding"
        q, rest = divmod(off - DATA, self.g) if self.g else (2, 0)
        if q >= 2:
            return "tail past both gather buffers"
        return f"gather parity {q}, byte {rest}" + (" (past gather_bytes)" if rest >= self.gather
                                                    else "")


def _slab_buffers(sizes, gen, fill=None):
    """One x buffer per rank: random uint8 slab at a 16-byte aligned offset
    that is not 256-aligned except for rank 0, XSENT around it.  Returns the
    (storage, pointer, slab view) triples."""
    out = []
    for r, nbytes in enumerate(sizes):
        off = (16 * r) % 256
        buf = torch.full((off + nbytes + 256,), XSENT, dtype=torch.uint8, device="cuda")
        slab = buf[off:off + nbytes]
        if nbytes:
            slab.copy_(torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda",
                                     generator=gen) if fill is None else fill[r])
        out.append((buf, buf.data_ptr() + off, slab))
    return out


def _gather_epochs(world, n16s, epochs=3, seed=0):
    sizes = [16 * n for n in n16s]
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(int).tolist()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    with VirtualRanks(world, sum(sizes)) as vr:
        vr.check("initial")
        for e in range(1, epochs + 1):
            xs = _slab_buffers(sizes, gen)
            full = torch.cat([s for _, _, s in xs]) if sum(sizes) else None
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            for r in range(world):
                vr.allgather(r, xs[r][1], sizes[r], offs[r], e)
            assert _lib.launch_count() == n0 + world
            vr.model_gather(e, full)
            vr.check(f"world {world}, slabs {n16s}, epoch {e}")


_N16 = {"1": lambda S: 1, "511": lambda S: 511, "512": lambda S: 512, "513": lambda S: 513,
        "512S": lambda S: 512 * S, "512S+1": lambda S: 512 * S + 1,
        "3*512S+7": lambda S: 3 * 512 * S + 7}


@pytest.mark.parametrize("n16", list(_N16))
@pytest.mark.parametrize("world", [1, 2, 3, 4, 7, 8, 16])
def test_allgather_bitwise_copy(world, n16):
    """Equal slabs of n16 16-byte words per rank: around the 512-thread CTA
    and the grid capped at one CTA per SM (S = SM count of this device)."""
    _gather_epochs(world, [_N16[n16](_sms())] * world, seed=world * 31 + len(n16))


@pytest.mark.parametrize("n16s", [
    [0],                                   # nothing to gather at all
    [3, 0, 5],                             # empty slab in the middle
    [0, 513, 1, "512S+1", 37],             # empty rank 0, gather_bytes % 256 = 128
    [(97 * r) % 600 for r in range(16)],   # 16 ragged ranks, rank 0 empty
    [511, 1, 0],                           # empty last rank
], ids=lambda v: "-".join(map(str, v)))
def test_allgather_ragged_and_empty_slabs(n16s):
    """Ragged slabs at prefix-sum offsets, including empty ones: a rank with
    no rows still raises its flags, so its peers complete and its own gather
    buffer holds the whole vector."""
    S = _sms()
    n16s = [_N16[n](S) if isinstance(n, str) else n for n in n16s]
    _gather_epochs(len(n16s), n16s, seed=sum(n16s))


def test_allgather_benchmark_vector_two_ranks():
    """The benchmark's Krylov vector: 1024 x 4096 float64 (32 MiB), row slabs
    of two ranks; the gathered buffer read as float64 is the matrix, bit for
    bit (NaN payloads and -0.0 planted)."""
    n, cols, world = 1024, 4096, 2
    g = torch.Generator(device="cuda").manual_seed(3)
    full = torch.randn((n, cols), dtype=torch.float64, device="cuda", generator=g)
    bits = full.view(torch.int64)
    bits[0, :4] = torch.tensor([0x7FF0000000000001, 0x7FF8DEADBEEF0001, -(1 << 63),
                                0x0000000000000001], device="cuda")
    bits[n - 1, -1] = 0xFFF4000000000123 - (1 << 64)
    slab = n // world * cols * 8
    raw = full.view(torch.uint8).reshape(-1)
    with VirtualRanks(world, n * cols * 8) as vr:
        xs = _slab_buffers([slab] * world, None, fill=[raw[r * slab:(r + 1) * slab]
                                                       for r in range(world)])
        for e in (1, 2):
            torch.cuda.synchronize()
            for r in range(world):
                vr.allgather(r, xs[r][1], slab, r * slab, e)
            vr.model_gather(e, raw)
            vr.check(f"benchmark vector, epoch {e}")
            for r in range(world):
                got = vr.parity_view(r, e).view(torch.float64).view(n, cols)
                assert torch.equal(got.view(torch.int64), bits)


# ------------------------------------------------------------------ all-reduce
_SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, 2.0 ** 53, -(2.0 ** 53), 0.5, 3.0, np.inf, -np.inf,
                     np.nan, 5e-324, -5e-324, 2.2250738585072014e-308, 1e-310,
                     np.finfo(np.float64).max, -np.finfo(np.float64).max, 1e308, 2.0 ** -60])


def _partials(world, m, kind, rng):
    """(world, m) float64 partials whose rank-order sum is sensitive to the
    order, the sign of zero and the non-finite classes."""
    if kind == "normal":
        P = rng.standard_normal((world, m)) * 2.0 ** rng.integers(-40, 40, (world, m))
    elif kind == "special":
        P = rng.choice(_SPECIAL, size=(world, m))
    else:   # "order": 2^53, 1, -2^53 ... summed left to right loses the 1
        P = rng.choice(np.array([2.0 ** 53, 1.0, -(2.0 ** 53), 1.0, 0.5, -0.5]), size=(world, m))
    fixed = [
        np.full(world, -0.0),                                         # -0.0 stays -0.0
        np.array([0.0] + [-0.0] * (world - 1)),                       # +0.0 wins
        np.array([-0.0] + [0.0] * (world - 1)),
        np.full(world, np.finfo(np.float64).max),                     # overflow to +Inf
        np.array([np.inf, -np.inf] * world)[:world],                  # NaN (world > 1)
        np.array([2.0 ** 53, 1.0, -(2.0 ** 53)] * world)[:world],     # 0 in rank order
        np.full(world, 5e-324),                                       # subnormal sums
        np.array([np.nan] + [1.0] * (world - 1)),
    ]
    for t, col in enumerate(fixed[:m]):
        P[:, t] = col
    # a NaN with a payload, so the identity on one rank is checked bitwise
    if kind == "special" and m > len(fixed):
        P[0, len(fixed)] = np.frombuffer(np.int64(0x7FF80000000ABCDE).tobytes(), np.float64)[0]
    return P


def _rank_order_sum(P):
    acc = P[0].copy()
    with np.errstate(all="ignore"):
        for r in range(1, P.shape[0]):
            acc = acc + P[r]
    return acc


def _x_buffers(P):
    """Per rank: 64 + 8 doubles of sentinel bytes, partials in front."""
    out = []
    for r in range(P.shape[0]):
        x = torch.full((8 * (RMAX + 8),), SENT, dtype=torch.uint8, device="cuda")
        if P.shape[1]:
            x[:8 * P.shape[1]] = _bytes(P[r])
        out.append(x)
    return out


def _check_reduced(xs, P, what):
    world, m = P.shape
    want = _rank_order_sum(P).view(np.int64) if m else np.zeros(0, np.int64)
    got = [x.cpu().numpy() for x in xs]
    for r, g in enumerate(got):
        assert (g[8 * m:] == SENT).all(), f"{what}: rank {r} wrote x[m:]"
        assert np.array_equal(g, got[0]), f"{what}: rank {r} differs in bits from rank 0"
    bits = got[0][:8 * m].view(np.int64)
    if world == 1:
        assert np.array_equal(bits, P[0].view(np.int64)), f"{what}: one rank is not the identity"
    nan = np.isnan(want.view(np.float64))
    assert np.array_equal(np.isnan(bits.view(np.float64)), nan), f"{what}: NaN positions"
    bad = np.flatnonzero((bits != want) & ~nan)
    assert bad.size == 0, (f"{what}: columns {bad[:8].tolist()}: got "
                           f"{bits.view(np.float64)[bad[:8]]}, want "
                           f"{want.view(np.float64)[bad[:8]]}, partials {P[:, bad[:1]].ravel()}")


@pytest.mark.parametrize("m", [0, 1, 2, 24, 63, 64])
@pytest.mark.parametrize("world", [1, 2, 3, 8, 16])
def test_allreduce_rank_order_sum(world, m):
    """In-place all-reduce of m doubles: bitwise the sequential IEEE sum in
    rank order from rank 0's partial, identical on every rank; x[m:] and the
    slot columns >= m and rows >= world keep their sentinel."""
    rng = np.random.default_rng(world * 100 + m)
    with VirtualRanks(world, 0) as vr:
        for e, kind in enumerate(["special", "order", "normal", "special", "special"], 1):
            P = _partials(world, m, kind, rng)
            xs = _x_buffers(P)
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            for r in range(world):
                vr.allreduce(r, xs[r].data_ptr(), m, e)
            assert _lib.launch_count() == n0 + world
            vr.model_reduce(e, P)
            vr.check(f"all-reduce world {world}, m {m}, epoch {e} ({kind})")
            _check_reduced(xs, P, f"world {world}, m {m}, epoch {e} ({kind})")


# ------------------------------------------------------------ epoch protocol
@pytest.mark.parametrize("world", [2, 4])
def test_epochs_one_ahead_with_interleaved_reductions(world):
    """K = 8 epochs without a synchronisation in between.  Per epoch every
    rank gathers, snapshots its gather buffer at once, runs the reductions of a
    Gram-Schmidt pass (two of m inner products and a norm) and snapshots the
    buffer again; the last rank sleeps before that second snapshot, a slow
    consumer.  A faster rank completes the reductions, pushes the next epoch
    into the other parity buffer of the slow rank and only then waits for it,
    so every snapshot must still be its epoch's vector and every reduction
    exact.

    The launches go out operation by operation (the gathers of all ranks,
    then the first snapshots, ...), not all of rank 0's epochs first: torch
    streams of one process may share a hardware queue, and then a rank's
    stream-ordered work at the head of the queue blocks a peer's kernel behind
    it until the 4 s bound.  In this order nothing waits on work queued behind
    it, and on separate queues the ranks still drift one epoch apart."""
    K, S = 8, _sms()
    n16s = [512 * S + 1 + 37 * r for r in range(world)]
    sizes = [16 * n for n in n16s]
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(int).tolist()
    gen = torch.Generator(device="cuda").manual_seed(world)
    rng = np.random.default_rng(world)
    with VirtualRanks(world, sum(sizes)) as vr:
        xs, fulls, reds = {}, {}, {}
        for e in range(1, K + 1):
            xs[e] = _slab_buffers(sizes, gen)
            fulls[e] = torch.cat([s for _, _, s in xs[e]])
            for j, m in enumerate((min(e, RMAX), min(e, RMAX), 1)):
                P = _partials(world, m, ("special", "order", "normal")[j], rng)
                reds[3 * (e - 1) + j + 1] = (P, _x_buffers(P))
        # allocated up front: nothing between the launches may wait for the
        # device while a rank spins on a peer that is not enqueued yet
        snaps = {(r, e, k): torch.empty_like(fulls[e])
                 for r in range(world) for e in fulls for k in (0, 1)}
        torch.cuda.synchronize()
        n0 = _lib.launch_count()

        def on_each_rank(op):
            for r in range(world):
                with torch.cuda.stream(vr.streams[r]):
                    op(r)

        for e in range(1, K + 1):
            on_each_rank(lambda r: vr.allgather(r, xs[e][r][1], sizes[r], offs[r], e))
            on_each_rank(lambda r: snaps[r, e, 0].copy_(vr.parity_view(r, e)))
            for q in range(3 * (e - 1) + 1, 3 * e + 1):
                P, x = reds[q]
                on_each_rank(lambda r: vr.allreduce(r, x[r].data_ptr(), P.shape[1], q))

            def late_snapshot(r):
                if r == world - 1:
                    torch.cuda._sleep(2_000_000)      # the slow consumer
                snaps[r, e, 1].copy_(vr.parity_view(r, e))
            on_each_rank(late_snapshot)
        assert _lib.launch_count() == n0 + 4 * K * world
        for e in range(1, K + 1):
            vr.model_gather(e, fulls[e])
        for q in range(1, 3 * K + 1):
            vr.model_reduce(q, reds[q][0])
        vr.check(f"{K} epochs, world {world}")
        for (r, e, k), snap in snaps.items():
            assert torch.equal(snap, fulls[e]), \
                f"rank {r} epoch {e}: gather buffer overwritten before snapshot {k}"
        for q, (P, x) in reds.items():
            _check_reduced(x, P, f"reduction epoch {q}")


# ------------------------------------------------- two processes, one device
def test_two_processes_share_one_gpu_over_ipc():
    """tests/p2p_worker.py on two ranks of a gloo group, both on cuda:0, with
    BondShard(exchange='p2p'): gathers and small reductions go through the
    CUDA IPC mapped blocks and must be bitwise exact (the two contexts are
    time-sliced, so this is slow per epoch)."""
    t0 = time.time()
    rc, out, err = run_process_group(torchrun_cmd("p2p_worker.py", 2), timeout=300)
    print(f"two-process p2p exchange: {time.time() - t0:.1f} s wall")
    assert rc == 0 and "P2P_WORKER_OK" in out, out[-3000:] + err[-3000:]
