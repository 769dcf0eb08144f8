"""Worker of the two-process peer-exchange test (run under torch.distributed.run).

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 \
      --master-port P tests/p2p_worker.py

Both ranks sit on cuda:0 in a gloo group and use ``BondShard(exchange='p2p')``:
the blocks are mapped between the two processes through CUDA IPC and the
exchange runs in the kernels of csrc/p2p.cu.  Every rank generates the inputs
of all ranks from a shared seed, so the oracle is local:
  * ``all_gather_rows`` is the full matrix bit for bit, as a transient view
    (consumed before the next gather) and as a copy, over several epochs;
  * a larger vector rebuilds the exchange with a larger gather buffer;
  * ragged row counts and complex input take the host-staged path, exactly;
  * ``all_reduce_`` of <= 64 doubles is the rank-order IEEE sum in every bit.
Rank 0 prints P2P_WORKER_OK when every rank passed.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def matrix(n, cols, seed, dtype=torch.float64):
    """Seeded (n, cols) matrix, the same on every rank, with -0.0 and NaN
    payloads planted (the exchange must move bits, not values)."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn((n, cols), dtype=dtype, generator=g)
    if dtype == torch.float64:
        bits = a.view(torch.int64)
        bits[0, 0] = -(1 << 63)
        bits[n - 1, cols - 1] = 0x7FF80000DEAD0001
        bits[n // 2, 1] = 0x7FF0000000000005
    return a


def same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    if a.is_complex():
        a, b = torch.view_as_real(a), torch.view_as_real(b)
    return a.shape == b.shape and torch.equal(a.view(torch.int64), b.view(torch.int64))


def run(rank, world, dev):
    from quimb_b200.dist import BondShard
    sh = BondShard(exchange="p2p")
    fails = []

    def expect(cond, what):
        if not cond:
            fails.append(what)

    # p2p gathers: transient view and copy, several epochs
    n, cols = 256, 512
    lo, hi = sh.slab(n)
    for e in range(5):
        full = matrix(n, cols, 100 + e).to(dev)
        local = full[lo:hi].contiguous()
        view = sh.all_gather_rows(local, n, transient=True)
        expect(same_bits(view, full), f"transient gather, epoch {e}")
        copy = sh.all_gather_rows(local * 2, n)
        expect(same_bits(copy, full * 2), f"copied gather, epoch {e}")
    expect(sh.exchange_name.startswith("p2p"), f"exchange is {sh.exchange_name!r}")
    px = sh._px
    expect(px is not None and px.g_epoch == 10, "ten p2p gathers")

    # a larger vector closes the exchange and builds one with a larger buffer
    n2 = 1024
    lo2, hi2 = sh.slab(n2)
    for e in range(3):
        full = matrix(n2, cols, 200 + e).to(dev)
        got = sh.all_gather_rows(full[lo2:hi2].contiguous(), n2, transient=True)
        expect(same_bits(got, full), f"gather after rebuild, epoch {e}")
    expect(sh._px is not px and sh._px.gather_bytes == n2 * cols * 8 and sh._px.g_epoch == 3,
           "exchange rebuilt for the larger vector")

    # ragged rows and complex input take the staged path
    epochs = sh._px.g_epoch
    n3 = 255
    full = matrix(n3, cols, 300).to(dev)
    lo3, hi3 = sh.slab(n3)
    expect(same_bits(sh.all_gather_rows(full[lo3:hi3], n3), full), "ragged gather")
    full = matrix(n, cols, 301, dtype=torch.complex128).to(dev)
    expect(same_bits(sh.all_gather_rows(full[lo:hi], n), full), "complex gather")
    expect(sh._px.g_epoch == epochs, "ragged / complex gathers stayed off the p2p kernels")

    # small all-reduces: the rank-order sum, bit for bit
    rng = np.random.default_rng(7)
    specials = np.array([0.0, -0.0, 1.0, 2.0 ** 53, -(2.0 ** 53), np.inf, -np.inf, np.nan,
                         5e-324, np.finfo(np.float64).max, 1e-310])
    for q, m in enumerate((1, 24, 64, 63, 2)):
        P = rng.choice(specials, size=(world, m)) if q % 2 == 0 else \
            rng.standard_normal((world, m)) * 2.0 ** rng.integers(-30, 30, (world, m))
        P[:, 0] = -0.0
        h = torch.from_numpy(P[rank].copy()).to(dev)
        sh.all_reduce_(h)
        want = P[0].copy()
        with np.errstate(all="ignore"):
            for r in range(1, world):
                want = want + P[r]
        got = h.cpu().numpy()
        nan = np.isnan(want)
        expect(np.array_equal(np.isnan(got), nan)
               and np.array_equal(got.view(np.int64)[~nan], want.view(np.int64)[~nan]),
               f"all-reduce m={m}")
    expect(sh._px.r_epoch == 5, "five p2p reductions")

    sh.check()
    sh.close()
    return fails


def main():
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    fails = run(rank, world, dev)
    flag = torch.tensor([0.0 if fails else 1.0])
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if fails:
        print(f"rank {rank} failed: {fails}", flush=True)
    if rank == 0 and flag.item() == 1.0:
        print("P2P_WORKER_OK", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
