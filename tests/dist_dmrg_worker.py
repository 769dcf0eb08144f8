"""Worker for the bond-sharded DMRG check (run under torch.distributed.run).

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 \
      --master-port P tests/dist_dmrg_worker.py [--backend gloo|nccl] [--same-gpu]

Every rank runs the same DMRG2 twice -- local eigensolves row-sharded over the
ranks (quimb_b200.dist.BondShard) and unsharded -- and checks that the
energies agree with each other and with exact diagonalisation, and that the
sharded states are identical on all ranks.  ``--same-gpu`` puts all ranks on
cuda:0 with the gloo backend (collectives staged through the host), which is
how the single-GPU test tier exercises the exchange logic.
"""
import argparse
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="gloo")
    ap.add_argument("--same-gpu", action="store_true")
    ap.add_argument("--L", type=int, default=10)
    ap.add_argument("--chi", type=int, default=24)
    ap.add_argument("--dtype", default="float64")
    ap.add_argument("--exchange", default="auto",
                    help="BondShard exchange; 'p2p' runs the peer-memory kernels over CUDA IPC")
    ap.add_argument("--emulate", action="store_true",
                    help="CPU tier: host layer on tests/abi_emulator.py (no device)")
    args = ap.parse_args()
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
    import contextlib
    ctx = contextlib.nullcontext()
    if args.emulate:
        from tests.abi_emulator import emulated_abi
        ctx = emulated_abi()
    else:
        local = 0 if args.same_gpu else int(os.environ.get("LOCAL_RANK", rank))
        torch.cuda.set_device(local)
    dist.init_process_group(args.backend, rank=rank, world_size=world)
    with ctx:
        run(args, rank, world)


def run(args, rank, world):
    import quimb_b200 as qb
    from quimb_b200.dist import BondShard
    from oracle import dmrg_np as dm

    mpo = dm.mpo_heis(args.L)
    sh = BondShard(exchange=args.exchange)
    ds = qb.DMRG2(mpo, [8, args.chi], cutoffs=1e-12, mpo_shape="lrdu", seed=5,
                  dtype=args.dtype, shard=sh)
    ds.shard_min_bond = 2            # shard every bond >= 2 * world rows
    ds.solve(tol=1e-9, max_sweeps=6)
    p2p_ok = True
    if args.exchange == "p2p":
        # the kernels carried (some of) the exchange and never timed out
        p2p_ok = sh.exchange_name.startswith("p2p") and sh._px is not None
        sh.check()
        if rank == 0:
            print(f"exchange={sh.exchange_name} p2p gathers={sh._px.g_epoch if sh._px else 0} "
                  f"reductions={sh._px.r_epoch if sh._px else 0}")
        sh.close()
    d1 = qb.DMRG2(mpo, [8, args.chi], cutoffs=1e-12, mpo_shape="lrdu", seed=5,
                  dtype=args.dtype)
    d1.solve(tol=1e-9, max_sweeps=6)
    e0 = float(np.linalg.eigvalsh(dm.mpo_to_dense(mpo))[0]) if args.L <= 12 else None
    ok = abs(ds.energy - d1.energy) < 1e-8
    if e0 is not None:
        ok = ok and abs(ds.energy - e0) < 1e-6
    ok = ok and sh.bytes_gathered > 0 and p2p_ok
    # the replicated part of the sweep stays bit-identical on all ranks
    cdev = "cuda" if args.backend == "nccl" else "cpu"   # NCCL reduces device tensors only
    chk = torch.stack([a.t.abs().sum().double() for a in ds.state]).to(cdev)
    lo, hi = chk.clone(), chk.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    ok = ok and bool(torch.equal(lo, hi))
    flag = torch.tensor([1.0 if ok else 0.0], device=cdev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(f"sharded E={ds.energy:.12f} unsharded E={d1.energy:.12f} exact={e0} "
              f"gathered={sh.bytes_gathered} matvecs={sum(ds.nmatvecs)}/{sum(d1.nmatvecs)}")
        print("DIST_DMRG_OK" if flag.item() == 1.0 else "DIST_DMRG_FAIL", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
