"""Circuit-amplitude contraction benchmark (BASELINE configs[3]: Lx x Ly qubit
grid, depth d, random U3 + fSim layers cycling the bond patterns A B C D,
complex128).  Not the driver's bench.py contract (that is configs[1]); run
under gpurun:

  python tools/bench_circuit.py [--Lx 5] [--Ly 5] [--depth 16] [--target-width 28]
                                [--max-slices 64] [--out gpurun_out/x.json]
  torchrun --nproc-per-node 8 tools/bench_circuit.py --Lx 6 --Ly 6 --depth 24 \\
           --target-width 32 --max-slices 64

The tree and the sliced indices are found once on the host (`find_sliced_tree`,
quimb_b200/treeopt.py), every slice is one pass of the tree executor (one
launch of the pairwise contraction kernel per node), slices are dealt
round-robin to the ranks and summed with ONE all-reduce.  When the slice count
exceeds ``--max-slices`` only that many slices are executed and the time is
reported per slice together with the extrapolated total (``partial: true``;
the amplitude is then not the full sum).  For <= 20 qubits the exact amplitude
from a dense state-vector simulation is compared.
"""
import argparse
import itertools
import json
import math
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--Lx", type=int, default=5)
    ap.add_argument("--Ly", type=int, default=5)
    ap.add_argument("--depth", type=int, default=16)
    ap.add_argument("--target-width", type=int, default=28)
    ap.add_argument("--max-slices", type=int, default=64)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--max-gb", type=float, default=70.0,
                    help="refuse trees whose live intermediates exceed this many GB")
    ap.add_argument("--out", default=None)
    ap.add_argument("--tree-file", default=None,
                    help="JSON with a previously found sliced tree (ssa steps + sliced index "
                         "positions) for exactly this circuit: skips the host search")
    args = ap.parse_args()
    import numpy as np
    import torch
    import quimb_b200 as qb
    from quimb_b200 import tree as T
    from tests.circuit_util import random_grid_circuit_amplitude
    rank, world = 0, 1
    if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist
        rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl")
    nq = args.Lx * args.Ly
    arrays, inputs, output, amp = random_grid_circuit_amplitude(
        args.Lx, args.Ly, args.depth, seed=3, dense=nq <= 20)
    sd = {ix: 2 for t in inputs for ix in t}
    t0 = time.perf_counter()
    loaded = None
    if args.tree_file and os.path.exists(args.tree_file):
        rec = json.load(open(args.tree_file))
        if (rec.get("config") == [args.Lx, args.Ly, args.depth, args.target_width]
                and rec.get("n_inputs") == len(inputs)):
            loaded = rec
    if loaded is not None:
        sliced = [ix for ix in loaded["sliced"]]
        s_ = set(sliced)
        red = [tuple(ix for ix in t if ix not in s_) for t in inputs]
        tr = T.Tree(red, tuple(output), sd, [tuple(st) for st in loaded["ssa"]])
    else:
        tr, sliced = T.find_sliced_tree(inputs, output, sd, args.target_width,
                                        min_slices=world if world > 1 else None)
        if args.tree_file and rank == 0:
            json.dump({"config": [args.Lx, args.Ly, args.depth, args.target_width],
                       "n_inputs": len(inputs), "sliced": list(sliced),
                       "ssa": [[i, j] for i, j, _, _ in tr.steps]},
                      open(args.tree_file, "w"))
    t_find = time.perf_counter() - t0
    n_slices = 2 ** len(sliced)
    macs_slice = tr.contraction_cost()
    units = list(itertools.islice(itertools.product(*[range(2)] * len(sliced)),
                                  min(n_slices, args.max_slices * world)))
    mine = units[rank::world]
    dev = [qb.asarray(a) for a in arrays]
    red_inputs = tr.inputs

    def run_slice(vals):
        fix = dict(zip(sliced, vals))
        sub = [Array_slice(x, t, fix) for x, t in zip(dev, inputs)]
        return T.execute(tr, sub)

    def Array_slice(x, t, fix):
        if not any(ix in fix for ix in t):
            return x
        return x[tuple(fix[ix] if ix in fix else slice(None) for ix in t)]

    from quimb_b200 import treeopt
    elems_slice = 2.0 ** treeopt.tree_traffic(tr.inputs, tr.output, sd, [(i, j) for i, j, _, _ in tr.steps])
    peak_gb = 16.0 * 2.0 ** treeopt.tree_peak(tr.inputs, tr.output, sd,
                                             [(i, j) for i, j, _, _ in tr.steps]) / 1e9
    if peak_gb > args.max_gb:
        # never drive the box out of memory: refuse instead
        if rank == 0:
            print(json.dumps({"refused": f"the tree needs about {peak_gb:.0f} GB alive at once "
                              f"(> --max-gb {args.max_gb}); lower --target-width"}))
        return
    res = {"config": f"{args.Lx}x{args.Ly} depth {args.depth} complex128", "n_gpus": world,
           "peak_gbytes_estimate": round(peak_gb, 1),
           "algorithmic_gbytes_per_slice": round(16.0 * elems_slice / 1e9, 3),
           "tensors": len(inputs), "log2_width": tr.contraction_width(),
           "n_sliced": len(sliced), "log2_macs_per_slice": round(math.log2(macs_slice), 2),
           "find_seconds": round(t_find, 1), "runs": []}
    for rep in range(args.reps + 1):                    # first pass = warm-up
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        n0 = qb.launch_count()
        t0 = time.perf_counter()
        total = None
        for vals in mine:
            part = run_slice(vals)
            total = part if total is None else total + part
        tt = total.resolve() if total is not None else torch.zeros((), dtype=torch.complex128, device="cuda")
        if world > 1:
            dist.all_reduce(tt)
        val = complex(tt.item())
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if world > 1:
            tmax = torch.tensor([dt], device="cuda")
            dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
            dt = float(tmax.item())
        done = len(units)
        flops = 8.0 * macs_slice * done                  # complex multiply-add = 8 real flop
        res["runs"].append({"seconds": dt, "slices_done": done, "launches": qb.launch_count() - n0,
                            "tflops": flops / dt / 1e12,
                            # operands read + results written by every tree node, complex128
                            "algorithmic_GBps": 16.0 * elems_slice * done / dt / 1e9,
                            "seconds_all_slices_extrapolated": dt * n_slices / done})
    res["partial"] = len(units) < n_slices
    res["value"] = [val.real, val.imag]
    if amp is not None and not res["partial"]:
        res["abs_error_vs_statevector"] = abs(val - amp)
    if rank == 0:
        print(json.dumps(res))
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
