"""PEPS boundary-MPS contraction benchmark (BASELINE configs[4]: 10x10 PEPS,
bond 8, boundary chi 128, complex64 -- sized for one 80 GB GPU; at chi 256 the
intermediates need more than 80 GB).  bench.py measures configs[1]:

  python tools/bench_boundary.py [--Lx 10] [--Ly 10] [--D 8] [--chi 128]
                                 [--dtype complex64] [--reps 1]
  torchrun --nproc-per-node 2 tools/bench_boundary.py --two-sided

Reports wall time (CUDA-synchronised) of one `contract_boundary` of the
two-layer norm network, kernel launches, the largest boundary bond met and the
value; with --two-sided the xmin / xmax half-sweeps run on two ranks
(`contract_boundary_two_sided`, one broadcast per boundary line over NCCL).
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402


def rand_peps(Lx, Ly, D, d, dtype, seed):
    """Site arrays in quimb's PEPS order (up, right, down, left, phys) with
    i.i.d. normal entries scaled like quimb's `sensibly_scale`."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(Lx):
        row = []
        for j in range(Ly):
            shape = []
            if i < Lx - 1:
                shape.append(D)
            if j < Ly - 1:
                shape.append(D)
            if i > 0:
                shape.append(D)
            if j > 0:
                shape.append(D)
            shape.append(d)
            x = rng.standard_normal(shape)
            if np.dtype(dtype).kind == "c":
                x = x + 1j * rng.standard_normal(shape)
            x = x / np.linalg.norm(x) ** (1.5 / len(shape))
            row.append(x.astype(dtype))
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--Lx", type=int, default=10)
    ap.add_argument("--Ly", type=int, default=10)
    ap.add_argument("--D", type=int, default=8)
    ap.add_argument("--chi", type=int, default=128)
    ap.add_argument("--dtype", default="complex64")
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--two-sided", action="store_true")
    ap.add_argument("--profile", action="store_true",
                    help="synchronised timers around qr / svd / contraction / permute calls "
                         "(serialises the streams: use for the split, not for the total)")
    args = ap.parse_args()
    import torch
    import quimb_b200 as qb
    from quimb_b200 import boundary as bd
    rank = 0
    if args.two_sided and "RANK" in os.environ:
        import torch.distributed as dist
        rank = int(os.environ["RANK"])
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl")
    prof = {}
    if args.profile:
        from quimb_b200 import contract as qc, linalg as ql, ops as qo, split as qs

        def wrap(mod, name, tag, shape_of):
            fn = getattr(mod, name)

            def timed(*a, **k):
                torch.cuda.synchronize(); t0 = time.perf_counter()
                r = fn(*a, **k)
                torch.cuda.synchronize(); dt = time.perf_counter() - t0
                key = (tag, shape_of(*a, **k))
                e = prof.setdefault(key, [0, 0.0])
                e[0] += 1; e[1] += dt
                return r
            setattr(mod, name, timed)
        mat = lambda x, *a, **k: (tuple(qo.asarray(x).shape), str(qo.asarray(x).dtype))
        wrap(ql, "qr", "qr", mat)
        wrap(ql, "svd", "svd", mat)
        wrap(ql, "svd_trunc", "svd_trunc", mat)
        wrap(qc, "contract_pair", "contract",
             lambda a, la, b, lb, lc, *r, **k: (tuple(a.shape), tuple(b.shape), str(a.dtype)))
        wrap(qc, "convert", "convert", lambda t, dt: (tuple(t.shape), str(t.dtype)))
        # modules that imported the names directly
        for m in (qs, bd, qo):
            for nm in ("contract_pair", "convert"):
                if hasattr(m, nm):
                    setattr(m, nm, getattr(qc, nm))
    arrays = rand_peps(args.Lx, args.Ly, args.D, 2, args.dtype, seed=4)
    dev = [[qb.asarray(a) for a in row] for row in arrays]
    tensors, Lx, Ly = bd.peps_norm_tensors(dev)
    out = {"Lx": Lx, "Ly": Ly, "D": args.D, "chi": args.chi, "dtype": args.dtype,
           "two_sided": bool(args.two_sided), "runs": []}
    for rep in range(args.reps + 1):                 # first run = warm-up
        torch.cuda.synchronize()
        n0 = qb.launch_count()
        t0 = time.perf_counter()
        if args.two_sided:
            val = bd.contract_boundary_two_sided(tensors, Lx, Ly, max_bond=args.chi,
                                                 cutoff=0.0, layer_tags=("KET", "BRA"))
        else:
            val = bd.contract_boundary(tensors, Lx, Ly, max_bond=args.chi, cutoff=0.0,
                                       layer_tags=("KET", "BRA"))
        torch.cuda.synchronize()
        out["runs"].append({"seconds": time.perf_counter() - t0,
                            "launches": qb.launch_count() - n0,
                            "value": [float(np.real(val)), float(np.imag(val))],
                            "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30})
    if prof:
        tot = {}
        for (tag, shp), (n, t) in prof.items():
            e = tot.setdefault(tag, [0, 0.0]); e[0] += n; e[1] += t
        out["profile_totals"] = {k: {"calls": v[0], "seconds": round(v[1], 3)} for k, v in tot.items()}
        top = sorted(prof.items(), key=lambda kv: -kv[1][1])[:12]
        out["profile_top"] = [{"what": k[0], "shape": str(k[1]), "calls": v[0],
                               "seconds": round(v[1], 3)} for k, v in top]
    if rank == 0:
        print(json.dumps(out), flush=True)
        os.makedirs("gpurun_out", exist_ok=True)
        json.dump(out, open(os.path.join("gpurun_out", "bench_boundary.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
