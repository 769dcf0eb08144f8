"""Successive-compression benchmark (``mps_gate_with_mpo_successive``).

  python tools/bench_successive.py [--L 100] [--chis 256,1024]
                                   [--dtypes float64,complex128]
                                   [--methods src,src-oversample,...] [--budget-s 900]

The workload of tools/bench_mpo_compress.py: the open Heisenberg MPO
(D_w = 5) applied to a random MPS (d = 2) with ``max_bond = chi``.  For every
(chi, dtype, method) one JSON line, after a warm-up on a shorter chain:
  seconds        one application (host clock around a synchronised call);
  peak_bytes     torch.cuda.max_memory_allocated during that call;
  shares         of a second, instrumented application (each step
                 synchronised and timed): contractions, QR / SVD splits,
                 qb_sketch_env and the direct sweep of '-oversample';
  fidelity_vs_dm |<x|y>|^2 / (<x|x><y|y>) against 'dm' from the same run.
'dm' and 'zipup' (``mps_gate_with_mpo``) run first as yardsticks.  A
configuration is skipped, with its reason, when its predicted time (the
same method at a smaller chi in this run, scaled by chi^3) exceeds
--budget-s or its predicted footprint 90 % of free memory.  Then, per
(chi, dtype), ``qb_sketch_env`` against the two-launch ``contract_pair``
composition on the same bulk-site operands (CUDA events over --reps calls),
with its bytes (LE read once, H written once) over 3.35 TB/s.  The card name
and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tools.bench_mpo_compress import _close_end, fidelity  # noqa: E402
from tools.bench_observables import card, rand_sites  # noqa: E402

D_W = 5
HBM_BYTES_PER_S = 3.35e12
SUCCESSIVE = ("src", "src-oversample", "srcmps", "srcmps-oversample", "sdc", "sdc-oversample")


class StepTimer:
    """Synchronised timing of the steps of one application."""
    STEPS = {"contract": "_cp", "split": "array_split", "sketch_env": "sketch_env",
             "direct_sweep": "_direct_sweep"}

    def __init__(self):
        import torch
        from quimb_b200 import successive
        self.mod = successive
        self.sync = torch.cuda.synchronize
        self.seconds = {k: 0.0 for k in self.STEPS}
        self.depth = 0
        self.saved = []
        for step, name in self.STEPS.items():
            f = getattr(successive, name)
            self.saved.append((name, f))
            setattr(successive, name, self.wrap(step, f))

    def wrap(self, step, f):
        def g(*a, **k):
            if self.depth:
                return f(*a, **k)
            self.depth += 1
            self.sync()
            t0 = time.perf_counter()
            try:
                return f(*a, **k)
            finally:
                self.sync()
                self.seconds[step] += time.perf_counter() - t0
                self.depth -= 1
        return g

    def close(self):
        for n, f in self.saved:
            setattr(self.mod, n, f)


def predicted_bytes(method, L, chi, d, esize):
    k = chi if method in ("src", "srcmps", "sdc") else max(round(1.5 * chi), chi + 10)
    base = L * chi * chi * d * esize
    if method in ("dm",):
        return base + (L + 4) * (chi * D_W) ** 2 * esize
    # left environments k chi D_w per site, plus a few sketches
    return base + L * k * chi * D_W * esize + 8 * k * chi * D_W * d * esize + L * k * k * d * esize


def kernel_vs_compose(chi, dtype, reps):
    """qb_sketch_env against LE W (one GEMM) then . Omega (batched) on the
    bulk operands of an SRC step at k = chi."""
    import torch
    from quimb_b200 import contract_pair
    from quimb_b200.successive import sketch_env
    tdt = {"float64": torch.float64, "complex128": torch.complex128}[dtype]
    g = torch.Generator(device="cuda").manual_seed(chi)
    LE = torch.randn((chi, chi, D_W), dtype=tdt, device="cuda", generator=g)
    W = torch.randn((D_W, D_W, 2, 2), dtype=tdt, device="cuda", generator=g)
    Om = torch.randn((chi, 2), dtype=tdt, device="cuda", generator=g)

    def compose():
        X = contract_pair(LE, [0, 1, 2], W, [2, 3, 4, 5], [0, 1, 3, 4, 5])
        return contract_pair(X, [0, 1, 3, 4, 5], Om, [0, 4], [0, 1, 3, 5])

    def timed(f):
        for _ in range(3):
            f()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / reps
    a, b = sketch_env(LE, W, Om), compose()
    err = float((a - b).abs().max() / b.abs().max())
    tk, tc = timed(lambda: sketch_env(LE, W, Om)), timed(compose)
    esize = LE.element_size()
    nbytes = (LE.numel() + chi * chi * D_W * 2) * esize + (W.numel() + Om.numel()) * esize
    return {"kernel_vs_compose": True, "chi": chi, "k": chi, "dtype": dtype,
            "sketch_env_s": tk, "contract_pair_x2_s": tc, "speedup": tc / tk,
            "bytes": nbytes, "share_of_3.35TB/s": nbytes / tk / HBM_BYTES_PER_S,
            "max_rel_diff": err}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--chis", default="256,1024")
    ap.add_argument("--dtypes", default="float64,complex128")
    ap.add_argument("--methods", default="dm,zipup," + ",".join(SUCCESSIVE))
    ap.add_argument("--budget-s", type=float, default=900.0)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()

    import torch
    import quimb_b200 as qb
    from quimb_b200.mps import mpo_ham_heis
    print(json.dumps(card()), flush=True)
    L, d = args.L, 2
    measured = {}
    for chi in (int(c) for c in args.chis.split(",")):
        for dtype in args.dtypes.split(","):
            esize = 8 if dtype == "float64" else 16
            psi = rand_sites(L, chi, d, dtype, seed=chi)
            mpo = [qb.asarray(w.astype(dtype)) for w in mpo_ham_heis(L)]
            Lw = min(L, 2 * int(np.ceil(np.log2(chi))) + 6)
            ref = None
            for method in args.methods.split(","):
                row = {"chi": chi, "dtype": dtype, "L": L, "d": d, "D_w": D_W,
                       "method": method, "max_bond": chi}
                free, _ = torch.cuda.mem_get_info()
                pred = predicted_bytes(method, L, chi, d, esize)
                if pred > 0.9 * free:
                    row["skipped"] = f"predicted footprint {pred / 1e9:.1f} GB > 90% of free"
                    print(json.dumps(row), flush=True)
                    continue
                if (method, dtype) in measured:
                    c0, s0 = measured[method, dtype]
                    row["predicted_seconds"] = s0 * (chi / c0) ** 3
                    if row["predicted_seconds"] > args.budget_s:
                        row["skipped"] = (f"predicted {row['predicted_seconds']:.0f} s > budget "
                                          f"{args.budget_s:.0f} s")
                        print(json.dumps(row), flush=True)
                        continue
                if method in SUCCESSIVE:
                    def run(p, m):
                        return qb.mps_gate_with_mpo_successive(p, m, chi, method=method, seed=1,
                                                               mpo_shape="lrdu")
                else:
                    def run(p, m):
                        return qb.mps_gate_with_mpo(p, m, method=method, max_bond=chi,
                                                    mpo_shape="lrdu")
                run(psi[:Lw - 1] + [_close_end(psi[Lw - 1])], mpo[:Lw - 1] + [mpo[-1]])
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                m0 = torch.cuda.memory_allocated()
                t0 = time.perf_counter()
                out = run(psi, mpo)
                torch.cuda.synchronize()
                row["seconds"] = time.perf_counter() - t0
                measured[method, dtype] = (chi, row["seconds"])
                row["peak_bytes"] = int(torch.cuda.max_memory_allocated() - m0)
                row["bonds_max"] = max(x.shape[2] for x in out)
                if method in SUCCESSIVE:
                    timer = StepTimer()
                    try:
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        run(psi, mpo)
                        torch.cuda.synchronize()
                        wall = time.perf_counter() - t0
                    finally:
                        timer.close()
                    row["instrumented_seconds"] = wall
                    row["shares"] = {k: v / wall for k, v in timer.seconds.items() if v}
                if method == "dm":
                    ref = out
                elif ref is not None:
                    row["fidelity_vs_dm"] = float(fidelity(out, ref))
                print(json.dumps(row), flush=True)
                del out
                torch.cuda.empty_cache()
            ref = None
            del psi
            torch.cuda.empty_cache()
            print(json.dumps(kernel_vs_compose(chi, dtype, args.reps)), flush=True)


if __name__ == "__main__":
    main()
