"""Variational fit benchmark (``mps_gate_with_mpo_fit``).

  python tools/bench_fit.py [--L 100] [--chis 256,1024]
                            [--dtypes float64,complex128] [--skip-dm]
                            [--budget-s 120]

Workload (as tools/bench_mpo_compress.py): the open Heisenberg MPO (D_w = 5)
applied to a random MPS (d = 2, bonds min(chi, 2^i, 2^(L-i))), fitted at
``max_bond = chi`` from the random start with the defaults (one-site sweeps,
bond doubling from 8, ``max_iterations=10``).  For every (chi, dtype) it
prints one JSON line with, after a warm-up fit on a chain long enough to
reach every bulk shape:
  seconds          one fit (host clock around a synchronised call);
  seconds_tol      one fit with tol=1e-8, and sweeps_tol, the sweeps it ran;
  peak_bytes       torch.cuda.max_memory_allocated during the default fit;
  share            of a third, instrumented fit (every step synchronised and
                   timed): contractions (contract_pair), QR moves
                   (left / right_canonize_site, QR + absorb launch) and
                   two-site SVDs (array_split), with their seconds;
  flops_per_sweep  the contraction flops of one sweep of the last sweep's
                   shapes (2 M N K real, 8 M N K complex per launch);
  fidelity_vs_dm   |<x|y>|^2 / (<x|x><y|y>) against
                   mps_gate_with_mpo(method='dm') at the same max_bond.
A configuration is skipped, with its reason, when its predicted time per fit
(the same dtype at a smaller chi in this run, scaled by chi^3) exceeds
--budget-s: each configuration runs three fits and a 'dm' application.  The
card name and power limit are read in the same run.
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


class StepTimer:
    """Synchronised host-clock timers around the fit's steps, by kind, and
    the flops of every contraction launch from its operand shapes."""

    STEPS = {"contract": ("fit", "contract_pair"),
             "qr": ("tebd", "left_canonize_site"),
             "qr_r": ("tebd", "right_canonize_site"),
             "svd": ("fit", "array_split")}

    def __init__(self):
        import torch
        from quimb_b200 import fit, tebd
        mods = {"fit": fit, "tebd": tebd}
        self.sync = torch.cuda.synchronize
        self.seconds = {k: 0.0 for k in self.STEPS}
        self.flops = []          # per launch, in call order
        self.depth = 0
        self.saved = []
        for step, (mod, name) in self.STEPS.items():
            m = mods[mod]
            f = getattr(m, name)
            self.saved.append((m, name, f))
            setattr(m, name, self.wrap(step, f))

    @staticmethod
    def launch_flops(a, la, b, lb):
        ext = dict(zip(la, a.shape))
        ext.update(zip(lb, b.shape))
        n = float(np.prod([float(v) for v in ext.values()]))
        return (8 if a.dtype.is_complex else 2) * n

    def wrap(self, step, f):
        def g(*a, **k):
            if self.depth:
                return f(*a, **k)
            if step == "contract":
                self.flops.append(self.launch_flops(a[0], a[1], a[2], a[3]))
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
        for m, n, f in self.saved:
            setattr(m, n, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--chis", default="256,1024")
    ap.add_argument("--dtypes", default="float64,complex128")
    ap.add_argument("--skip-dm", action="store_true")
    ap.add_argument("--budget-s", type=float, default=120.0,
                    help="skip a configuration whose predicted seconds per fit exceed this")
    args = ap.parse_args()

    import torch
    import quimb_b200 as qb
    from quimb_b200.mps import mpo_ham_heis
    print(json.dumps(card()), flush=True)
    L, d = args.L, 2
    measured = {}          # dtype -> (chi, seconds) of the last run
    for chi in (int(c) for c in args.chis.split(",")):
        for dtype in args.dtypes.split(","):
            row = {"chi": chi, "dtype": dtype, "L": L, "d": d, "D_w": 5, "max_bond": chi,
                   "bsz": 1, "max_iterations": 10}
            if dtype in measured:
                c0, s0 = measured[dtype]
                row["predicted_seconds"] = s0 * (chi / c0) ** 3
                if row["predicted_seconds"] > args.budget_s:
                    row["skipped"] = (f"predicted {row['predicted_seconds']:.0f} s per fit "
                                      f"(chi^3 from {s0:.1f} s at chi={c0}) > budget "
                                      f"{args.budget_s:.0f} s")
                    print(json.dumps(row), flush=True)
                    continue
            psi = rand_sites(L, chi, d, dtype, seed=chi)
            mpo = [qb.asarray(w.astype(dtype)) for w in mpo_ham_heis(L)]
            kw = dict(mpo_shape="lrdu", seed=1)
            Lw = min(L, 2 * int(np.ceil(np.log2(chi))) + 6)
            qb.mps_gate_with_mpo_fit(psi[:Lw - 1] + [_close_end(psi[Lw - 1])],
                                     mpo[:Lw - 1] + [mpo[-1]], chi, **kw)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            m0 = torch.cuda.memory_allocated()
            t0 = time.perf_counter()
            out = qb.mps_gate_with_mpo_fit(psi, mpo, chi, **kw)
            torch.cuda.synchronize()
            row["seconds"] = time.perf_counter() - t0
            measured[dtype] = (chi, row["seconds"])
            row["peak_bytes"] = int(torch.cuda.max_memory_allocated() - m0)
            row["bonds_max"] = max(x.shape[2] for x in out)
            info = {}
            t0 = time.perf_counter()
            qb.mps_gate_with_mpo_fit(psi, mpo, chi, tol=1e-8, info=info, **kw)
            torch.cuda.synchronize()
            row["seconds_tol"] = time.perf_counter() - t0
            row["sweeps_tol"] = info["sweeps"]
            row["max_tdiff_tol"] = info["max_tdiff"]
            timer = StepTimer()
            try:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                qb.mps_gate_with_mpo_fit(psi, mpo, chi, **kw)
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
            finally:
                timer.close()
            sec = timer.seconds
            qr = sec["qr"] + sec["qr_r"]
            row["instrumented_seconds"] = wall
            row["share"] = {"contract": sec["contract"] / wall, "qr": qr / wall,
                            "svd": sec["svd"] / wall,
                            "other": 1 - (sec["contract"] + qr + sec["svd"]) / wall}
            row["step_seconds"] = {"contract": sec["contract"], "qr": qr, "svd": sec["svd"]}
            # the last sweep: 4 L - 1 launches (one-site, one MPO target)
            row["flops_per_sweep"] = float(sum(timer.flops[-(4 * L - 1):]))
            if not args.skip_dm:
                dm = qb.mps_gate_with_mpo(psi, mpo, method="dm", max_bond=chi, mpo_shape="lrdu")
                row["fidelity_vs_dm"] = float(fidelity(out, dm))
                del dm
            print(json.dumps(row), flush=True)
            del out, psi
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
