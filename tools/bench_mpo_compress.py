"""MPO application with compression benchmark (``mps_gate_with_mpo``).

  python tools/bench_mpo_compress.py [--L 100] [--chis 256,1024]
                                     [--dtypes float64,complex128]
                                     [--methods direct,dm,zipup,zipup-first]
                                     [--oracle-chi 256]

Workload: the open Heisenberg MPO (D_w = 5) applied to a random MPS (d = 2,
bonds min(chi, 2^i, 2^(L-i))) with ``max_bond = chi``.  For every (chi,
dtype, method) it prints one JSON line with, after a warm-up application on a
chain long enough to reach every bulk shape:
  seconds        one application (host clock around a synchronised call);
  peak_bytes     torch.cuda.max_memory_allocated during that call, and the
                 footprint predicted from the shapes;
  split_share    share of a second, instrumented application spent in the
                 factorisation steps (QR, SVD, eigh: each call synchronised
                 and timed), and split_seconds per step (see SplitTimer);
  fidelity_vs_direct  |<x|y>|^2 / (<x|x><y|y>) against the 'direct' result,
                 where direct ran.
A configuration is skipped, with its reason, when its predicted footprint
exceeds 90 % of the free device memory, or when its predicted time per
application (the same method and dtype at a smaller chi in this run, scaled
by chi^3) exceeds --budget-s.  At ``--oracle-chi`` the numpy oracle
(oracle/mpo_compress_np.py) is timed on the host CPU, float64.  The card
name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tools.bench_observables import card, rand_sites  # noqa: E402

D_W = 5


def predicted_bytes(method, L, chi, d, esize):
    """Resident footprint from the shapes: inputs plus what each method keeps
    (direct: L sites at chi D_w bonds; dm: L - 1 left environments of
    (chi D_w)^2; zip-up: one carry and its split), with a 4-site-sized margin
    for the temporaries of one step."""
    cw = chi * D_W
    base = L * chi * chi * d * esize
    if method == "direct":
        keep = (L + 4) * d * cw * cw * esize
    elif method == "dm":
        keep = (L + 4) * cw * cw * esize + 4 * (d * chi) ** 2 * esize
    elif method == "zipup":
        keep = L * chi * chi * d * esize + 8 * cw * d * chi * esize
    else:
        c2 = 2 * chi
        keep = L * c2 * c2 * d * esize + 8 * D_W * c2 * d * c2 * esize
    return base + keep


class SplitTimer:
    """Synchronised host-clock timers around every factorisation step of the
    methods, by step:
      gauge_qr         zip-up's canonize_around QR moves (QR + absorb launch)
      method_split     the zip-up SVD / the dm eigh (array_split)
      direct_canonize  direct's QR of each product site (QR + absorb launch)
      direct_sweep     the direct sweeps' compress_between (QR / LQ / SVD of
                       the reduced factor + absorb launch)"""

    STEPS = {"gauge_qr": ("mpo_compress", "tensor_canonize_bond"),
             "method_split": ("mpo_compress", "array_split"),
             "direct_canonize": ("tebd", "left_canonize_site"),
             "direct_sweep": ("tebd", "right_compress_site")}

    def __init__(self):
        import torch
        from quimb_b200 import mpo_compress, tebd
        mods = {"mpo_compress": mpo_compress, "tebd": tebd}
        self.sync = torch.cuda.synchronize
        self.seconds = {k: 0.0 for k in self.STEPS}
        self.depth = 0
        self.saved = []
        for step, (mod, name) in self.STEPS.items():
            m = mods[mod]
            f = getattr(m, name)
            self.saved.append((m, name, f))
            setattr(m, name, self.wrap(step, f))

    @property
    def total(self):
        return sum(self.seconds.values())

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
        for m, n, f in self.saved:
            setattr(m, n, f)


def fidelity(x, y):
    from quimb_b200.tebd import mps_overlap
    xy = mps_overlap(x, y)
    return abs(xy) ** 2 / (mps_overlap(x, x).real * mps_overlap(y, y).real)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--chis", default="256,1024")
    ap.add_argument("--dtypes", default="float64,complex128")
    ap.add_argument("--methods", default="direct,dm,zipup,zipup-first")
    ap.add_argument("--oracle-chi", type=int, default=256)
    ap.add_argument("--budget-s", type=float, default=900.0,
                    help="skip a configuration whose predicted seconds per application "
                         "exceed this")
    args = ap.parse_args()

    import torch
    import quimb_b200 as qb
    from quimb_b200.mps import mpo_ham_heis
    print(json.dumps(card()), flush=True)
    L, d = args.L, 2
    methods = args.methods.split(",")
    measured = {}          # (method, dtype) -> (chi, seconds) of the last run
    for chi in (int(c) for c in args.chis.split(",")):
        for dtype in args.dtypes.split(","):
            esize = 8 if dtype == "float64" else 16
            psi = rand_sites(L, chi, d, dtype, seed=chi)
            mpo = [qb.asarray(w.astype(dtype)) for w in mpo_ham_heis(L)]
            Lw = min(L, 2 * int(np.ceil(np.log2(chi))) + 6)
            results = {}
            for method in methods:
                row = {"chi": chi, "dtype": dtype, "L": L, "d": d, "D_w": D_W,
                       "method": method, "max_bond": chi}
                free, _ = torch.cuda.mem_get_info()
                pred = predicted_bytes(method, L, chi, d, esize)
                row["predicted_bytes"] = int(pred)
                if pred > 0.9 * free:
                    row["skipped"] = f"predicted footprint {pred / 1e9:.1f} GB > 90% of " \
                                     f"{free / 1e9:.1f} GB free"
                    print(json.dumps(row), flush=True)
                    continue
                if (method, dtype) in measured:
                    # every step is a chi^3 GEMM or factorisation
                    c0, s0 = measured[method, dtype]
                    row["predicted_seconds"] = s0 * (chi / c0) ** 3
                    if row["predicted_seconds"] > args.budget_s:
                        row["skipped"] = (f"predicted {row['predicted_seconds']:.0f} s per "
                                          f"application (chi^3 from {s0:.1f} s at chi={c0}) > "
                                          f"budget {args.budget_s:.0f} s")
                        print(json.dumps(row), flush=True)
                        continue
                kw = dict(method=method, max_bond=chi, mpo_shape="lrdu")
                qb.mps_gate_with_mpo(psi[:Lw - 1] + [_close_end(psi[Lw - 1])],
                                     mpo[:Lw - 1] + [mpo[-1]], **kw)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                m0 = torch.cuda.memory_allocated()
                t0 = time.perf_counter()
                out = qb.mps_gate_with_mpo(psi, mpo, **kw)
                torch.cuda.synchronize()
                row["seconds"] = time.perf_counter() - t0
                measured[method, dtype] = (chi, row["seconds"])
                row["peak_bytes"] = int(torch.cuda.max_memory_allocated() - m0)
                row["bonds_max"] = max(x.shape[2] for x in out)
                timer = SplitTimer()
                try:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    qb.mps_gate_with_mpo(psi, mpo, **kw)
                    torch.cuda.synchronize()
                    wall = time.perf_counter() - t0
                    row["split_share"] = timer.total / wall
                    row["split_seconds"] = {k: v for k, v in timer.seconds.items() if v}
                    row["instrumented_seconds"] = wall
                finally:
                    timer.close()
                results[method] = out
                if "direct" in results and method != "direct":
                    row["fidelity_vs_direct"] = float(fidelity(out, results["direct"]))
                print(json.dumps(row), flush=True)
                if method != "direct":
                    del out
                    results.pop(method)
                torch.cuda.empty_cache()
            results.clear()
            del psi
            torch.cuda.empty_cache()
            if chi == args.oracle_chi and dtype == "float64":
                from oracle import mpo_compress_np as onp
                A = [np.ascontiguousarray(x.to_numpy()) for x in
                     rand_sites(L, chi, d, dtype, seed=chi)]
                W = [np.ascontiguousarray(w.transpose(0, 1, 3, 2)) for w in mpo_ham_heis(L)]
                for method in methods:
                    t0 = time.perf_counter()
                    onp.gate_with_mpo(A, W, method=method, max_bond=chi)
                    print(json.dumps({"oracle_numpy_cpu": True, "chi": chi, "dtype": dtype,
                                      "L": L, "method": method,
                                      "seconds": time.perf_counter() - t0,
                                      "cpu_threads": torch.get_num_threads()}), flush=True)


def _close_end(A):
    """Site A cut to a right bond of 1 (the last site of a shorter warm-up
    chain)."""
    import quimb_b200 as qb
    return qb.Array(A.t[:, :, :1].contiguous())


if __name__ == "__main__":
    main()
