"""Long-range, multi-site and controlled gates on an MPS: the sub-MPO path
(``nonlocal_gates``) against the swap network of ``gate_with_auto_swap``.

  python tools/bench_nonlocal.py [--L 100] [--chis 256,1024]
                                 [--dtypes float64,complex128] [--budget-s 120]
                                 [--gates cx10,cx50,ccx10,c2x]
                                 [--methods swap,direct,dm,zipup]

A random MPS (d = 2, bonds up to chi) and, with ``max_bond = chi``:
  cx10 / cx50     a CNOT on (i, i + 10) / (i, i + 50), by 'swap' (the swap
                  network) and by ``mps_gate_nonlocal`` with 'direct', 'dm'
                  and 'zipup';
  ccx10           a Toffoli on (i, i + 5, i + 10), sub-MPO only;
  c2x             an X on site 80 controlled by sites 20 and 50
                  (``mps_gate_controlled``), sub-MPO only.
Every gate starts from the same state, canonical around the gate's first
site (so no method is charged for the canonicalisation the reference's
``info`` tracking would have skipped).  One JSON line per (chi, dtype, gate,
method), after a warm-up of the same call on a 24-site chain:
  seconds      one application (host clock around a synchronised call);
  peak_bytes   torch.cuda.max_memory_allocated during it, over the input;
  split_share  of a second, instrumented application: time inside QR / SVD /
               eigh splits (each synchronised) over its wall time;
  fidelity     |<x|y>|^2 / (<x|x><y|y>) against the exact product (the
               gate as a full-length MPO through ``tebd.mpo_apply``).
A configuration is skipped, with its reason, when its predicted time (the
same gate and method at a smaller chi in this run, scaled by chi^3) exceeds
--budget-s.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tools.bench_mpo_compress import fidelity  # noqa: E402
from tools.bench_observables import card, rand_sites  # noqa: E402

CX = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1], [0, 0, 1, 0]], dtype=float)
X = np.array([[0, 1], [1, 0]], dtype=float)
CCX = np.eye(8)
CCX[6:, 6:] = X
METHODS = ("direct", "dm", "zipup")


def gates(L):
    i = L // 2 - 5
    j = max(0, L // 2 - 25)
    return {
        "cx10": (CX, (i, i + 10), ()),
        "cx50": (CX, (j, j + 50), ()),
        "ccx10": (CCX, (i, i + 5, i + 10), ()),
        "c2x": (X, (int(0.8 * L),), (int(0.2 * L), L // 2)),
    }


class SplitTimer:
    """Synchronised time inside every factorisation the gate paths call."""
    SITES = (("mpo_compress", "array_split"), ("mpo_compress", "tensor_canonize_bond"),
             ("tebd", "qr_stabilized"), ("tebd", "tensor_split"),
             ("split", "tensor_compress_bond"))

    def __init__(self):
        import importlib
        import torch
        self.sync = torch.cuda.synchronize
        self.seconds = 0.0
        self.depth = 0
        self.saved = []
        for mod, name in self.SITES:
            m = importlib.import_module(f"quimb_b200.{mod}")
            f = getattr(m, name)
            self.saved.append((m, name, f))
            setattr(m, name, self.wrap(f))

    def wrap(self, f):
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
                self.seconds += time.perf_counter() - t0
                self.depth -= 1
        return g

    def close(self):
        for m, name, f in self.saved:
            setattr(m, name, f)


def exact(psi, G, where, controls):
    """The gate applied without truncation: its sub-MPO as a full-length MPO
    (identities elsewhere, bonds carried past) through ``tebd.mpo_apply``."""
    import quimb_b200 as qb
    from quimb_b200 import nonlocal_gates as nl
    L = len(psi)
    if controls:
        sub, present = nl._controlled_mpo(G, (2,) * len(where), list(where), list(controls),
                                          psi[0].dtype, psi[0].device)
    else:
        sub, present = qb.mpo_from_dense(G, 2, where)
    full, k, D = [], 0, 1
    for s in range(L):
        if k < len(present) and s == present[k]:
            w = sub[k].t
            D = w.shape[1]
            k += 1
            full.append(qb.Array(w.transpose(2, 3).contiguous()))   # mpo_apply contracts u
        else:
            import torch
            eye = torch.eye(D, dtype=sub[0].t.dtype, device=sub[0].t.device)
            full.append(qb.Array((eye[:, :, None, None]
                                  * torch.eye(2, dtype=eye.dtype, device=eye.device))))
    return qb.tebd.mpo_apply(full, psi)


def apply(method, psi, G, where, controls, chi):
    import quimb_b200 as qb
    if method == "swap":
        out = list(psi)
        qb.gate_with_auto_swap(out, G, where, max_bond=chi, cutoff=1e-10)
        return out
    info = {"cur_orthog": (min(where + controls), min(where + controls))}
    if controls:
        return qb.mps_gate_controlled(psi, G, where, controls, method=method, max_bond=chi,
                                      info=info)
    return qb.mps_gate_nonlocal(psi, G, where, method=method, max_bond=chi, info=info)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--chis", default="256,1024")
    ap.add_argument("--dtypes", default="float64,complex128")
    ap.add_argument("--budget-s", type=float, default=120.0)
    ap.add_argument("--gates", default="cx10,cx50,ccx10,c2x")
    ap.add_argument("--methods", default="swap," + ",".join(METHODS))
    args = ap.parse_args()
    wanted = args.methods.split(",")

    import torch
    import quimb_b200 as qb
    print(json.dumps(card()), flush=True)
    L = args.L
    measured = {}
    for chi in (int(c) for c in args.chis.split(",")):
        for dtype in args.dtypes.split(","):
            for gname, (G, where, controls) in gates(L).items():
                if gname not in args.gates.split(","):
                    continue
                psi = rand_sites(L, chi, 2, dtype, seed=chi)
                qb.mps_canonicalize(psi, min(where + controls))
                ref = exact(psi, G, where, controls)
                methods = (("swap",) if not controls and len(where) == 2 else ()) + METHODS
                methods = [m for m in methods if m in wanted]
                for method in methods:
                    row = {"chi": chi, "dtype": dtype, "L": L, "gate": gname,
                           "where": list(where), "controls": list(controls), "method": method}
                    key = (gname, method, dtype)
                    if key in measured:
                        c0, s0 = measured[key]
                        row["predicted_seconds"] = s0 * (chi / c0) ** 3
                        if row["predicted_seconds"] > args.budget_s:
                            row["skipped"] = (f"predicted {row['predicted_seconds']:.0f} s > "
                                              f"budget {args.budget_s:.0f} s")
                            print(json.dumps(row), flush=True)
                            continue
                    # warm-up: the same call on a short chain
                    lo = min(where + controls)
                    short = rand_sites(24, min(chi, 64), 2, dtype, seed=1)
                    sh = tuple(w - lo + 1 for w in where)
                    sc = tuple(c - lo + 1 for c in controls)
                    if max(sh + sc) < 24:
                        apply(method, short, G, sh, sc, min(chi, 64))
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    m0 = torch.cuda.memory_allocated()
                    t0 = time.perf_counter()
                    out = apply(method, psi, G, where, controls, chi)
                    torch.cuda.synchronize()
                    row["seconds"] = time.perf_counter() - t0
                    measured[key] = (chi, row["seconds"])
                    row["peak_bytes"] = int(torch.cuda.max_memory_allocated() - m0)
                    row["bonds_max"] = max(x.shape[2] for x in out)
                    row["fidelity"] = float(fidelity(out, ref))
                    del out
                    if row["seconds"] * 2 < args.budget_s:
                        timer = SplitTimer()
                        try:
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                            apply(method, psi, G, where, controls, chi)
                            torch.cuda.synchronize()
                            wall = time.perf_counter() - t0
                        finally:
                            timer.close()
                        row["split_share"] = timer.seconds / wall
                    print(json.dumps(row), flush=True)
                    torch.cuda.empty_cache()
                del psi, ref
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
