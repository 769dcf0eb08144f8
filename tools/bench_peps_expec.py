"""PEPS local-expectation benchmark (``quimb_b200.peps_expec``).

  python tools/bench_peps_expec.py [--sizes 8x8:4:32,10x10:6:64]
                                   [--dtypes complex128,complex64] [--reps 2]
                                   [--no-oracle]

For each workload (seeded random PEPS, d = 2, sites scaled to O(1) norm
contributions) it computes the normalized energy of the Heisenberg model with
a Z field (bonds on 1x2 / 2x1 plaquettes, fields on 1x2 plaquettes) and
prints one JSON line with, after one warm-up call:
  total_s            wall time of peps_compute_local_expectation, ending in a
                     device synchronise (median of --reps);
  envs_s, rho_s,     the same call split into plaquette environments, the
  terms_s            reduced density matrices and the term kernel (each
                     part synchronised);
  per_term_s         the term evaluation with one qb_plaquette_expec launch,
                     descriptor copy and read-back per term, on the same rho;
  launches, host_reads, peak_bytes   of one call (the instrumented one);
  oracle_s           the numpy oracle's time for the same energy (first size
                     only; the CPU column).
The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402


def card():
    import torch
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = q
    except Exception as e:  # noqa: BLE001
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def workload(Lx, Ly, D, dtype, seed=7):
    from oracle import peps_expec_np as pe
    arrays = pe.rand_peps(Lx, Ly, D, 2, seed, dtype)
    # O(1) entries per boundary step: scale each site by its bond count
    arrays = [[(a / np.sqrt(a.size / 2)).astype(dtype) for a in row] for row in arrays]
    terms = pe.heis_terms(Lx, Ly, 2, field=0.3)
    return arrays, terms


class Parts:
    """Synchronised timers around the three parts of one call."""

    def __init__(self, px):
        import torch
        self.px, self.t, self.saved = px, {}, {}
        for name in ("plaquette_environments", "plaquette_rhos", "plaquette_expec"):
            fn = getattr(px, name)
            self.saved[name] = fn

            def timed(*a, _fn=fn, _name=name, **kw):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = _fn(*a, **kw)
                torch.cuda.synchronize()
                self.t[_name] = self.t.get(_name, 0.0) + time.perf_counter() - t0
                return out
            setattr(px, name, timed)

    def restore(self):
        for name, fn in self.saved.items():
            setattr(self.px, name, fn)


class HostReads:
    """Counts device-to-host reads (item / cpu / tolist) during a call."""

    def __init__(self):
        import torch
        self.n, self.saved = 0, {}
        for name in ("item", "cpu", "tolist"):
            orig = getattr(torch.Tensor, name)
            self.saved[name] = orig

            def counted(t, *a, _orig=orig, **kw):
                if t.device.type == "cuda":
                    self.n += 1
                return _orig(t, *a, **kw)
            setattr(torch.Tensor, name, counted)

    def restore(self):
        import torch
        for name, fn in self.saved.items():
            setattr(torch.Tensor, name, fn)


def run(Lx, Ly, D, chi, dtype, reps, oracle):
    import torch
    import quimb_b200 as qb
    from quimb_b200 import peps_expec as px
    arrays, terms = workload(Lx, Ly, D, dtype)
    dev = [[qb.asarray(a) for a in row] for row in arrays]
    kw = dict(cutoff=0.0, normalized=True)

    def call():
        return qb.peps_compute_local_expectation(dev, terms, chi, **kw)

    value = call()                              # warm-up of every shape
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    # one instrumented call: the split, launches, host reads and peak; the
    # term kernel's arguments are kept for the one-launch-per-term comparison
    kept = {}
    inner = px.plaquette_expec

    def keep(rho, offsets, items):
        kept.update(rho=rho, offsets=offsets, items=items)
        return inner(rho, offsets, items)
    px.plaquette_expec = keep
    parts = Parts(px)
    torch.cuda.reset_peak_memory_stats()
    n0 = qb.launch_count()
    reads = HostReads()
    try:
        call()
    finally:
        reads.restore()
        parts.restore()
        px.plaquette_expec = inner
    launches = qb.launch_count() - n0
    peak = torch.cuda.max_memory_allocated()
    rho, offsets, items = kept["rho"], kept["offsets"], kept["items"]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    batched = px.plaquette_expec(rho, offsets, items)
    torch.cuda.synchronize()
    one_launch = time.perf_counter() - t0
    t0 = time.perf_counter()
    single = [px.plaquette_expec(rho, offsets, [it])[0] for it in items]
    torch.cuda.synchronize()
    per_term = time.perf_counter() - t0
    assert all(a[0] == b[0] for a, b in zip(batched, single))
    rec = {"workload": f"{Lx}x{Ly} D={D} chi={chi}", "dtype": np.dtype(dtype).name,
           "terms": len(terms), "plaquettes": len(offsets), "value": complex(value).real,
           "total_s": statistics.median(times), "total_all_s": times,
           "envs_s": parts.t.get("plaquette_environments"),
           "rho_s": parts.t.get("plaquette_rhos"), "terms_s": parts.t.get("plaquette_expec"),
           "terms_one_launch_s": one_launch, "per_term_s": per_term,
           "launches": launches, "host_reads": reads.n, "peak_bytes": peak}
    if oracle:
        from oracle import peps_expec_np as pe
        t0 = time.perf_counter()
        want, _ = pe.compute_local_expectation(arrays, terms, chi, cutoff=0.0, normalized=True)
        rec["oracle_s"] = time.perf_counter() - t0
        rec["oracle_rel_diff"] = abs(complex(value) - complex(want)) / abs(complex(want))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8x8:4:32,10x10:6:64")
    ap.add_argument("--dtypes", default="complex128,complex64")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_peps_expec.py needs a CUDA device")
    print(json.dumps(card()), flush=True)
    for k, spec in enumerate(args.sizes.split(",")):
        lat, D, chi = spec.split(":")
        Lx, Ly = map(int, lat.split("x"))
        for dt in args.dtypes.split(","):
            rec = run(Lx, Ly, int(D), int(chi), np.dtype(dt).type, args.reps,
                      oracle=(k == 0 and dt == "complex128" and not args.no_oracle))
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
