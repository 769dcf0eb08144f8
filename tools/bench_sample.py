"""Batched MPS sampling benchmark (``quimb_b200.tebd.mps_sample``).

  python tools/bench_sample.py [--L 100] [--d 2] [--chis 256,1024]
                               [--Cs 10000,100000] [--dtypes float64,complex128]
                               [--oracle-samples 1000] [--out FILE]

For each workload (random right-canonicalisable MPS, ragged bonds
min(chi, d^i, d^(L-i))) it reports, as one JSON line:
  samples_per_s    end-to-end mps_sample (canonicalisation, uniforms, H2D,
                   the sampling loop, D2H), wall clock around a synchronised
                   call, after a warm-up call of the same shape;
  loop_s           the sampling loop alone (CUDA events around every step);
  gemm_tflops      2 C chi_l d chi_r per site (x4 complex) over the time of
                   the contraction launches;
  select_gbps      bytes qb_sample_select must move (W read once, V written,
                   u / config / omega) over its time;
  select_share     share of the loop spent in qb_sample_select;
  oracle_*         the numpy oracle (oracle/sample_np.py) on the CPU over the
                   first --oracle-samples samples of the chi <= 256 workloads,
                   from the same prepared state and uniforms (its
                   configurations are checked equal to the device's).
The card name and power limit are read in the same run.
"""
import argparse
import json
import os
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


def rand_sites(L, chi, d, dtype, seed):
    import torch
    import quimb_b200 as qb
    g = torch.Generator(device="cuda").manual_seed(seed)
    tdt = {"float64": torch.float64, "complex128": torch.complex128}[dtype]
    bonds = [1] + [min(chi, d ** min(i, 30), d ** min(L - i, 30)) for i in range(1, L)] + [1]
    out = []
    for i in range(L):
        x = torch.randn((bonds[i], d, bonds[i + 1]), generator=g, device="cuda", dtype=tdt)
        out.append(qb.Array(x / (bonds[i] * d) ** 0.5))
    return out


def run(L, d, chi, C, dtype, oracle_samples, seed=0):
    import torch
    from quimb_b200 import tebd as tb
    sites = rand_sites(L, chi, d, dtype, seed)
    # warm-up of every shape the timed call uses
    tb.mps_sample(sites, C, seed=seed)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cfgs, oms = tb.mps_sample(sites, C, seed=seed + 1)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0

    psi, _ = tb._sample_prepare(sites)
    u = np.random.default_rng(seed + 1).random((C, L))
    ud = torch.from_numpy(u).cuda()
    cd = torch.empty((C, L), dtype=torch.int64, device="cuda")
    od = torch.ones(C, dtype=torch.float64, device="cuda")
    events = []
    torch.cuda.synchronize()
    n_chunks = tb._sample_chunks(psi, ud, cd, od, events=events)
    torch.cuda.synchronize()
    t_gemm = t_sel = 0.0
    flops = sel_bytes = 0
    esz = 16 if dtype == "complex128" else 8
    for rows, i, e0, e1, e2 in events:
        l, dd, r = psi[i].shape
        t_gemm += e0.elapsed_time(e1) * 1e-3
        t_sel += e1.elapsed_time(e2) * 1e-3
        flops += 2 * rows * l * dd * r * (4 if dtype == "complex128" else 1)
        sel_bytes += rows * (dd * r * esz + r * esz + 8 + 8 + 16)
    assert np.array_equal(cd.cpu().numpy(), cfgs), "loop and mps_sample disagree"
    rec = {"L": L, "d": d, "chi": chi, "C": C, "dtype": dtype, "chunks": n_chunks,
           "wall_s": wall, "samples_per_s": C / wall, "loop_s": t_gemm + t_sel,
           "gemm_s": t_gemm, "gemm_tflops": flops / t_gemm * 1e-12,
           "select_s": t_sel, "select_gbps": sel_bytes / t_sel * 1e-9,
           "select_share": t_sel / (t_gemm + t_sel)}
    if oracle_samples and chi <= 256:
        from oracle import sample_np
        host = [np.asarray(a.to_numpy()) for a in psi]
        n = min(oracle_samples, C)
        t0 = time.perf_counter()
        oc, _, margin = sample_np.sample_uniforms(host, u[:n])
        t_or = time.perf_counter() - t0
        rec.update({"oracle_samples": n, "oracle_samples_per_s": n / t_or,
                    "oracle_configs_equal": bool(np.array_equal(oc, cfgs[:n])),
                    "oracle_margin": margin})
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--d", type=int, default=2)
    ap.add_argument("--chis", default="256,1024")
    ap.add_argument("--Cs", default="10000,100000")
    ap.add_argument("--dtypes", default="float64,complex128")
    ap.add_argument("--oracle-samples", type=int, default=1000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import quimb_b200 as qb  # noqa: F401
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample.py needs a CUDA device")
    head = card()
    print(json.dumps(head), flush=True)
    recs = []
    for dtype in a.dtypes.split(","):
        for chi in map(int, a.chis.split(",")):
            for C in map(int, a.Cs.split(",")):
                rec = run(a.L, a.d, chi, C, dtype, a.oracle_samples)
                recs.append(rec)
                print(json.dumps(rec), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump({"card": head, "runs": recs}, fh, indent=1)


if __name__ == "__main__":
    main()
