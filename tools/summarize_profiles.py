"""Turn the ncu artefacts in gpurun_out/ into the committed text summaries
under profiles/ (run here, no GPU needed)."""
import collections
import csv
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "gpurun_out")
P = os.path.join(ROOT, "profiles")
TAG = sys.argv[1] if len(sys.argv) > 1 else "r01"

KEYS = [
    "Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum",
    "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
    "launch__cluster_size", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_tensor_subpipe_dmma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tensor.sum",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_ld.sum",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__inst_executed.sum",
]


def launches():
    f = os.path.join(G, f"launches_{TAG}.csv")
    if not os.path.exists(f):
        return
    rows = [r for r in csv.reader(open(f)) if len(r) > 10]
    hdr = rows[0]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    gi, bi = hdr.index("Grid Size"), hdr.index("Block Size")
    tot = collections.OrderedDict()
    for r in rows[1:]:
        try:
            v = float(r[vi].replace(",", ""))
        except ValueError:
            continue
        if r[ui] == "us":
            v *= 1e3
        key = (r[ki].split("(")[0][:64], r[gi], r[bi])
        d = tot.setdefault(key, [0, 0.0])
        d[0] += 1
        d[1] += v
    T = sum(v[1] for v in tot.values())
    lines = [
        f"# ncu launch list, {TAG}: `ncu --metrics gpu__time_duration.sum --clock-control none "
        "-k regex:<our kernels> python bench.py --steps 1 --warmup 3 --no-e2e --no-cpu-baseline`",
        "# per-launch times are cold-cache / serialised under the profiler: compare SHARES, not absolutes",
        "# workload: 4 passes of the L=200 chi=1024 fp64 MPS norm",
        "", f"{'launches':>8} {'total_ms':>10} {'share':>7} {'avg_us':>9}  kernel  grid  block"]
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1][1]):
        lines.append(f"{v[0]:8d} {v[1] / 1e6:10.3f} {100 * v[1] / T:6.2f}% {v[1] / v[0] / 1e3:9.1f}  "
                     f"{k[0]}  {k[1]}  {k[2]}")
    lines.append(f"\ntotal {T / 1e6:.3f} ms over {sum(v[0] for v in tot.values())} launches")
    open(os.path.join(P, f"{TAG}_launches_bench_mps_norm.txt"), "w").write("\n".join(lines) + "\n")


def full(rep, out, header):
    f = os.path.join(G, rep)
    if not os.path.exists(f):
        return
    raw = subprocess.run(["ncu", "-i", f, "--page", "raw", "--csv"], capture_output=True,
                         text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    rows = [r for r in rows if len(r) > 20]
    hdr, units = rows[0], rows[1]
    lines = list(header) + [""]
    for k in KEYS:
        for i, h in enumerate(hdr):
            if h == k:
                lines.append(f"{h} [{units[i]}]: " + " | ".join(r[i] for r in rows[2:]))
    open(os.path.join(P, out), "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    os.makedirs(P, exist_ok=True)
    launches()
    full(f"prof_contract_{TAG}.ncu-rep", f"{TAG}_contract_kernel_ncu_full.txt", [
        f"# ncu --set full --clock-control none --import-source on -k regex:contract_f64_streamk -s 1000 -c 2 "
        "(bench.py: MPS norm L=200 chi=1024 fp64)",
        "# persistent stream-K launch of the 128x128x32 (3-stage, 8 warps, compile-time tile layouts) DMMA",
        "# contraction kernel, 148 CTAs, programmatic dependent launch",
        "# launch 1: E[a',a].A[a,(b,p)]  M=1024 N=2048 K=1024;  launch 2: conj(A)[(a',p),b'].T  M=N=1024 K=2048",
        "# algorithmic per launch: 4.295 GFLOP, 33.5 MB (fp64) -> tensor bound; DMMA peak measured 37.16 TFLOP/s"])
    full(f"prof_ozaki_{TAG}.ncu-rep", f"{TAG}_ozaki_gemm_ncu_full.txt", [
        "# ncu --set full --clock-control none -k regex:ozaki_gemm -s 2 -c 1 (tools/oz_prof.py: 4096^3 fp64)",
        "# tcgen05 kind::i8 error-free-split GEMM, 128x64 tiles, 36 slice products, TMA + TMEM",
        "# algorithmic: 137.4 GFLOP fp64 = 4.95 int8 POP; 3.03 ms -> 1.63 POP/s int8, L2 bound"])
    full(f"prof_jacobi_{TAG}.ncu-rep", f"{TAG}_jacobi_svd_ncu_full.txt", [
        "# ncu --set full --clock-control none --import-source on -k regex:jacobi_pair -s 300 -c 2 (tools/svd_prof.py 2048)",
        "# committed kernel: cluster 2, symmetric Gram, single-pass warp reduction, one inner sweep with",
        "# one barrier per step (per-warp rotations, ping-pong Gram), fused rotations"])
    print(os.listdir(P))
