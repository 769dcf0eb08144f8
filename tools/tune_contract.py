"""Time the DMMA contraction kernel (GPU only): plain fp64 GEMMs (4096³ and
the two GEMM shapes of the chi=1024 MPS-norm step, row-major), then the two
launches of the MPS-norm step at the strides bench.py runs them with (an
"lrp" site viewed as (l, p, r)).  Prints one JSON line per shape (ms per
call, TFLOP/s, and for the smaller shapes the max error against
torch.matmul).

  python tools/tune_contract.py [--out result.json]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [[4096, 4096, 4096], [1024, 2048, 1024], [1024, 1024, 2048]]  # (M, N, K)


def main():
    import torch
    from quimb_b200.contract import contract_pair
    dev = torch.device("cuda:0")
    out = {}
    for (M, N, K) in SHAPES:
        g = torch.Generator(device=dev); g.manual_seed(1)
        A = torch.randn((M, K), dtype=torch.float64, device=dev, generator=g)
        B = torch.randn((K, N), dtype=torch.float64, device=dev, generator=g)
        C = torch.empty((M, N), dtype=torch.float64, device=dev)
        for _ in range(3):
            contract_pair(A, [0, 1], B, [1, 2], [0, 2], out=C)
        torch.cuda.synchronize()
        reps = 10 if M * N * K >= 2 ** 34 else 50
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            contract_pair(A, [0, 1], B, [1, 2], [0, 2], out=C)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        err = float((C - A @ B).abs().max().item()) if M <= 2048 else None
        out[f"{M}x{N}x{K}"] = r = {"ms": round(ms, 4),
                                   "tflops": round(2.0 * M * N * K / ms / 1e9, 2), "err": err}
        print(json.dumps({f"{M}x{N}x{K}": r}), flush=True)
    # E[a', a] A[a, p, b] -> T[a', p, b], then conj(A)[a', p, b'] T[a', p, b] -> E'[b', b]
    chi, d = 1024, 2
    g = torch.Generator(device=dev); g.manual_seed(2)
    site = torch.randn((chi, chi, d), dtype=torch.float64, device=dev, generator=g).permute(0, 2, 1)
    E = torch.randn((chi, chi), dtype=torch.float64, device=dev, generator=g)
    T = torch.empty((chi, d, chi), dtype=torch.float64, device=dev)
    E2 = torch.empty((chi, chi), dtype=torch.float64, device=dev)
    LB, L, P, R, RB = 0, 1, 2, 3, 4
    steps = {"mps_ket_1024x2048x1024": (E, [LB, L], site, [L, P, R], [LB, P, R], T),
             "mps_bra_1024x1024x2048": (site, [LB, P, RB], T, [LB, P, R], [RB, R], E2)}
    for name, (x, lx, y, ly, lz, z) in steps.items():
        for _ in range(3):
            contract_pair(x, lx, y, ly, lz, out=z)
        torch.cuda.synchronize()
        reps = 50
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            contract_pair(x, lx, y, ly, lz, out=z)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        out[name] = r = {"ms": round(ms, 4), "tflops": round(2.0 * chi ** 3 * d / ms / 1e9, 2)}
        print(json.dumps({name: r}), flush=True)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
