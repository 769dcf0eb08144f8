"""Time the DMMA contraction kernel on plain fp64 GEMMs (GPU only): 4096³ and
two shapes of the chi=1024 MPS-norm step.  Prints one JSON line per shape
(ms per call, TFLOP/s, and for the smaller shapes the max error against
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
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
