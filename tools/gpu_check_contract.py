"""Developer check (run under gpurun): contraction kernel vs torch.einsum on
the device, plus quick timings.  Not part of the test-suite (tests/ compare
against the numpy oracle); this is the fast iteration loop for the kernel."""

import itertools
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from quimb_b200 import _lib  # noqa: E402
from quimb_b200.contract import contract_pair  # noqa: E402

torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda:0")
LET = "abcdefghijklmnopqrstuvwxyz"


def rnd(shape, dtype):
    g = torch.Generator(device="cpu").manual_seed(hash(tuple(shape)) % 2**31)
    if dtype.is_complex:
        x = torch.randn(tuple(shape) + (2,), generator=g, dtype=torch.float64)
        return torch.view_as_complex(x).to(dev)
    return torch.randn(tuple(shape), generator=g, dtype=dtype).to(dev)


def check(name, ea, eb, ec, sizes, dtype=torch.float64, conj=(False, False),
          views=None):
    a = rnd([sizes[c] for c in ea], dtype)
    b = rnd([sizes[c] for c in eb], dtype)
    if views:
        a, b = views(a, b)
    la = [LET.index(c) for c in ea]
    lb = [LET.index(c) for c in eb]
    lc = [LET.index(c) for c in ec]
    out = contract_pair(a, la, b, lb, lc, conj_a=conj[0], conj_b=conj[1])
    ra = a.conj() if conj[0] else a
    rb = b.conj() if conj[1] else b
    ref = torch.einsum(f"{ea},{eb}->{ec}", ra, rb)
    err = (out - ref).abs().max().item() if ref.numel() else 0.0
    scale = max(ref.abs().max().item() if ref.numel() else 1.0, 1e-300)
    ok = err <= 1e-11 * max(scale, 1.0) * 50
    print(f"{'OK ' if ok else 'BAD'} {name:34s} {ea},{eb}->{ec} err={err:.2e} "
          f"scale={scale:.2e}", flush=True)
    return ok


def main():
    lib = _lib.load()
    ok = True
    S = dict(a=37, b=45, c=29, d=18, e=6, f=50, g=3)
    ok &= check("gemm", "ab", "bc", "ac", S)
    ok &= check("gemm big-ish", "ab", "bc", "ac", dict(a=300, b=257, c=190))
    ok &= check("gemm TN", "ba", "bc", "ac", S)
    ok &= check("gemm NT", "ab", "cb", "ac", S)
    ok &= check("gemm TT out-T", "ba", "cb", "ca", S)
    ok &= check("tensordot cfg1", "abcd", "cdef", "abef", dict(a=12, b=11, c=10, d=9, e=8, f=7))
    ok &= check("tensordot perm", "acbd", "dfce", "abef", dict(a=12, b=11, c=10, d=9, e=8, f=7))
    ok &= check("out permuted", "abcd", "cdef", "feba", dict(a=12, b=11, c=10, d=9, e=8, f=7))
    ok &= check("batch", "gab", "gbc", "gac", S)
    ok &= check("batch mid", "agb", "bcg", "acg", S)
    ok &= check("outer", "ab", "cd", "abcd", S)
    ok &= check("scalar out", "abc", "abc", "", S)
    ok &= check("rank0 operand", "", "ab", "ab", S)
    ok &= check("sum index A", "abe", "bc", "ac", S)
    ok &= check("sum index B", "ab", "bce", "ac", S)
    ok &= check("matvec", "ab", "b", "a", dict(a=1000, b=777))
    ok &= check("vec-mat", "a", "ab", "b", dict(a=1000, b=777))
    ok &= check("dot long", "a", "a", "", dict(a=1_000_003))
    ok &= check("mps step1", "ax", "abp", "xbp", dict(a=64, x=64, b=64, p=2))
    ok &= check("mps step2", "xbp", "xyp", "by", dict(x=64, b=64, y=64, p=2))
    ok &= check("dmrg L.x", "xwa", "asbt", "xwsbt", dict(x=32, w=5, a=32, s=2, b=32, t=2))
    ok &= check("dmrg .W", "xwsbt", "wvsu", "xvubt", dict(x=32, w=5, s=2, b=32, t=2, v=5, u=2))
    ok &= check("dmrg .R", "xvubz", "yvb", "xuyz",
                dict(x=32, v=5, u=2, b=32, z=2, y=32))
    ok &= check("dim2 many", "abcdefg", "gfedcba"[::1], "", {c: 2 for c in "abcdefg"})
    ok &= check("dim2 mixed", "abcdefg", "cdexyz", "abfgxyz", {c: 2 for c in "abcdefgxyz"})

    # explicit non-contiguous views
    a = rnd([40, 90], torch.float64)[3:, ::2]
    b = rnd([90, 33], torch.float64)[::2, :-3]
    out = contract_pair(a, [0, 1], b, [1, 2], [0, 2])
    ref = a @ b
    e = (out - ref).abs().max().item()
    print(("OK " if e < 1e-10 else "BAD"), "sliced views err", e)
    ok &= e < 1e-10
    # transposed output view
    outT = torch.empty(30, 37, dtype=torch.float64, device=dev)
    a = rnd([37, 45], torch.float64)
    b = rnd([45, 30], torch.float64)
    contract_pair(a, [0, 1], b, [1, 2], [0, 2], out=outT.t())
    e = (outT.t() - a @ b).abs().max().item()
    print(("OK " if e < 1e-10 else "BAD"), "strided out err", e)
    ok &= e < 1e-10

    # complex128
    for conj in itertools.product((False, True), repeat=2):
        ok &= check(f"c128 gemm conj={conj}", "ab", "bc", "ac", S, torch.complex128, conj)
        ok &= check(f"c128 perm conj={conj}", "acbd", "dfce", "abef",
                    dict(a=6, b=7, c=5, d=9, e=8, f=7), torch.complex128, conj)
    ok &= check("c128 scalar", "abc", "abc", "", S, torch.complex128, (True, False))
    ok &= check("c128 batch", "gab", "gbc", "gac", S, torch.complex128)
    ok &= check("c128 dim2", "abcdefg", "cdexyz", "abfgxyz", {c: 2 for c in "abcdefgxyz"}, torch.complex128)
    ok &= check("c128 big", "ab", "bc", "ac", dict(a=300, b=257, c=190), torch.complex128)
    print("ALL OK" if ok else "SOME FAILED", flush=True)

    # ---------------- timings ----------------
    import ctypes
    tf = ctypes.c_double()
    rc = lib.qb_measure_dmma_peak(ctypes.byref(tf), None)
    print("dmma peak TFLOP/s:", tf.value, "rc", rc, flush=True)
    res = {"dmma_peak_tflops": tf.value}

    def timeit(fn, n=5):
        fn(); torch.cuda.synchronize()
        ts = []
        for _ in range(n):
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return min(ts), sorted(ts)[len(ts) // 2]

    n = 4096
    a = torch.randn(n, n, dtype=torch.float64, device=dev)
    b = torch.randn(n, n, dtype=torch.float64, device=dev)
    c = torch.empty(n, n, dtype=torch.float64, device=dev)
    fl = 2 * n ** 3
    tmin, tmed = timeit(lambda: contract_pair(a, [0, 1], b, [1, 2], [0, 2], out=c))
    print(f"gemm NN 4096^3 auto: {tmin:.3f} ms  {fl / tmin / 1e9:.2f} TFLOP/s", flush=True)
    res["gemm_nn_4096"] = fl / tmin / 1e9
    tmin, _ = timeit(lambda: contract_pair(a, [1, 0], b, [1, 2], [0, 2], out=c))
    print(f"gemm TN 4096^3: {tmin:.3f} ms  {fl / tmin / 1e9:.2f} TFLOP/s", flush=True)
    tmin, _ = timeit(lambda: contract_pair(a, [0, 1], b, [2, 1], [0, 2], out=c))
    print(f"gemm NT 4096^3: {tmin:.3f} ms  {fl / tmin / 1e9:.2f} TFLOP/s", flush=True)
    tmin, _ = timeit(lambda: torch.matmul(a, b, out=c))
    print(f"cublas dgemm 4096^3: {tmin:.3f} ms  {fl / tmin / 1e9:.2f} TFLOP/s", flush=True)
    res["cublas_dgemm_4096"] = fl / tmin / 1e9
    # cfg1-variant with permutations, chi=64
    A = torch.randn(64, 64, 64, 64, dtype=torch.float64, device=dev)
    B = torch.randn(64, 64, 64, 64, dtype=torch.float64, device=dev)
    tmin, _ = timeit(lambda: contract_pair(A, [0, 2, 1, 3], B, [3, 5, 2, 4], [0, 1, 4, 5]))
    print(f"cfg1 perm (acbd,dfce->abef) 64^4: {tmin:.3f} ms {fl / tmin / 1e9:.2f} TFLOP/s", flush=True)
    tmin, _ = timeit(lambda: torch.einsum("acbd,dfce->abef", A, B))
    print(f"torch.einsum same: {tmin:.3f} ms {fl / tmin / 1e9:.2f} TFLOP/s", flush=True)
    # MPS norm steps chi=1024
    chi, d = 1024, 2
    E = torch.randn(chi, chi, dtype=torch.float64, device=dev)
    T = torch.randn(chi, chi, d, dtype=torch.float64, device=dev)
    f1 = 2 * chi * chi * chi * d
    tmin, _ = timeit(lambda: contract_pair(E, [0, 1], T, [0, 2, 3], [1, 2, 3]))
    print(f"mps step1 chi=1024: {tmin:.3f} ms {f1 / tmin / 1e9:.2f} TFLOP/s", flush=True)
    X = torch.randn(chi, chi, d, dtype=torch.float64, device=dev)
    tmin, _ = timeit(lambda: contract_pair(X, [1, 2, 3], T, [1, 4, 3], [2, 4]))
    print(f"mps step2 chi=1024: {tmin:.3f} ms {f1 / tmin / 1e9:.2f} TFLOP/s", flush=True)
    res["mps_step2"] = f1 / tmin / 1e9
    # DMRG matvec steps
    w = 5
    L = torch.randn(chi, w, chi, dtype=torch.float64, device=dev)
    x = torch.randn(chi, d, chi, d, dtype=torch.float64, device=dev)
    f = 2 * chi * w * chi * d * chi * d
    tmin, _ = timeit(lambda: contract_pair(L, [0, 1, 2], x, [2, 3, 4, 5], [0, 1, 3, 4, 5]))
    print(f"dmrg L.x: {tmin:.3f} ms {f / tmin / 1e9:.2f} TFLOP/s", flush=True)
    T1 = torch.randn(chi, w, d, chi, d, dtype=torch.float64, device=dev)
    W = torch.randn(w, w, d, d, dtype=torch.float64, device=dev)
    f = 2 * chi * chi * d * (w * d) * (w * d)
    tmin, _ = timeit(lambda: contract_pair(T1, [0, 1, 2, 3, 4], W, [1, 6, 2, 7], [0, 6, 7, 3, 4]))
    byt = 2 * T1.numel() * 8
    print(f"dmrg .W: {tmin:.3f} ms {f / tmin / 1e9:.2f} TFLOP/s {byt / tmin / 1e6:.1f} GB/s", flush=True)
    # complex gemm
    n = 2048
    ac = torch.randn(n, n, dtype=torch.complex128, device=dev)
    bc = torch.randn(n, n, dtype=torch.complex128, device=dev)
    tmin, _ = timeit(lambda: contract_pair(ac, [0, 1], bc, [1, 2], [0, 2]))
    print(f"zgemm 2048^3: {tmin:.3f} ms {8 * n**3 / tmin / 1e9:.2f} TFLOP/s(real)", flush=True)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(res, open("gpurun_out/check_contract.json", "w"))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
