"""SVD profile helper (GPU box): sweeps, time, accuracy against LAPACK (when
asked) and -- with QB_TRACE=1 -- the phase breakdown of the Jacobi round kernel
from its in-kernel %globaltimer stamps (cluster 0 of every launch).

phases: 0 entry, 1 Gram streamed, 2 Gram reduced over the cluster + off-norm,
        3 32x32 eigen-solve done, 4 sorted, 5 rotation applied, 6 cluster exit
"""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import quimb_b200 as qb
from quimb_b200 import _lib

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
check = "--check" in sys.argv
g = torch.Generator(device="cuda").manual_seed(1)
X = qb.Array(torch.randn(n, n, dtype=torch.float64, device='cuda', generator=g))
qb.linalg.svd(X)
torch.cuda.synchronize()
ts = []
for _ in range(3):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    U, s, VH, sw = qb.linalg.svd(X, return_sweeps=True)
    e1.record(); torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
out = {"n": n, "sweeps": sw, "ms": min(ts), "ms_all": ts}
# fused truncated split (DMRG shape: keep half, absorb right)
for name, code in (("trunc_ms", 1), ("trunc_left_ms", -1), ("trunc_both_ms", 0)):
    ts2 = []
    for _ in range(2):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        l, _, r = qb.linalg.svd_trunc(X, cutoff=0.0, cutoff_mode=3, max_bond=n // 2, absorb=code)
        e1.record(); torch.cuda.synchronize()
        ts2.append(e0.elapsed_time(e1))
    out[name] = min(ts2)
l, _, r = qb.linalg.svd_trunc(X, cutoff=0.0, cutoff_mode=3, max_bond=n // 2, absorb=1)
if check:
    x = X.to_numpy()
    sref = np.linalg.svd(x, compute_uv=False)
    u, v = U.to_numpy(), VH.to_numpy()
    out["sv_err"] = float(np.abs(s.to_numpy() - sref).max() / sref[0])
    out["u_orth"] = float(np.abs(u.T @ u - np.eye(n)).max())
    out["v_orth"] = float(np.abs(v @ v.T - np.eye(n)).max())
    out["recon"] = float(np.abs((u * s.to_numpy()) @ v - x).max() / sref[0])
    out["trunc_l_orth"] = float(np.abs(l.to_numpy().T @ l.to_numpy() - np.eye(n // 2)).max())
    out["trunc_recon"] = float(np.abs(l.to_numpy() @ r.to_numpy() - (u[:, :n // 2] * sref[:n // 2]) @ v[:n // 2]).max() / sref[0])
print(json.dumps(out), flush=True)
if os.environ.get("QB_TRACE"):
    cnt = 17 * 8192
    buf = (ctypes.c_ulonglong * cnt)()
    assert _lib.load().qb_debug_trace_read(buf, cnt) == 0
    t = np.frombuffer(buf, dtype=np.uint64)[16 * 8192:16 * 8192 + 1024 * 8].reshape(1024, 8).astype(np.int64)
    ok = (t[:, 0] > 0) & (t[:, 6] > t[:, 0]) & (t[:, 3] > t[:, 2])   # rounds that rotated
    names = ["gram_stream", "reduce+offnorm", "eigensolve", "sort", "apply", "cluster_exit"]
    tr = {}
    for ph in range(6):
        a, b = t[ok, ph], t[ok, ph + 1]
        m = (b >= a) & (a > 0)
        if m.any():
            tr[names[ph]] = round(float(np.median((b - a)[m])) / 1e3, 2)
    starts = np.sort(t[ok, 0])
    tr["launch_period_us"] = round(float(np.median(np.diff(starts))) / 1e3, 2) if len(starts) > 2 else None
    tr["rounds_traced"] = int(ok.sum())
    print(json.dumps(tr), flush=True)
