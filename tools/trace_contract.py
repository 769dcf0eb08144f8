"""Phase timing of the contraction kernel from its in-kernel %globaltimer stamps
(QB_TRACE=1; GPU only).  Runs the two launches of one MPS-norm site
(chi=1024, d=2, an "lrp" site viewed as (l, p, r), as bench.py contracts it)
back to back and prints, per launch, the median over CTAs of each phase and
the gap between consecutive kernels.  The CTA count of each launch comes from
its route (the stream-K grid is one CTA per SM).

  python tools/trace_contract.py [--out trace.json]

phases: 0 entry, 1 tables done, 2 prologue issued, 3 first tile landed,
        4 main loop done, 5 stream-K fix-up done (pair schedule: the
        distributed-shared-memory exchange of the two k-halves), 6 stores issued

Each launch also reports its thread-block cluster shape (CTAs per cluster: 2
for the stream-K pair schedule, 1 otherwise) and, where every CTA runs the
same number of k-blocks (classic grid, pair schedule), the median main-loop
time per k-block, to set against the DMMA issue rate of the 8-warp tile
(DESIGN §5).
"""
import ctypes
import json
import os
import sys

os.environ.setdefault("QB_TRACE", "1")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import quimb_b200 as qb
from quimb_b200 import _lib, mps


def read_trace():
    n = 16 * 8192
    buf = (ctypes.c_ulonglong * n)()
    rc = _lib.load().qb_debug_trace_read(buf, n)
    assert rc == 0, rc
    return np.frombuffer(buf, dtype=np.uint64).reshape(16, 8192).copy()


def analyse(slot, G, schedule=None):
    t = slot[: G * 32].reshape(G, 4, 8).astype(np.int64)
    out = {}
    seg_used = (t[:, :, 0] > 0)
    t0 = t[:, 0, 0][seg_used[:, 0]]
    out["entry_spread_us"] = float((t0.max() - t0.min()) / 1e3)
    ends = np.where(seg_used, t[:, :, 6], 0).max(axis=1)
    out["start_ns"] = int(t0.min()); out["end_ns"] = int(ends.max())
    out["total_us"] = (out["end_ns"] - out["start_ns"]) / 1e3
    names = ["tables", "prologue_issue", "first_tile_wait", "main_loop",
             "exchange" if schedule == "pair" else "fixup", "stores"]
    for s in range(4):
        m = seg_used[:, s]
        if not m.any():
            continue
        d = {}
        for ph in range(6):
            a, b = t[m, s, ph], t[m, s, ph + 1]
            ok = (a > 0) & (b > 0)
            if ok.any():
                d[names[ph]] = round(float(np.median((b - a)[ok])) / 1e3, 2)
        d["n_cta"] = int(m.sum())
        out[f"seg{s}"] = d
    return out


def main():
    dev = torch.device("cuda:0")
    chi, d = 1024, 2
    g = torch.Generator(device=dev); g.manual_seed(0)
    # lrp storage, (l, p, r) view: strides (chi * d, 1, d)
    A = mps.site_lpr(torch.randn((chi, chi, d), dtype=torch.float64, device=dev, generator=g),
                     "lrp", 1, 3)
    E = qb.asarray(torch.randn((chi, chi), dtype=torch.float64, device=dev, generator=g))
    for _ in range(3):
        E2 = mps.norm_step(E, A)
    torch.cuda.synchronize()
    read_trace()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(4):
        E2 = mps.norm_step(E, A)
    e1.record(); torch.cuda.synchronize()
    print("4 sites:", e0.elapsed_time(e1) * 1e3, "us")
    tr = read_trace()
    used = [i for i in range(16) if tr[i].any()]
    # the CTAs of each launch: ket E . A, then bra conj(A) . T
    LB, L, P, R, RB = 0, 1, 2, 3, 4
    T = torch.empty((chi, d, chi), dtype=torch.float64, device=dev)
    a = A.t
    grids = []
    for (x, lx, y, ly, z, lz) in ((E.t, [LB, L], a, [L, P, R], T, [LB, P, R]),
                                  (a, [LB, P, RB], T, [LB, P, R], E2.t, [RB, R])):
        args = (list(x.shape), list(x.stride()), lx, list(y.shape), list(y.stride()), ly,
                list(z.shape), list(z.stride()), lz)
        ptrs = (x.data_ptr(), y.data_ptr(), z.data_ptr())
        r = qb.route_pair(*args, ptrs=ptrs)
        f = qb.feed_pair(*args, ptrs=ptrs)
        r["schedule"] = qb.schedule_pair(*args, ptrs=ptrs)
        tiles = (x.shape[0] // 128) * (z.numel() // x.shape[0] // 128) if r["streamk"] == 0 else 0
        K = int(np.prod([x.shape[i] for i, l in enumerate(lx) if l in ly and l not in lz]))
        nkb = -(-K // r["bk"])
        # k-blocks of one CTA: a classic CTA runs its split, a pair CTA one
        # k-half; stream-K segments differ from CTA to CTA
        kb_cta = {"pair": nkb / 2, None: nkb / r["splitk"]}.get(r["schedule"])
        grids.append((r["streamk"] or tiles, r, f, 2 if r["schedule"] == "pair" else 1, kb_cta))
        print(json.dumps({"route": r, "feed": f}))
    res = []
    for n, i in enumerate(used):
        G, r, f, cluster, kb_cta = grids[n % 2]
        a = analyse(tr[i], G, r["schedule"])
        loop = a.get("seg0", {}).get("main_loop")
        res.append({"kind": r["kind"], "layout": r["layout"], "ctas": G, "cluster": cluster,
                    "feed": f, "schedule": r["schedule"], "kblocks_per_cta": kb_cta,
                    "main_loop_us_per_kblock": round(loop / kb_cta, 3) if loop and kb_cta else None,
                    **a})
    res.sort(key=lambda r: r["start_ns"])
    for k, r in enumerate(res):
        gap = (r["start_ns"] - res[k - 1]["end_ns"]) / 1e3 if k else None
        print(json.dumps({"launch": k, "gap_before_us": gap, **{a: b for a, b in r.items()
                                                               if a not in ("start_ns", "end_ns")}}))
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
