"""DMRG-X benchmark (``quimb_b200.DMRGX``).

  python tools/bench_dmrgx.py [--configs 32x32,64x64] [--sweeps 2]
                              [--max-sites 0] [--oracle-L 32] [--oracle-sites 9]
                              [--out DIR]

Workload: the random-field Heisenberg (MBL) chain, fields uniform in
[-8, 8], from a computational basis state with bonds padded by noise of
strength 1e-9 to chi, so that every bulk site solves a local problem of
D = chi * 2 * chi (2048 at chi = 32, 8192 at chi = 64).  After one warm-up
sweep, ``--sweeps`` sweeps (alternating direction, no re-canonisation) are
timed.  For every configuration it prints one JSON line with
  seconds_timed       host clock around the synchronised timed sweeps, and
                      seconds_per_sweep when they ran to the end;
  split_seconds_timed device-event seconds in: assembly (the dense Heff),
                      eigh, selection (overlaps and candidate <H^2>, host
                      reads included), environments (the three moving
                      environments) and canonisation (QR moves);
  sites_timed         the site updates these cover: with --max-sites N a
                      sweep stops after N updates;
  seconds_per_bulk_site, seconds_per_sweep_from_sites
                      every update is also timed on its own (synchronised):
                      the median at the bulk D, and the sweep it implies
                      (edge ramp measured, the rest at the bulk time).
The numpy oracle is timed on the same host at --oracle-L (chi = 32): its
first --oracle-sites updates of a sweep, and the sweep they imply.  The card name and power limit are read in the same
run; everything is also written to <out>/bench_dmrgx.json.
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tools.bench_observables import card  # noqa: E402


class _Stop(Exception):
    pass


class PhaseTimer:
    """CUDA events around the sweep's phases (wrapped module attributes)."""

    def __init__(self):
        import torch
        from quimb_b200 import dmrgx, tebd
        self.torch = torch
        self.pairs = {k: [] for k in ("assembly", "eigh", "selection", "environments",
                                      "canonisation")}
        self.saved = []
        phases = [
            (dmrgx.DMRGX, "dense_heff", "assembly"),
            (dmrgx, "eigh", "eigh"),
            (dmrgx.DMRGX, "_overlaps", "selection"),
            (dmrgx.DMRGX, "_candidate_en2", "selection"),
            (tebd, "left_canonize_site", "canonisation"),
            (tebd, "right_canonize_site", "canonisation"),
        ]
        for name in ("env_left_step", "env_right_step", "env2_left_step",
                     "env2_right_step", "norm_step", "norm_step_right"):
            phases.append((dmrgx, name, "environments"))
        for obj, name, phase in phases:
            self._wrap(obj, name, phase)

    def _wrap(self, obj, name, phase):
        inner = getattr(obj, name)
        torch = self.torch
        pairs = self.pairs[phase]

        def wrapped(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = inner(*a, **k)
            e1.record()
            pairs.append((e0, e1))
            return out
        self.saved.append((obj, name, inner))
        setattr(obj, name, wrapped)

    def reset(self):
        for v in self.pairs.values():
            v.clear()

    def seconds(self):
        self.torch.cuda.synchronize()
        return {k: sum(a.elapsed_time(b) for a, b in v) / 1e3 for k, v in self.pairs.items()}

    def close(self):
        for obj, name, inner in reversed(self.saved):
            setattr(obj, name, inner)


def chain(L, seed=0):
    from oracle import dmrgx_np as onp
    fields = np.random.default_rng(seed).uniform(-8.0, 8.0, L)
    bits = np.random.default_rng(seed + 1).integers(0, 2, L)
    p0 = []
    for b in bits:
        a = np.zeros((1, 2, 1))
        a[0, b, 0] = 1.0
        p0.append(a)
    return onp.mpo_mbl(fields), p0


def run_config(L, chi, sweeps, max_sites):
    import torch
    import quimb_b200 as qb
    from quimb_b200 import dmrgx
    mpo, p0 = chain(L)
    d = qb.DMRGX([qb.asarray(w) for w in mpo], [qb.asarray(a) for a in p0], chi, seed=0)
    d.expand_bond_dimension(chi, rand_strength=d.opts["bond_expand_rand_strength"])
    D = max(a.shape[0] * a.shape[1] * a.shape[2] for a in d._k)
    inner = dmrgx.DMRGX._update_local_state_1site_dmrgx
    count = {"n": 0}

    per_site = []

    def limited(self, i, direction):
        if max_sites and count["n"] >= max_sites:
            raise _Stop
        count["n"] += 1
        a, s, b = self._k[i].shape
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = inner(self, i, direction)
        torch.cuda.synchronize()
        per_site.append((a * s * b, time.perf_counter() - t0))
        return out
    dmrgx.DMRGX._update_local_state_1site_dmrgx = limited
    try:
        def one(direction, canonize):
            count["n"] = 0
            try:
                d.sweep(direction, canonize=canonize)
            except _Stop:
                pass
            return count["n"]
        one("R", True)                                   # warm-up (and canonical form)
        torch.cuda.synchronize()
        per_site.clear()
        timer = PhaseTimer()
        try:
            direction, sites, t0 = "L", 0, time.perf_counter()
            for _ in range(sweeps):
                sites += one(direction, max_sites > 0)
                direction = "R" if direction == "L" else "L"
            torch.cuda.synchronize()
            secs = time.perf_counter() - t0
            split = timer.seconds()
        finally:
            timer.close()
    finally:
        dmrgx.DMRGX._update_local_state_1site_dmrgx = inner
    whole = sites == L * sweeps
    row = {"L": L, "chi": chi, "D": D, "dtype": "float64", "sweeps": sweeps,
           "sites_timed": sites, "seconds_timed": secs,
           "seconds_per_sweep": secs / sweeps if whole else None,
           "split_seconds_timed": split,
           "energy_after": d.total_energies[-1][-1] if d.total_energies else None}
    row.update(_from_sites(per_site[-count["n"]:], L, D))
    return row


def _from_sites(per_site, L, D):
    """The median bulk-site update time and the sweep it implies from the
    site updates of one sweep (in sweep order): the measured sites as
    measured, the rest at the bulk time except the far edge's ramp, which
    mirrors the measured near edge (the bonds grow as min(chi, 2^i) from
    both ends)."""
    bulk = [t for dd, t in per_site if dd == D]
    if not bulk:
        return {}
    med = float(np.median(bulk))
    ramp = []
    for dd, t in per_site:
        if dd == D:
            break
        ramp.append(t)
    rest = L - len(per_site)
    far = min(len(ramp), rest)
    est = sum(t for _, t in per_site) + sum(ramp[:far]) + (rest - far) * med
    return {"seconds_per_bulk_site": med, "seconds_per_sweep_from_sites": est}


def run_oracle(L, chi, max_sites):
    """The numpy oracle's sweep on the same chain: its first ``max_sites``
    site updates are timed (0: the whole sweep) and the sweep they imply is
    reported as for the device."""
    from oracle import dmrgx_np as onp
    mpo, p0 = chain(L)
    o = onp.DMRGX(mpo, p0, chi)
    onp.expand_bond_dimension(o.k, chi, 1e-9, o.rng)
    D = max(a.shape[0] * a.shape[1] * a.shape[2] for a in o.k)
    inner, per_site = o._update, []

    def timed(i, direction):
        if max_sites and len(per_site) >= max_sites:
            raise _Stop
        a, s, b = o.k[i].shape
        t0 = time.perf_counter()
        out = inner(i, direction)
        per_site.append((a * s * b, time.perf_counter() - t0))
        return out
    o._update = timed
    t0 = time.perf_counter()
    try:
        o.sweep("R")
    except _Stop:
        pass
    secs = time.perf_counter() - t0
    row = {"L": L, "chi": chi, "D": D, "oracle": "numpy", "sites_timed": len(per_site),
           "seconds_timed": secs}
    row.update({"oracle_" + k: v for k, v in _from_sites(per_site, L, D).items()})
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="32x32,64x64", help="LxCHI,...")
    ap.add_argument("--sweeps", type=int, default=2)
    ap.add_argument("--max-sites", default="0",
                    help="per config, comma separated: stop a sweep after N updates (0: all)")
    ap.add_argument("--oracle-L", type=int, default=32)
    ap.add_argument("--oracle-sites", type=int, default=9,
                    help="oracle site updates to time (0: a whole sweep)")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_dmrgx"))
    args = ap.parse_args()
    rows = [card()]
    print(json.dumps(rows[0]), flush=True)
    configs = [tuple(int(v) for v in c.split("x")) for c in args.configs.split(",")]
    limits = [int(v) for v in args.max_sites.split(",")]
    limits += [limits[-1]] * (len(configs) - len(limits))
    for (L, chi), lim in zip(configs, limits):
        row = run_config(L, chi, args.sweeps, lim)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.oracle_L:
        row = run_oracle(args.oracle_L, 32, args.oracle_sites)
        rows.append(row)
        print(json.dumps(row), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_dmrgx.json"), "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
