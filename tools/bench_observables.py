"""MPS observables benchmark (``quimb_b200.observables``).

  python tools/bench_observables.py [--L 100] [--chis 256,1024]
                                    [--dtypes float64,complex128] [--reps 20]

For each workload (random MPS, d = 2, bonds min(chi, 2^i, 2^(L-i))) it prints
one JSON line with, after a warm-up of every timed shape:
  expec_one_site_s   compute_local_expectation of the L one-site Z terms,
                     return_all=True, from a right-canonical state (CUDA
                     events around the call, synchronised);
  expec_nn_s         the same for the L - 1 nearest-neighbour ZZ terms;
  entropy_profile_s  mps_entropy at every bond, one shared info;
  rdm_share_*        share of each of those calls spent in qb_rdm_reduce
                     (CUDA events around every reduction);
and, per D in (2, 4, 8), qb_rdm_reduce against contract_pair on the same
rho operands theta (chi, D, chi), alternated in one run: their times, the
kernel's bytes/s (theta read once) and its share of 3.35 TB/s.
The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

HBM_BPS = 3.35e12


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


class RdmTimer:
    """Wraps observables.rdm_reduce with CUDA events around every call."""

    def __init__(self, obs):
        self.obs, self.orig, self.events = obs, obs.rdm_reduce, []

    def __enter__(self):
        import torch

        def timed(U, V):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = self.orig(U, V)
            b.record()
            self.events.append((a, b))
            return out
        self.obs.rdm_reduce = timed
        return self

    def __exit__(self, *exc):
        self.obs.rdm_reduce = self.orig

    def seconds(self):
        return sum(a.elapsed_time(b) for a, b in self.events) / 1e3


def timed_call(fn, reps=1):
    import torch
    from quimb_b200 import observables as obs
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with RdmTimer(obs) as t:
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        total = a.elapsed_time(b) / 1e3 / reps
        share = t.seconds() / reps / total
    return total, share


def workload(L, chi, dtype, reps):
    import quimb_b200 as qb
    from quimb_b200 import tebd
    Z = np.diag([1.0, -1.0])
    one = {(i,): Z for i in range(L)}
    nn = {(i, i + 1): np.kron(Z, Z) for i in range(L - 1)}
    base = rand_sites(L, chi, 2, dtype, seed=chi)
    tebd.right_canonize(base)
    row = {"L": L, "chi": chi, "dtype": dtype}

    def expec(terms):
        return lambda: qb.mps_compute_local_expectation(base, terms, return_all=True,
                                                        info={"cur_orthog": 0})

    def profile():
        psi, info = list(base), {"cur_orthog": 0}
        for i in range(1, L):
            qb.mps_entropy(psi, i, info=info)

    for key, fn in (("expec_one_site", expec(one)), ("expec_nn", expec(nn)),
                    ("entropy_profile", profile)):
        fn()                                              # warm-up
        t, share = timed_call(fn)
        row[key + "_s"] = t
        row["rdm_share_" + key] = share
    row["kernel_vs_contract_pair"] = kernel_vs_engine(chi, dtype, reps)
    return row


def kernel_vs_engine(chi, dtype, reps):
    import torch
    from quimb_b200 import observables as obs
    from quimb_b200.contract import contract_pair
    tdt = {"float64": torch.float64, "complex128": torch.complex128}[dtype]
    out = []
    for D in (2, 4, 8):
        theta = torch.randn((chi, D, chi), dtype=tdt, device="cuda")

        def kern():
            obs.rdm_reduce(theta, theta)

        def engine():
            contract_pair(theta, [0, 1, 2], theta, [0, 3, 2], [1, 3], conj_b=True)

        a = obs.rdm_reduce(theta, theta)
        b = contract_pair(theta, [0, 1, 2], theta, [0, 3, 2], [1, 3], conj_b=True)
        err = float((a - b).abs().max() / b.abs().max())
        tk = te = 0.0
        for _ in range(5):                               # alternate the two routes
            tk += timed_call(lambda: [kern() for _ in range(reps)])[0] / reps
            te += timed_call(lambda: [engine() for _ in range(reps)])[0] / reps
        tk, te = tk / 5, te / 5
        nbytes = theta.numel() * theta.element_size()
        out.append({"D": D, "rdm_reduce_s": tk, "contract_pair_s": te,
                    "speedup": te / tk, "rdm_bytes_per_s": nbytes / tk,
                    "rdm_share_of_3.35TBps": nbytes / tk / HBM_BPS, "rel_diff": err})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--chis", default="256,1024")
    ap.add_argument("--dtypes", default="float64,complex128")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_observables: needs a CUDA device")
    print(json.dumps(card()), flush=True)
    for dtype in args.dtypes.split(","):
        for chi in map(int, args.chis.split(",")):
            print(json.dumps(workload(args.L, chi, dtype, args.reps)), flush=True)


if __name__ == "__main__":
    main()
