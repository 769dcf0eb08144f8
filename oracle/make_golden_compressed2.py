"""Generate tests/golden/compressed2.{npz,json} by running the UNMODIFIED
reference (quimb @ 97ceeae, numpy backend, through oracle/shims as
oracle/make_golden.py does): ``_contract_compressed_tid_sequence``
(compress_mode='basic', tree_gauge_distance=0) where the rescaling of the
tensors matters:

  * ``equalize_norms=True`` with a nonzero cutoff in the scale-dependent
    modes 'abs' and 'sum2', and in 'rel': every tensor is divided by its
    Frobenius norm after each contraction and compression, so that norm sets
    what an absolute cutoff keeps;
  * ``strip_exponent=True`` on networks with open output indices: the
    mantissa has unit Frobenius norm.

Run in the build container only:   python oracle/make_golden_compressed2.py
Before writing, every run is replayed on oracle/compressed_np.py and asserted
equal, and every truncation is asserted to be decided at a relative gap of at
least MIN_GAP, so that rounding cannot change a kept rank.
"""

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden import OUT, qtn  # noqa: E402
from oracle import compressed_np as cnp  # noqa: E402

MIN_GAP = 1e-6

RUNS = [
    dict(max_bond=8, cutoff=0.05, cutoff_mode="abs", equalize_norms=True),
    dict(max_bond=8, cutoff=0.2, cutoff_mode="abs", equalize_norms=True),
    dict(max_bond=8, cutoff=2e-3, cutoff_mode="sum2", equalize_norms=True),
    dict(max_bond=8, cutoff=0.02, cutoff_mode="rel", equalize_norms=True),
    dict(max_bond=4, cutoff=0.0, strip_exponent=True),
    dict(max_bond=6, cutoff=0.05, cutoff_mode="abs", strip_exponent=True),
    dict(max_bond=6, cutoff=0.0, strip_exponent=True, equalize_norms=False),
    dict(max_bond=5, cutoff=0.0, equalize_norms=True, compress_late=False),
]


def _kw(run):
    """Split the run into the sequence function's options and compress_opts."""
    kw = {k: v for k, v in run.items() if k != "cutoff_mode"}
    if "cutoff_mode" in run:
        kw["compress_opts"] = {"cutoff_mode": run["cutoff_mode"]}
    return kw


def main():
    store, meta = {}, {}
    nets = {
        "peps33_open": qtn.PEPS.rand(3, 3, bond_dim=3, phys_dim=2, seed=21),
        "peps34_open_c": qtn.PEPS.rand(3, 4, bond_dim=3, phys_dim=2, seed=22,
                                       dtype="complex128"),
        "flat55": qtn.TN2D_rand(5, 5, D=3, seed=23),
        "reg12": qtn.TN_rand_reg(12, 3, D=3, seed=24),
    }
    for name, tn in nets.items():
        tids = list(tn.tensor_map)
        arrays = [np.asarray(tn.tensor_map[t].data) for t in tids]
        inputs = [list(map(str, tn.tensor_map[t].inds)) for t in tids]
        output = list(map(str, tn.outer_inds()))
        seq = cnp.greedy_sequence(arrays, inputs, output)
        for k, a in enumerate(arrays):
            store[f"{name}__t{k}"] = a
        exact = tn.contract(all, optimize="auto-hq", output_inds=tn.outer_inds())
        store[f"{name}__exact"] = np.asarray(exact.data if hasattr(exact, "data") else exact)
        runs = []
        for run in RUNS:
            res = tn.copy()._contract_compressed_tid_sequence(
                [(tids[a], tids[b]) for a, b in seq], output_inds=tn.outer_inds(),
                tree_gauge_distance=0, compress_mode="basic", **_kw(run))
            if run.get("strip_exponent"):
                res, expo = res
            else:
                expo = None
            if hasattr(res, "inds"):
                res = res.transpose(*tn.outer_inds()).data
            val = np.asarray(res)
            key = f"{name}__run{len(runs)}"
            store[key] = val
            # replay on the oracle: same value, every cut far from rounding
            got, info = cnp.contract_compressed(arrays, inputs, output, seq, **_kw(run))
            if expo is not None:
                got, gexp = got
                assert abs(gexp - float(expo)) < 1e-10, (name, run, gexp, expo)
            err = np.abs(got - val).max() / np.abs(val).max()
            assert err < 1e-11, (name, run, err)
            gap = min([r["gap"] for r in info["trace"]] + [np.inf])
            assert gap >= MIN_GAP, (name, run, gap)
            runs.append({"kw": run, "key": key,
                         "exponent": None if expo is None else float(expo),
                         "n_compress": info["n_compress"],
                         "max_bond_seen": info["max_bond_seen"],
                         "ranks": [r["rank"] for r in info["trace"]],
                         "min_gap": float(gap)})
            print(name, run, "n_compress", info["n_compress"], "min gap", f"{gap:.2e}")
        meta[name] = {"inputs": inputs, "output": output, "seq": [list(s) for s in seq],
                      "runs": runs, "dtype": str(tn.dtype)}
    np.savez_compressed(os.path.join(OUT, "compressed2.npz"), **store)
    with open(os.path.join(OUT, "compressed2.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
