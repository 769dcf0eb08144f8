"""Generate tests/golden/successive.{npz,json} by running the UNMODIFIED
reference (numpy backend, through oracle/shims as oracle/make_golden.py
does): MatrixProductState.gate_with_mpo with the successive-compression
methods 'src', 'src-oversample', 'srcmps', 'srcmps-oversample', 'sdc' and
'sdc-oversample' (tn1d/compress.py:1115-2339).

Run in the build container only:   python oracle/make_golden_successive.py

The autoray shim has no ``random.array`` for numpy; the reference's SRC
draws its noise through it (compress.py:1283).  This script registers
``quimb_b200``'s host draw rule (``quimb_b200._random_host``, the rule
``quimb_b200.random.array`` uploads) as the shim's ``random.array``, and
numpy's own ``default_rng`` as ``random.default_rng``, so the reference and
this project see the same noise from the same seed.  The fixtures therefore
pin the algorithm given the noise, not the noise itself.  'srcmps' cases
pass their sampling MPS explicitly (stored with the inputs).

Each case stores bond sizes, per-bond singular values and the dense output,
all independent of the gauge.  Before writing, every case is replayed on
oracle/successive_np.py and asserted equal, and every truncation cut (SDC
splits, the direct sweeps of the '-oversample' methods) is asserted to lie
far from rounding noise.
"""

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden_sample import OUT, _lpr, qtn  # noqa: E402
from oracle.make_golden_mpo_compress import MIXED, _lrud, _mixed_dims, _rand_mpo  # noqa: E402
from oracle import successive_np as onp  # noqa: E402

import autoray  # noqa: E402  (the shim, first on sys.path)
from quimb_b200 import _random_host  # noqa: E402


def _shim_random_array(shape, dist="normal", dtype="float64", rng=None, seed=None, **kw):
    return _random_host(shape, dist, dtype, rng=rng, seed=seed)


autoray.register_function("numpy", "random.array", _shim_random_array)
autoray.register_function("numpy", "random.default_rng", np.random.default_rng)


def check_cut(s, kept, cutoff, cutoff_mode):
    """A truncation that discards more than rounding noise is decided by a
    singular-value gap, and a cutoff decision by a tail weight, both far
    from the noise of either implementation."""
    if kept == s.size or s[kept] <= 1e-13 * s[0]:
        return 0.0
    gap = (s[kept - 1] - s[kept]) / s[0]
    assert gap > 1e-6, (kept, gap)
    if cutoff and cutoff > 0:
        assert cutoff_mode == "rsum2"
        tail = np.sum(s[kept:] ** 2) / np.sum(s ** 2)
        prev = np.sum(s[kept - 1:] ** 2) / np.sum(s ** 2)
        assert tail < cutoff or abs(tail - cutoff) > 1e-3 * cutoff, (tail, cutoff)
        assert abs(prev - cutoff) > 1e-3 * cutoff, (prev, cutoff)
    return gap


def _sampling_mps(dims, bond, dtype, seed):
    """A random open-boundary (l, p, r) sampling MPS."""
    rng = np.random.default_rng(seed)
    L = len(dims)
    out = []
    for i, d in enumerate(dims):
        shape = (1 if i == 0 else bond, d, 1 if i == L - 1 else bond)
        x = rng.standard_normal(shape)
        if np.dtype(dtype).kind == "c":
            x = x + 1j * rng.standard_normal(shape)
        out.append((x / np.sqrt(shape[0] * d)).astype(dtype))
    return out


def _to_mps(F):
    arrays = [F[0][0]] + list(F[1:-1]) + [F[-1][:, :, 0]] if len(F) > 1 else [F[0][0, :, 0]]
    return qtn.MatrixProductState(arrays, shape="lpr")


def cases():
    states = {
        "real": qtn.MPS_rand_state(8, 6, seed=3, dtype="float64"),
        "cplx": qtn.MPS_rand_state(10, 8, seed=5, dtype="complex128"),
        "mixed": _mixed_dims(MIXED, 31),
        "two": qtn.MPS_rand_state(2, 2, seed=9, dtype="complex128"),
    }
    mpos = {
        "heis": qtn.MPO_ham_heis(8),
        "rand3": _rand_mpo(10, 3, 2, 21),
        "rand5": _rand_mpo(8, 5, 2, 22),
        "rand_mixed": _rand_mpo(7, 3, MIXED, 25),
        "rand2": _rand_mpo(2, 3, 2, 26),
    }
    store, meta = {}, {"states": {}, "mpos": {}, "fits": {}}
    for name, p in states.items():
        for i, x in enumerate(_lpr(p)):
            store[f"{name}__site{i}"] = np.ascontiguousarray(x)
        meta["states"][name] = {"L": p.L}
    for name, m in mpos.items():
        for i, x in enumerate(_lrud(m)):
            store[f"{name}__mpo{i}"] = x
        meta["mpos"][name] = {"L": m.L}
    out_dims = {"real": [2] * 8, "cplx": [2] * 10, "mixed": MIXED, "two": [2, 2]}
    fits = {
        "fit_real": ("real", 7, "float64", 41),
        "fit_cplx": ("cplx", 9, "complex128", 42),
        "fit_mixed": ("mixed", 6, "complex128", 43),
        "fit_two": ("two", 3, "complex128", 44),
        "fit_real_wide": ("real", 40, "float64", 45),
    }
    for name, (st, bond, dt, seed) in fits.items():
        F = _sampling_mps(out_dims[st], bond, dt, seed)
        for i, x in enumerate(F):
            store[f"{name}__fit{i}"] = x
        meta["fits"][name] = {"L": len(F)}

    runs = []
    for method in ("src", "src-oversample", "sdc", "sdc-oversample", "srcmps",
                   "srcmps-oversample"):
        srcmps = method.startswith("srcmps")
        runs += [
            dict(state="real", mpo="heis", method=method, max_bond=6, seed=1, fit="fit_real"),
            dict(state="real", mpo="heis", method=method, max_bond=40, seed=2,
                 fit="fit_real_wide"),
            dict(state="cplx", mpo="rand3", method=method, max_bond=10, seed=3, fit="fit_cplx"),
            dict(state="cplx", mpo="rand3", method=method, max_bond=10, seed=4, transpose=True,
                 sweep_reverse=True, fit="fit_cplx"),
            dict(state="real", mpo="rand5", method=method, max_bond=9, seed=5, normalize=True,
                 fit="fit_real"),
            dict(state="mixed", mpo="rand_mixed", method=method, max_bond=7, seed=6,
                 fit="fit_mixed"),
            dict(state="two", mpo="rand2", method=method, max_bond=3, seed=7, fit="fit_two"),
        ]
        if not srcmps and method.startswith("src"):
            runs += [
                dict(state="cplx", mpo="rand3", method=method, max_bond=8, seed=8,
                     noise_dist="uniform"),
                dict(state="cplx", mpo="rand3", method=method, max_bond=8, seed=10,
                     seed_generator=True),
            ]
    runs += [
        # +-1 noise repeats sample directions; this case keeps every sketch
        # well posed (checked below), most small ones do not
        dict(state="real", mpo="rand5", method="src", max_bond=3, seed=12,
             noise_dist="rademacher"),
        dict(state="cplx", mpo="rand3", method="src-oversample", max_bond=8,
             max_bond_oversample=1.5, seed=11),
        dict(state="real", mpo="rand5", method="sdc-oversample", max_bond=7,
             max_bond_oversample=12),
        dict(state="real", mpo="heis", method="sdc", max_bond=None, cutoff=1e-3),
    ]
    out_cases = []
    min_gap = np.inf
    for run in runs:
        p, m = states[run["state"]], mpos[run["mpo"]]
        method = run["method"]
        kw = {k: v for k, v in run.items() if k not in ("state", "mpo", "fit", "seed_generator")}
        if not method.startswith("srcmps"):
            kw.pop("fit", None)
        if method.startswith("sdc"):
            kw.pop("seed", None)
        ref_kw = dict(kw)
        base = method.split("-")[0]
        over = method.endswith("-oversample")
        if base in ("src", "srcmps") and not over:
            ref_kw.setdefault("cutoff", 0.0)
        F = None
        if base == "srcmps":
            F = [store[f"{run['fit']}__fit{i}"] for i in range(meta["fits"][run["fit"]]["L"])]
            ref_kw["tn_fit"] = _to_mps(F)
            ref_kw.pop("seed", None)
            kw.pop("seed", None)
        if run.get("seed_generator"):
            ref_kw["seed"] = np.random.default_rng(run["seed"])
        q = p.gate_with_mpo(m, **ref_kw)
        lpr = _lpr(q)
        bonds = [int(x.shape[2]) for x in lpr[:-1]]
        svals = [np.asarray(q.copy().singular_values(i)) for i in range(1, q.L)]
        vec = np.asarray(q.to_dense()).reshape(-1)

        okw = dict(kw)
        if run.get("seed_generator"):
            okw["seed"] = np.random.default_rng(run["seed"])
        cuts = []
        got = onp.gate_with_mpo_successive(_lpr(p), _lrud(m), tn_fit=F, cuts=cuts, **okw)
        if run.get("seed_generator"):
            okw["seed"] = np.random.default_rng(run["seed"])
        assert [x.shape[2] for x in got[:-1]] == bonds, (run, bonds)
        scale = np.max(np.abs(vec))
        err = np.max(np.abs(onp.dense(got) - vec))
        assert err <= 1e-10 * scale, (run, err / scale)
        for s_o, s_r in zip(onp.schmidt_values(got), svals):
            assert np.allclose(s_o, s_r, rtol=0, atol=1e-10 * s_r[0]), run
        # a sketch whose QR leaves Q to rounding would pin LAPACK, not SRC
        jit = onp.gate_with_mpo_successive(_lpr(p), _lrud(m), tn_fit=F,
                                           sketches=np.random.default_rng(0), **okw)
        assert np.max(np.abs(onp.dense(jit) - vec)) <= 1e-8 * scale, ("ill-posed", run)
        inner_cut = kw.get("cutoff_oversample", 0.0) if over else kw.get("cutoff", 1e-10)
        for j, (s, kept) in enumerate(cuts):
            # the sdc splits come first, then the direct sweep's
            cut = inner_cut if (base == "sdc" and j < q.L - 1) else kw.get("cutoff", 1e-10)
            g = check_cut(s, kept, cut, kw.get("cutoff_mode", "rsum2"))
            if g:
                min_gap = min(min_gap, g)
        k = len(out_cases)
        store[f"case{k}__vec"] = vec
        for i, s in enumerate(svals):
            store[f"case{k}__S{i}"] = s
        out_cases.append(dict(run, bonds=bonds))
    meta["cases"] = out_cases
    meta["min_cut_gap"] = float(min_gap)
    np.savez_compressed(os.path.join(OUT, "successive.npz"), **store)
    json.dump(meta, open(os.path.join(OUT, "successive.json"), "w"), indent=1)
    print(f"{len(out_cases)} cases, smallest relative gap at a truncating cut {min_gap:.3g}")


if __name__ == "__main__":
    cases()
    print("golden fixtures written to", OUT)
    for f in ("successive.npz", "successive.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))
