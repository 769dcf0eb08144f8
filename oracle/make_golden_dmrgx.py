"""Generate tests/golden/dmrgx.{npz,json} by running the UNMODIFIED reference
(quimb @ 97ceeae, numpy backend, through oracle/shims as oracle/make_golden.py
does): ``DMRGX`` (quimb/tensor/tn1d/dmrg.py:1185-1466) on ``MPO_ham_mbl``
chains.

Run in the build container only:   python oracle/make_golden_dmrgx.py

Pinned cases start from a full-rank random MPS (every bond min(chi, 2^i,
2^(L-i)), no zero padding) and drive ``sweep_right`` / ``sweep_left``
directly: no bond expansion and no QR completion of null directions is
involved, so the sweep is determined by the state.  They store every step's
local energy, every sweep's total energies and the final dense state.  Each
selection decision is asserted to be made far from rounding: the overlaps'
distance to the candidate threshold and the gap of the winning overlap or
variance are at least ``MIN_MARGIN`` relative.

Property cases mirror the reference's own tests (test_dmrg.py:339-385) plus
``overlap_thresh=1``, the shift-invert branch (forced by
``local_eig_partial_cutoff = 2**7``) and complex128; their expansion noise
is drawn by the reference (seeded with ``qu.seed_rand``), so only the final
energy, variance and dense state are stored.

Before writing, every case is replayed on oracle/dmrgx_np.py and asserted
equal: pinned cases step by step, property cases by final energy.
"""

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden_sample import OUT, _lpr, qtn  # noqa: E402
from oracle.make_golden_mpo_compress import _lrud  # noqa: E402
from oracle import dmrgx_np as onp  # noqa: E402
import quimb as qu  # noqa: E402

MIN_MARGIN = 1e-6
REPLAY_TOL = 1e-12


def _full_rank_mps(L, chi, dtype, seed):
    rng = np.random.default_rng(seed)
    bonds = [1] + [min(chi, 2 ** i, 2 ** (L - i)) for i in range(1, L)] + [1]
    out = []
    for i in range(L):
        shape = (bonds[i], 2, bonds[i + 1])
        x = rng.standard_normal(shape)
        if np.dtype(dtype).kind == "c":
            x = x + 1j * rng.standard_normal(shape)
        out.append((x / np.sqrt(bonds[i] * 2)).astype(dtype))
    n2 = onp.mps_dense(out)
    out[0] = out[0] / np.linalg.norm(n2)
    return out


def _ref_mps(sites):
    """A reference MatrixProductState from (l, p, r) arrays."""
    L = len(sites)
    arrs = []
    for i, A in enumerate(sites):
        x = np.transpose(A, (0, 2, 1))            # (l, r, p)
        if i == 0:
            x = x[0]
        elif i == L - 1:
            x = x[:, 0]
        arrs.append(x)
    return qtn.MatrixProductState(arrs, shape="lrp")


def _store(data, name, mpo, p0, d):
    for i, w in enumerate(mpo):
        data[f"{name}__mpo{i}"] = w
    for i, a in enumerate(p0):
        data[f"{name}__p0_{i}"] = a
    data[f"{name}__state"] = onp.mps_dense(_lpr(d._k))


PINNED = [
    # name, L, chi, dh, mpo seed, mps seed, dtype, opts, sweeps
    ("pin_real", 10, 8, 4.0, 3, 11, "float64", {}, [("R", True), ("L", False), ("L", True)]),
    ("pin_wide", 12, 16, 6.0, 5, 21, "float64", {}, [("R", True), ("R", True)]),
    ("pin_complex", 8, 8, 4.0, 7, 31, "complex128", {}, [("L", True), ("R", False)]),
    ("pin_thresh1", 10, 8, 4.0, 9, 41, "float64", {"overlap_thresh": 1},
     [("R", True), ("L", False)]),
]

PROPERTY = [
    # name, L, chi, dh, mpo seed, p0, dtype, opts, solve kwargs / sweeps
    ("explicit", 8, 16, 4.0, 42, "rand", "float64", {},
     [("R", True), ("L", False), ("R", False), ("R", True)]),
    ("bigger", 14, 16, 8.0, 42, "00110111000101", "float64", {},
     {"tol": 1e-5, "sweep_sequence": "R"}),
    ("thresh1", 10, 16, 8.0, 13, "0110100110", "float64", {"overlap_thresh": 1},
     {"tol": 1e-5, "sweep_sequence": "R"}),
    ("partial", 10, 16, 8.0, 20, "1001011010", "float64", {"local_eig_partial_cutoff": 2**7},
     {"tol": 1e-5, "sweep_sequence": "R"}),
    ("complex", 10, 16, 8.0, 19, "0011010110", "complex128", {},
     {"tol": 1e-5, "sweep_sequence": "R"}),
]


def _replay_pinned(mpo, p0, opts, sweeps):
    o = onp.DMRGX(mpo, p0, p0[len(p0) // 2].shape[0])
    o.opts.update(opts)
    for direction, canonize in sweeps:
        o.sweep(direction, canonize=canonize)
    return o


def main():
    data, cases = {}, []
    for name, L, chi, dh, mseed, pseed, dtype, opts, sweeps in PINNED:
        H = qtn.MPO_ham_mbl(L, dh=dh, seed=mseed)
        mpo = _lrud(H)
        fields = onp.mpo_fields(mpo)
        assert onp.mpo_dist2(mpo, onp.mpo_mbl(fields)) < 1e-20
        # a start state whose sweeps are ill-conditioned (two independent
        # numpy implementations drift apart by more than REPLAY_TOL, or a
        # decision lies within MIN_MARGIN of a tie) is replaced by the next seed
        for seed in range(pseed, pseed + 20):
            p0 = _full_rank_mps(L, chi, dtype, seed)
            d = qtn.DMRGX(H, _ref_mps(p0), chi)
            d.opts.update(opts)
            en2_p0 = float(np.real(d.TN_energy2 ^ ...))
            for direction, canonize in sweeps:
                (d.sweep_right if direction == "R" else d.sweep_left)(canonize=canonize)
            loc = np.array([[float(np.real(e)) for e in s] for s in d.local_energies])
            tot = np.array([[float(np.real(e)) for e in s] for s in d.total_energies])
            o = _replay_pinned(mpo, p0, opts, sweeps)
            psi = onp.mps_dense(_lpr(d._k))
            fid = abs(np.vdot(onp.mps_dense(o.k), psi)) ** 2
            thr = min(m for _, _, m, _ in o.decisions)
            gap = min(g for _, _, _, g in o.decisions)
            ncand = max(n for _, n, _, _ in o.decisions)
            drift = max(np.max(np.abs(np.array(o.local_energies) - loc)),
                        np.max(np.abs(np.array(o.total_energies) - tot)))
            print(f"{name} seed {seed}: drift {drift:.1e} fid-1 {fid - 1:.1e} "
                  f"thr margin {thr:.2e} gap {gap:.2e} max cand {ncand}")
            if (drift <= REPLAY_TOL and fid > 1 - 1e-11 and thr >= MIN_MARGIN
                    and gap >= MIN_MARGIN):
                break
        else:
            raise AssertionError(f"{name}: no well-conditioned start state")
        _store(data, name, mpo, p0, d)
        data[f"{name}__local"] = loc
        data[f"{name}__total"] = tot
        cases.append({"name": name, "kind": "pinned", "L": L, "chi": chi, "dh": dh,
                      "dtype": dtype, "opts": opts, "sweeps": sweeps, "fields": fields,
                      "en2_p0": en2_p0, "energy0": float(np.real(d.energies[0])),
                      "min_threshold_margin": thr, "min_winner_gap": gap,
                      "max_candidates": ncand, "mps_seed": seed})

    for name, L, chi, dh, mseed, p0spec, dtype, opts, run in PROPERTY:
        H = qtn.MPO_ham_mbl(L, dh=dh, seed=mseed)
        mpo = _lrud(H)
        fields = onp.mpo_fields(mpo)
        assert onp.mpo_dist2(mpo, onp.mpo_mbl(fields)) < 1e-20
        qu.seed_rand(1000 + mseed)
        if p0spec == "rand":
            pr = qtn.MPS_rand_state(L, 2, dtype=dtype)
            pr.expand_bond_dimension(chi, inplace=True)
        else:
            pr = qtn.MPS_computational_state(p0spec, dtype=dtype)
        p0 = [np.ascontiguousarray(a) for a in _lpr(pr)]
        d = qtn.DMRGX(H, pr, chi)
        d.opts.update(opts)
        if isinstance(run, list):
            for direction, canonize in run:
                (d.sweep_right if direction == "R" else d.sweep_left)(canonize=canonize)
            energy = float(np.real(d.total_energies[-1][-1]))
            k = d._k
            variance = float(np.real((d.TN_energy2 ^ ...))) - energy ** 2
        else:
            assert d.solve(**run), name
            energy, variance = float(np.real(d.energy)), float(np.real(d.variance))
        psi = onp.mps_dense(_lpr(d._k))
        # replay on the oracle (its own expansion noise)
        o = onp.DMRGX(mpo, p0, chi, seed=mseed)
        o.opts.update(opts)
        if isinstance(run, list):
            for direction, canonize in run:
                o.sweep(direction, canonize=canonize)
            oe = o.total_energies[-1][-1]
        else:
            assert o.solve(**run), name
            oe = o.energy
        assert abs(oe - energy) < 1e-8, (name, oe, energy)
        fid = abs(np.vdot(onp.mps_dense(o.k), psi)) ** 2 / np.vdot(psi, psi).real
        assert fid > 1 - 1e-8, (name, fid)
        _store(data, name, mpo, p0, d)
        cases.append({"name": name, "kind": "property", "L": L, "chi": chi, "dh": dh,
                      "dtype": dtype, "opts": opts, "run": run, "fields": fields,
                      "energy": energy, "variance": variance,
                      "sweeps_done": len(d.local_energies),
                      "tol": run["tol"] if isinstance(run, dict) else 1e-10})
        print(f"{name}: E={energy:.12f} var={variance:.2e} sweeps={len(d.local_energies)}")

    np.savez_compressed(os.path.join(OUT, "dmrgx.npz"), **data)
    meta = {"source": "quimb @ 97ceeae tn1d/dmrg.py DMRGX via oracle/shims",
            "min_margin": MIN_MARGIN, "cases": cases}
    with open(os.path.join(OUT, "dmrgx.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
