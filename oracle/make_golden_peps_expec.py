"""Generate tests/golden/peps_expec.{npz,json} by running the UNMODIFIED
reference (quimb @ 97ceeae, numpy backend, through oracle/shims as
oracle/make_golden.py does): PEPS.compute_local_expectation and
PEPS.normalize, quimb/tensor/tn2d/core.py:4223-4415.

Run in the build container only:   python oracle/make_golden_peps_expec.py
Site arrays are stored in the (up, right, down, left, phys) convention of
quimb_b200.boundary.peps_norm_tensors ("<name>__site<i>_<j>").  Every run
stores its options, the reference's value (or its ``return_all`` entries)
and the smallest singular-value gap the oracle recorded.  Exact values come
from the reference's to_dense() and a numpy tensordot.  Before writing, every
run is replayed on oracle/peps_expec_np.py and asserted equal.
"""

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("QUIMB_REFERENCE", "/root/reference")
sys.path.insert(0, os.path.join(HERE, "shims"))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)

import quimb.tensor as qtn  # noqa: E402

from oracle import peps_expec_np as pe  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def site_arrays(p):
    """The reference PEPS's site arrays in (up, right, down, left, phys) order."""
    out = []
    for i in range(p.Lx):
        row = []
        for j in range(p.Ly):
            t = p[i, j]
            want = []
            for di, dj in ((1, 0), (0, 1), (-1, 0), (0, -1)):
                if 0 <= i + di < p.Lx and 0 <= j + dj < p.Ly:
                    (b,) = qtn.bonds(t, p[i + di, j + dj])
                    want.append(b)
            want.append(p.site_ind(i, j))
            row.append(np.transpose(np.asarray(t.data), [t.inds.index(ix) for ix in want]))
        out.append(row)
    return out


def dense_value(p, terms, normalized):
    """Exact sum of <G> from the reference's dense state."""
    psi = np.asarray(p.to_dense()).reshape(-1)
    dims = [p.phys_dim(i, j) for i in range(p.Lx) for j in range(p.Ly)]
    psi_t = psi.reshape(dims)
    tot = 0.0
    for where, G in terms.items():
        tsites = (where,) if pe.is_lone_coo(where) else where
        ax = [i * p.Ly + j for i, j in tsites]
        dg = [dims[a] for a in ax]
        g = np.asarray(G).reshape(dg + dg)
        gp = np.tensordot(g, psi_t, axes=(list(range(len(ax), 2 * len(ax))), ax))
        gp = np.moveaxis(gp, list(range(len(ax))), ax)
        tot = tot + np.vdot(psi, gp.reshape(-1))
    return tot / np.vdot(psi, psi) if normalized else tot


def _key(where):
    return [list(where)] if pe.is_lone_coo(where) else [list(w) for w in where]


def _c(x):
    x = complex(x)
    return [x.real, x.imag]


def main():
    states = {
        "c128_33": (qtn.PEPS.rand(3, 3, bond_dim=2, phys_dim=2, seed=11, dtype="complex128"),
                    dict(field=0.3, nnn=0.5, seed=1)),
        "f64_34": (qtn.PEPS.rand(3, 4, bond_dim=2, phys_dim=2, seed=12, dtype="float64"),
                   dict(field=0.2, long=0.25, seed=2)),
        "c64_43": (qtn.PEPS.rand(4, 3, bond_dim=2, phys_dim=2, seed=13, dtype="complex64"),
                   dict(field=0.4, nnn=0.3, seed=3)),
        "f64_d3_33": (qtn.PEPS.rand(3, 3, bond_dim=2, phys_dim=3, seed=14, dtype="float64"),
                      dict(field=0.5, seed=4)),
        "f32_d3_34": (qtn.PEPS.rand(3, 4, bond_dim=2, phys_dim=3, seed=15, dtype="float32"),
                      dict(field=0.1, long=0.2, seed=5)),
    }
    runs_for = {
        "c128_33": [dict(max_bond=3, cutoff=0.0), dict(max_bond=3, cutoff=0.0, autogroup=False),
                    dict(max_bond=3, cutoff=0.0, normalized=True, return_all=True),
                    dict(max_bond=3, cutoff=0.0, first_contract="y"),
                    dict(max_bond=64, cutoff=0.0, normalized=True),
                    dict(max_bond=64, cutoff=0.0)],
        "f64_34": [dict(max_bond=4, cutoff=0.0), dict(max_bond=4, cutoff=0.0, normalized=True),
                   dict(max_bond=4, cutoff=0.0, first_contract="y", return_all=True),
                   dict(max_bond=4, cutoff=0.0, normalized=True, return_all=True),
                   dict(max_bond=64, cutoff=0.0)],
        "c64_43": [dict(max_bond=3, cutoff=0.0, normalized=True),
                   dict(max_bond=3, cutoff=0.0, first_contract="x", autogroup=False),
                   dict(max_bond=64, cutoff=0.0, normalized=True)],
        "f64_d3_33": [dict(max_bond=4, cutoff=0.0), dict(max_bond=4, cutoff=0.0, normalized=True,
                                                         first_contract="y"),
                      dict(max_bond=64, cutoff=0.0)],
        "f32_d3_34": [dict(max_bond=4, cutoff=0.0, return_all=True, normalized=True),
                      dict(max_bond=64, cutoff=0.0)],
    }
    store, meta = {}, {"states": {}, "runs": []}
    for name, (p, topts) in states.items():
        arrays = site_arrays(p)
        for i, row in enumerate(arrays):
            for j, x in enumerate(row):
                store[f"{name}__site{i}_{j}"] = x
        d = p.phys_dim(0, 0)
        terms = pe.heis_terms(p.Lx, p.Ly, d, **topts)
        terms = {k: np.asarray(v, dtype=p.dtype) for k, v in terms.items()}
        keys = list(terms)
        for k, where in enumerate(keys):
            store[f"{name}__G{k}"] = terms[where]
        exact = dense_value(p, terms, False)
        exact_n = dense_value(p, terms, True)
        assert abs(exact - pe.dense_expectation(arrays, terms)) <= 1e-10 * abs(exact)
        # PEPS.normalize at a truncating and an exact boundary
        norms = []
        for mb in (3, 64):
            q = p.normalize(max_bond=mb, cutoff=0.0)
            qa = site_arrays(q)
            oa, nfact = pe.normalize(arrays, max_bond=mb, cutoff=0.0)
            tol = 2e-5 if p.dtype in ("complex64", "float32") else 1e-10
            for r1, r2 in zip(qa, oa):
                for a, b in zip(r1, r2):
                    assert np.allclose(a, b, rtol=tol, atol=tol * np.abs(a).max()), name
            norms.append({"max_bond": mb, "nfact": _c(nfact)})
            for i, row in enumerate(qa):
                for j, x in enumerate(row):
                    store[f"{name}__norm{mb}_site{i}_{j}"] = x
        meta["states"][name] = {
            "Lx": p.Lx, "Ly": p.Ly, "d": int(d), "dtype": p.dtype,
            "keys": [_key(w) for w in keys], "exact": _c(exact), "exact_normalized": _c(exact_n),
            "normalize": norms}
        for kw in runs_for[name]:
            ref = p.compute_local_expectation(terms, **kw)
            got, trace = pe.compute_local_expectation(arrays, terms, **kw)
            tol = 2e-5 if p.dtype in ("complex64", "float32") else 1e-10
            rec = {"state": name, "kw": kw, "min_gap": float(pe.min_gap(trace))}
            if kw.get("return_all"):
                vals = []
                for where in keys:
                    e, n = ref[where]
                    ge, gn = got[where]
                    scale = max(1.0, abs(e))
                    assert abs(ge - e) <= tol * scale, (name, kw, where, ge, e)
                    if n is not None:
                        assert abs(gn - n) <= tol * max(1.0, abs(n)), (name, kw, where)
                    vals.append([_c(e), None if n is None else _c(n)])
                rec["values"] = vals
            else:
                assert abs(got - ref) <= tol * max(1.0, abs(ref)), (name, kw, got, ref)
                rec["value"] = _c(ref)
            if kw["max_bond"] == 64:
                want = exact_n if kw.get("normalized") else exact
                assert abs(complex(ref) - want) <= 1e-4 * abs(want) if tol > 1e-9 else \
                    abs(complex(ref) - want) <= 1e-10 * abs(want), (name, ref, want)
            meta["runs"].append(rec)
            print(name, kw, rec.get("value"), rec["min_gap"])
    np.savez_compressed(os.path.join(OUT, "peps_expec.npz"), **store)
    with open(os.path.join(OUT, "peps_expec.json"), "w") as fh:
        json.dump(meta, fh, indent=1)


if __name__ == "__main__":
    main()
