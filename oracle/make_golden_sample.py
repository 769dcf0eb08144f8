"""Generate tests/golden/sample.{npz,json} by running the UNMODIFIED reference
(quimb @ 97ceeae, numpy backend) -- MatrixProductState.sample and
sample_configuration, quimb/tensor/tn1d/core.py:3871-3990 -- the same way
oracle/make_golden.py generates the other fixtures (its shims route the
reference's third-party calls; all arithmetic is the reference's own).

Run in the build container only:   python oracle/make_golden_sample.py
Each case stores the site arrays in the reference's layout with a layout
string ('lrp', 'rp', ...; tests convert them with quimb_b200.mps.site_lpr),
the configurations and probabilities the reference yielded, and the margin
of oracle/sample_np.py on the same draws (its configurations are asserted
equal to the reference's here).
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

from oracle import sample_np  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def _layouts(p):
    out = []
    for i in range(p.L):
        t = p[i]
        lay = ""
        for ix in t.inds:
            if ix == p.site_ind(i):
                lay += "p"
            elif i > 0 and ix in qtn.bonds(p[i - 1], t):
                lay += "l"
            else:
                lay += "r"
        out.append(lay)
    return out


def _lpr(p):
    """(l, p, r) numpy copies of the reference's site arrays."""
    out = []
    for i, lay in enumerate(_layouts(p)):
        x = np.asarray(p[i].data)
        for c in "lpr":
            if c not in lay:
                x = x[..., None]
                lay += c
        out.append(np.transpose(x, [lay.index(c) for c in "lpr"]))
    return out


def _ragged_qutrit(seed):
    rng = np.random.default_rng(seed)
    bonds = [1, 3, 7, 4, 9, 2, 5, 1]
    arrays = []
    for i in range(len(bonds) - 1):
        shape = (bonds[i], bonds[i + 1], 3)          # 'lrp'
        x = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
        if i == 0:
            x = x[0]
        elif i == len(bonds) - 2:
            x = x[:, 0]
        arrays.append(x)
    return qtn.MatrixProductState(arrays, shape="lrp")


def sample_cases():
    store, meta = {}, {}
    states = {
        "real": qtn.MPS_rand_state(10, 8, seed=3, dtype="float64"),
        "cplx": qtn.MPS_rand_state(12, 16, seed=5, dtype="complex128"),
        "qutrit_ragged": _ragged_qutrit(9),
        "product": qtn.MPS_computational_state("0110100111"),
    }
    runs = [
        # (state, kind, C, seed): kind 'sample' / 'configuration' / 'generator'
        # ('generator': two consecutive sample() calls on one Generator)
        ("real", "sample", 200, 11),
        ("cplx", "sample", 200, 12),
        ("qutrit_ragged", "sample", 200, 13),
        ("product", "sample", 20, 14),
        ("cplx", "generator", (60, 40), 15),
        ("real", "configuration", 1, 16),
        ("qutrit_ragged", "configuration", 1, 17),
    ]
    for name, p in states.items():
        layouts = _layouts(p)
        for i in range(p.L):
            store[f"{name}__site{i}"] = np.asarray(p[i].data)
        meta[name] = {"L": p.L, "layouts": layouts, "dtype": str(p.dtype),
                      "bonds": [int(p.bond_size(i, i + 1)) for i in range(p.L - 1)]}
    cases = []
    for name, kind, C, seed in runs:
        p = states[name]
        if kind == "configuration":
            cfg, om = p.sample_configuration(seed=seed)
            parts = [([list(map(int, cfg))], [float(om)])]
        elif kind == "sample":
            got = list(p.sample(C, seed=seed))
            parts = [([list(map(int, c)) for c, _ in got], [float(o) for _, o in got])]
        else:
            rng = np.random.default_rng(seed)
            parts = []
            for c in C:
                got = list(p.sample(c, seed=rng))
                parts.append(([list(map(int, x)) for x, _ in got], [float(o) for _, o in got]))
        # the oracle on the same draws: equal configurations, and its margin
        rng = np.random.default_rng(seed)
        psi = sample_np.prepare(_lpr(p))
        margins = []
        for k, (cfgs, oms) in enumerate(parts):
            u = rng.random((len(cfgs), p.L))
            oc, oo, margin = sample_np.sample_uniforms(psi, u)
            assert np.array_equal(oc, np.array(cfgs)), (name, kind, k)
            assert np.allclose(oo, oms, rtol=1e-12, atol=0), (name, kind, k)
            margins.append(margin)
            key = f"case{len(cases)}__part{k}"
            store[key + "__configs"] = np.array(cfgs, dtype=np.int64)
            store[key + "__omegas"] = np.array(oms, dtype=np.float64)
        cases.append({"state": name, "kind": kind, "seed": seed,
                      "C": [len(c) for c, _ in parts], "margins": margins})
    meta["cases"] = cases
    np.savez_compressed(os.path.join(OUT, "sample.npz"), **store)
    json.dump(meta, open(os.path.join(OUT, "sample.json"), "w"), indent=1)


if __name__ == "__main__":
    sample_cases()
    print("golden fixtures written to", OUT)
    for f in ("sample.npz", "sample.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))
