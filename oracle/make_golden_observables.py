"""Generate tests/golden/observables.{npz,json} by running the UNMODIFIED
reference (quimb @ 97ceeae, numpy backend, through oracle/shims as
oracle/make_golden.py does): schmidt_values / entropy / schmidt_gap,
partial_trace_to_dense_canonical, compute_local_expectation ('canonical' and
'envs'), magnetization and correlation of quimb/tensor/tn1d/core.py.

Run in the build container only:   python oracle/make_golden_observables.py
Site arrays are stored as (l, p, r) copies ("<name>__site<i>"); every case
stores its inputs by name and the reference's values.  Before writing, every
case is replayed on oracle/observables_np.py and asserted equal.
"""

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden_sample import OUT, _lpr, _ragged_qutrit, qtn  # noqa: E402
from oracle import observables_np as onp  # noqa: E402
from oracle.observables_np import _ops, terms_for  # noqa: E402


def _close(a, b, what, tol=1e-10):
    # values of the unnormalised ragged state are not O(1): relative to the largest
    a, b = np.asarray(a), np.asarray(b)
    tol = tol * max(1.0, float(np.max(np.abs(b), initial=0.0)))
    assert a.shape == b.shape and np.allclose(a, b, rtol=0, atol=tol), (what, a, b)


def observables_cases():
    ghz = (qtn.MPS_computational_state("0000") + qtn.MPS_computational_state("1111")) / 2 ** 0.5
    states = {
        "real": qtn.MPS_rand_state(10, 8, seed=3, dtype="float64"),
        "cplx": qtn.MPS_rand_state(12, 16, seed=5, dtype="complex128"),
        "qutrit_ragged": _ragged_qutrit(9),
        "product": qtn.MPS_computational_state("0110100111"),
        "ghz": ghz,
    }
    store, meta, cases = {}, {"states": {}}, []
    sites = {}
    for name, p in states.items():
        sites[name] = _lpr(p)
        for i, x in enumerate(sites[name]):
            store[f"{name}__site{i}"] = x
        meta["states"][name] = {"L": p.L, "d": int(p.phys_dim(0))}

    def put(key, value):
        store[f"case{len(cases)}__{key}"] = np.asarray(value)

    def copy(name):
        return [x.copy() for x in sites[name]]

    # Schmidt values / entropy / gap at every bond, one info per sweep
    for name, method in [(n, "svd") for n in states] + [("real", "eig")]:
        p, info = states[name].copy(), {}
        o, oinfo = copy(name), {}
        ent, gap = [], []
        for i in range(1, p.L):
            S = p.schmidt_values(i, info=info, method=method)
            ent.append(float(p.entropy(i, info=info, method=method)))
            gap.append(float(p.schmidt_gap(i, info=info, method=method)))
            put(f"S{i}", S)
            _close(onp.schmidt_values(o, i, oinfo, method), S, (name, i), 1e-12 * S[0])
            _close(onp.entropy(o, i, oinfo, method), ent[-1], (name, i))
            _close(onp.schmidt_gap(o, i, oinfo, method), gap[-1], (name, i))
        put("entropy", ent)
        put("gap", gap)
        cases.append({"kind": "schmidt", "state": name, "method": method,
                      "cur_orthog": list(info["cur_orthog"])})

    # reduced density matrices
    for name in ("real", "cplx", "qutrit_ragged", "product"):
        L = states[name].L
        for where in (L // 2, (3, 4), (0, 3), (1, 2, 3), (0, 2, 4)):
            for normalized in (True, False):
                p, info = states[name].copy(), {}
                rho = p.partial_trace_to_dense_canonical(where, normalized=normalized, info=info)
                o, oinfo = copy(name), {}
                _close(onp.partial_trace_to_dense_canonical(o, where, normalized, oinfo), rho,
                       (name, where))
                assert tuple(oinfo["cur_orthog"]) == tuple(info["cur_orthog"])
                put("rho", rho)
                w = [where] if isinstance(where, int) else list(where)
                cases.append({"kind": "rho", "state": name, "where": w,
                              "normalized": normalized,
                              "cur_orthog": list(info["cur_orthog"])})

    # local expectations
    def run_terms(name, label, return_all, method, info=None, start=None, inplace=False):
        meta_s = meta["states"][name]
        terms = terms_for(label, meta_s["L"], meta_s["d"])
        p = states[name].copy()
        o = copy(name)
        if start is not None:
            # a state whose centre really is ``start``
            p.canonicalize_(start, info={"cur_orthog": "calc"})
            o = _lpr(p)
            for i, x in enumerate(o):
                store[f"case{len(cases)}__in{i}"] = x
        rinfo = None if info is None else dict(info)
        oinfo = None if info is None else dict(info)
        got = p.compute_local_expectation(terms, return_all=return_all, method=method,
                                          info=rinfo, inplace=inplace)
        ogot = onp.compute_local_expectation([x.copy() for x in o], terms,
                                             return_all=return_all, method=method,
                                             info=oinfo, inplace=inplace)
        keys = list(got) if return_all else []
        vals = [got[k] for k in keys] if return_all else [got]
        ovals = [ogot[k] for k in keys] if return_all else [ogot]
        assert (list(ogot) == keys) if return_all else True
        _close(ovals, vals, (name, label, method))
        put("values", np.asarray(vals, dtype=np.complex128))
        case = {"kind": "expec", "state": name, "terms": label, "method": method,
                "return_all": return_all, "keys": [list(k) for k in keys],
                "info": None if info is None else _js(info), "start": _js(start),
                "inplace": inplace}
        if rinfo is not None and "cur_orthog" in rinfo:
            case["cur_orthog_after"] = _js(rinfo["cur_orthog"])
            if oinfo is not None:
                assert _js(oinfo["cur_orthog"]) == _js(rinfo["cur_orthog"])
        if inplace:
            after = _lpr(p)
            for i, x in enumerate(after):
                put(f"out{i}", x)
        cases.append(case)

    for name in ("real", "cplx", "qutrit_ragged"):
        for method in ("canonical", "envs"):
            for c in "XZ":
                run_terms(name, c, True, method)
            run_terms(name, "heis", False, method)
            run_terms(name, "far", True, method)
    run_terms("real", "Z", True, "canonical", info={"cur_orthog": "calc"})
    run_terms("cplx", "Z", True, "canonical", info={"cur_orthog": 3}, start=3)
    run_terms("cplx", "heis", True, "canonical", info={"cur_orthog": (2, 4)}, start=(2, 4))
    run_terms("real", "heis", True, "canonical", info={}, inplace=True)
    run_terms("qutrit_ragged", "X", True, "canonical", info={"cur_orthog": "calc"},
              inplace=True)

    # magnetisation
    for name, i in (("cplx", 5), ("qutrit_ragged", 3), ("real", 2)):
        p, info = states[name].copy(), {}
        o, oinfo = copy(name), {}
        vals = []
        for c in "XYZ":
            vals.append(complex(p.magnetization(i, c, info=info)))
            _close(onp.magnetization(o, i, c, oinfo), vals[-1], (name, c))
        put("values", vals)
        cases.append({"kind": "mag", "state": name, "site": i,
                      "cur_orthog": list(info["cur_orthog"])})

    # correlation
    Z, X = _ops(2)["Z"], _ops(2)["X"]
    for name, i, j, withB in (("ghz", 0, 1, False), ("ghz", 0, 1, True),
                              ("real", 1, 6, False), ("cplx", 7, 2, True)):
        p = states[name]
        c = complex(p.correlation(Z, i, j, B=X if withB else None))
        _close(onp.correlation(copy(name), Z, i, j, B=X if withB else None), c, (name, i, j))
        put("value", c)
        cases.append({"kind": "corr", "state": name, "i": i, "j": j, "B": withB})
    meta["cases"] = cases
    np.savez_compressed(os.path.join(OUT, "observables.npz"), **store)
    json.dump(meta, open(os.path.join(OUT, "observables.json"), "w"), indent=1)


def _js(x):
    return list(x) if isinstance(x, tuple) else x


if __name__ == "__main__":
    observables_cases()
    print("golden fixtures written to", OUT)
    for f in ("observables.npz", "observables.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))
