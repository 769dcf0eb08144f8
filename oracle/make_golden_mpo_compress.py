"""Generate tests/golden/mpo_compress.{npz,json} by running the UNMODIFIED
reference (quimb @ 97ceeae, numpy backend, through oracle/shims as
oracle/make_golden.py does): MatrixProductState.gate_with_mpo with the
'direct', 'dm', 'zipup' and 'zipup-first' methods (tn1d/core.py:2446-2509,
tn1d/compress.py).

Run in the build container only:   python oracle/make_golden_mpo_compress.py
Inputs are stored as (l, p, r) MPS and (l, r, u, d) MPO copies; each case
stores the reference's bond sizes, per-bond singular values and dense output
vector, all independent of the gauge.  Before writing, every case is replayed
on oracle/mpo_compress_np.py and asserted equal, and the zip-up spanning tree
of quimb_b200.mpo_compress.ladder_tree_span is asserted equal to the
reference's get_tree_span.
"""

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden_sample import OUT, _lpr, _ragged_qutrit, qtn  # noqa: E402
from oracle import mpo_compress_np as onp  # noqa: E402
from quimb_b200.mpo_compress import ladder_tree_span  # noqa: E402


def _lrud(m):
    """(l, r, u, d) numpy copies of an MPO's site arrays."""
    out = []
    L = m.L
    for i in range(L):
        t = m[i]
        lay = ""
        for ix in t.inds:
            if ix == m.upper_ind(i):
                lay += "u"
            elif ix == m.lower_ind(i):
                lay += "d"
            elif i > 0 and ix in qtn.bonds(m[i - 1], t):
                lay += "l"
            else:
                lay += "r"
        x = np.asarray(t.data)
        for c in "lrud":
            if c not in lay:
                x = x[..., None]
                lay += c
        out.append(np.ascontiguousarray(np.transpose(x, [lay.index(c) for c in "lrud"])))
    return out


def _rand_mpo(L, D, d, seed):
    """A random non-Hermitian complex MPO; ``d`` an int or one per site."""
    rng = np.random.default_rng(seed)
    dims = [d] * L if isinstance(d, int) else list(d)
    arrays = []
    for i in range(L):
        shape = (1 if i == 0 else D, 1 if i == L - 1 else D, dims[i], dims[i])
        x = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)) / (D * dims[i]) ** 0.5
        if i == 0:
            x = x[0]
        elif i == L - 1:
            x = x[:, 0]
        arrays.append(x)
    return qtn.MatrixProductOperator(arrays, shape="lrud")


def _mixed_dims(dims, seed):
    """A complex MPS whose physical dimension differs from site to site."""
    rng = np.random.default_rng(seed)
    bonds = [1, 2, 5, 6, 4, 3, 2, 1]
    arrays = []
    for i, d in enumerate(dims):
        shape = (bonds[i], bonds[i + 1], d)          # 'lrp'
        x = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
        if i == 0:
            x = x[0]
        elif i == len(dims) - 1:
            x = x[:, 0]
        arrays.append(x)
    return qtn.MatrixProductState(arrays, shape="lrp")


MIXED = [2, 3, 2, 2, 3, 3, 2]


def _span_matches(p, m, transpose):
    """The reference's get_tree_span of the lazily gated ladder against
    ladder_tree_span, rooted at both ends."""
    L = p.L
    psi = p.copy()
    mps_tids = set(psi.tensor_map)
    psi.gate_with_op_lazy_(m, transpose=transpose)

    def node(tid):
        t = psi.tensor_map[tid]
        (i,) = [k for k in range(L) if psi.site_tag(k) in t.tags]
        return i if tid in mps_tids else L + i

    A, W = _lpr(p), _lrud(m)
    for root in (0, L - 1):
        tids = psi._get_tids_from_tags(psi.site_tag(root))
        ref = [(node(a), node(b)) for a, b, _ in psi.get_tree_span(tids, inwards=True)]
        ours = ladder_tree_span(L, [a.shape[2] for a in A[:-1]], [w.shape[1] for w in W[:-1]],
                                [a.shape[1] for a in A], root)
        assert ref == ours, (root, ref, ours)


def _bond_svals(q):
    out = []
    for i in range(1, q.L):
        out.append(np.asarray(q.copy().singular_values(i)))
    return out


def cases():
    L8 = 8
    states = {
        "real": qtn.MPS_rand_state(L8, 6, seed=3, dtype="float64"),
        "cplx": qtn.MPS_rand_state(10, 8, seed=5, dtype="complex128"),
        "qutrit_ragged": _ragged_qutrit(9),
        "long": qtn.MPS_rand_state(12, 16, seed=7, dtype="complex128"),
        "mixed": _mixed_dims(MIXED, 31),
    }
    mpos = {
        "heis": qtn.MPO_ham_heis(L8),
        "heis10": qtn.MPO_ham_heis(10),
        "rand3": _rand_mpo(10, 3, 2, 21),
        "rand5": _rand_mpo(L8, 5, 2, 22),
        "rand_q": _rand_mpo(7, 4, 3, 23),
        "rand12": _rand_mpo(12, 4, 2, 24),
        "rand_mixed": _rand_mpo(7, 3, MIXED, 25),
    }
    for p in states.values():
        assert all(t.left_inds is None for t in p), "inputs must not be flagged isometric"
    store, meta = {}, {"states": {}, "mpos": {}}
    for name, p in states.items():
        for i, x in enumerate(_lpr(p)):
            store[f"{name}__site{i}"] = np.ascontiguousarray(x)
        meta["states"][name] = {"L": p.L}
    for name, m in mpos.items():
        for i, x in enumerate(_lrud(m)):
            store[f"{name}__mpo{i}"] = x
        meta["mpos"][name] = {"L": m.L}

    runs = []
    for method in ("direct", "dm", "zipup", "zipup-first"):
        runs += [
            dict(state="real", mpo="heis", method=method, max_bond=10),
            dict(state="real", mpo="heis", method=method, max_bond=None, cutoff=0.0),
            dict(state="real", mpo="heis", method=method, max_bond=None, cutoff=1e-3),
            dict(state="cplx", mpo="rand3", method=method, max_bond=12),
            dict(state="cplx", mpo="rand3", method=method, max_bond=12, transpose=True),
            dict(state="real", mpo="rand5", method=method, max_bond=9, sweep_reverse=True),
            dict(state="cplx", mpo="heis10", method=method, max_bond=16, normalize=True),
            dict(state="qutrit_ragged", mpo="rand_q", method=method, max_bond=8),
            dict(state="long", mpo="rand12", method=method, max_bond=16),
            dict(state="mixed", mpo="rand_mixed", method=method, max_bond=7),
        ]
    runs += [
        dict(state="cplx", mpo="rand3", method="zipup-first", max_bond=10, max_bond_oversample=14),
        dict(state="real", mpo="rand5", method="zipup-first", max_bond=8, max_bond_oversample=1.5),
        dict(state="long", mpo="rand12", method="zipup-first", max_bond=12,
             max_bond_oversample=1.5, sweep_reverse=True),
        dict(state="cplx", mpo="rand3", method="zipup", max_bond=12, transpose=True,
             sweep_reverse=True, normalize=True),
    ]
    out_cases = []
    spans_checked = set()
    for run in runs:
        p, m = states[run["state"]], mpos[run["mpo"]]
        kw = {k: v for k, v in run.items() if k not in ("state", "mpo")}
        key = (run["state"], run["mpo"], kw.get("transpose", False))
        if key not in spans_checked:
            _span_matches(p, m, kw.get("transpose", False))
            spans_checked.add(key)
        q = p.gate_with_mpo(m, **kw)
        lpr = _lpr(q)
        bonds = [int(x.shape[2]) for x in lpr[:-1]]
        svals = _bond_svals(q)
        vec = np.asarray(q.to_dense()).reshape(-1)
        got = onp.gate_with_mpo(_lpr(p), _lrud(m), **kw)
        assert [x.shape[2] for x in got[:-1]] == bonds, (run, bonds)
        ov = onp.dense(got)
        scale = np.max(np.abs(vec))
        assert np.allclose(ov, vec, rtol=0, atol=1e-10 * scale), (run, np.max(np.abs(ov - vec)))
        for s_o, s_r in zip(onp.schmidt_values(got), svals):
            assert np.allclose(s_o, s_r, rtol=0, atol=1e-10 * s_r[0]), run
        k = len(out_cases)
        store[f"case{k}__vec"] = vec
        for i, s in enumerate(svals):
            store[f"case{k}__S{i}"] = s
        case = dict(run, bonds=bonds)
        out_cases.append(case)
    meta["cases"] = out_cases
    np.savez_compressed(os.path.join(OUT, "mpo_compress.npz"), **store)
    json.dump(meta, open(os.path.join(OUT, "mpo_compress.json"), "w"), indent=1)


if __name__ == "__main__":
    cases()
    print("golden fixtures written to", OUT)
    for f in ("mpo_compress.npz", "mpo_compress.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))
