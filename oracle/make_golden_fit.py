"""Generate tests/golden/fit.{npz,json} by running the UNMODIFIED reference
(quimb @ 97ceeae, numpy backend, through oracle/shims as oracle/make_golden.py
does): tensor_network_1d_compress(targets, method='fit') with the one- and
two-site sweeps (tn1d/compress.py:2345-2966).

Run in the build container only:   python oracle/make_golden_fit.py
Every case starts from an explicit guess -- a stored random MPS or
``tn_fit='zipup'`` -- since the reference's own random start is drawn through
a namespace the shims do not provide.  Targets are (mpo, psi) ladders and
MPSs from oracle/make_golden_mpo_compress.py, stored as (l, p, r) MPS and
(l, r, u, d) MPO copies.

Pinned cases store the reference's bond sizes, per-bond singular values and
dense output vector (all gauge-independent).  One-site cases are pinned only
from guesses already at max_bond: a one-site fit that has to pad its bonds
depends on how the QR completes the zero directions, i.e. on the guess's
gauge.  Those expansion cases ('property' cases) store the reference's
fidelity with the exact sum instead.  Before writing, every case is replayed
on oracle/fit_np.py and asserted equal (the property cases to within their
stated tolerance); every two-site truncation and every ``tol`` decision is
asserted to be made far from rounding noise.
"""

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden_sample import OUT, _lpr, _ragged_qutrit, qtn  # noqa: E402
from oracle.make_golden_mpo_compress import (MIXED, _bond_svals, _lrud, _mixed_dims,  # noqa: E402
                                             _rand_mpo)
from oracle import fit_np as onp  # noqa: E402
from oracle.fit_np import check_svd_margin, check_tol_margin  # noqa: E402

# one-site fits from a padded guess: the reference's fidelity with the exact
# sum, less this, bounds ours
PROPERTY_TOL = 1e-4


def _rand_guess(dims, bond, seed, dtype):
    """A random (l, p, r) MPS with bonds min(bond, prod d left, prod d right)."""
    rng = np.random.default_rng(seed)
    L = len(dims)
    bonds = [1] + [min(bond, int(np.prod(dims[:i])), int(np.prod(dims[i:])))
                   for i in range(1, L)] + [1]
    out = []
    for i, d in enumerate(dims):
        shape = (bonds[i], d, bonds[i + 1])
        x = rng.standard_normal(shape)
        if np.dtype(dtype).kind == "c":
            x = x + 1j * rng.standard_normal(shape)
        out.append((x / np.sqrt(bonds[i] * d)).astype(dtype))
    return out


def _to_mps(sites):
    """An (l, p, r) list as a reference MPS ('lrp', no outer bonds at the ends)."""
    arrays = []
    L = len(sites)
    for i, a in enumerate(sites):
        x = a.transpose(0, 2, 1)
        if L == 1:
            x = x[0, 0]
        elif i == 0:
            x = x[0]
        elif i == L - 1:
            x = x[:, 0]
        arrays.append(x)
    return qtn.MatrixProductState(arrays, shape="lrp")


def _one_site_chain():
    """The reference does not fit a one-site chain: with an explicit guess
    the guess has no bond to read its size from, and the zip-up guess has no
    bond to split.  Returns the exception names it raises."""
    rng = np.random.default_rng(45)
    p = qtn.MatrixProductState([rng.standard_normal(3) + 0j], shape="lrp")
    m = qtn.MatrixProductOperator([rng.standard_normal((3, 3)) + 0j], shape="lrud")
    out = []
    for tn_fit in (p.copy(), "zipup"):
        try:
            qtn.tensor_network_1d_compress([p.gate_with_op_lazy(m)], method="fit",
                                           tn_fit=tn_fit, max_bond=1, cutoff=None)
        except (TypeError, AttributeError) as e:
            out.append(type(e).__name__)
        else:
            raise AssertionError("the reference fitted a one-site chain")
    return out


def cases():
    states = {
        "real": qtn.MPS_rand_state(8, 6, seed=3, dtype="float64"),
        "real_b": qtn.MPS_rand_state(8, 5, seed=13, dtype="float64"),
        "cplx": qtn.MPS_rand_state(10, 8, seed=5, dtype="complex128"),
        "cplx_b": qtn.MPS_rand_state(10, 6, seed=15, dtype="complex128"),
        "qutrit_ragged": _ragged_qutrit(9),
        "mixed": _mixed_dims(MIXED, 31),
        "two": qtn.MPS_rand_state(2, 2, seed=41, dtype="complex128"),
        "two_b": qtn.MPS_rand_state(2, 2, seed=42, dtype="complex128"),
    }
    mpos = {
        "heis": qtn.MPO_ham_heis(8),
        "heis10": qtn.MPO_ham_heis(10),
        "rand3": _rand_mpo(10, 3, 2, 21),
        "rand5": _rand_mpo(8, 5, 2, 22),
        "rand_q": _rand_mpo(7, 4, 3, 23),
        "rand_mixed": _rand_mpo(7, 3, MIXED, 25),
        "two": _rand_mpo(2, 3, 2, 26),
    }
    store, meta = {}, {"states": {}, "mpos": {}, "guesses": {}}
    for name, p in states.items():
        for i, x in enumerate(_lpr(p)):
            store[f"{name}__site{i}"] = np.ascontiguousarray(x)
        meta["states"][name] = {"L": p.L}
    for name, m in mpos.items():
        for i, x in enumerate(_lrud(m)):
            store[f"{name}__mpo{i}"] = x
        meta["mpos"][name] = {"L": m.L}

    def guess(name, state, bond, seed):
        p = _lpr(states[state])
        dt = np.result_type(*p)
        g = _rand_guess([x.shape[1] for x in p], bond, seed, dt)
        for i, x in enumerate(g):
            store[f"{name}__guess{i}"] = x
        meta["guesses"][name] = {"L": len(g)}
        return name

    g = {
        "real4": guess("real4", "real", 4, 101),
        "real8": guess("real8", "real", 8, 102),
        "cplx6": guess("cplx6", "cplx", 6, 103),
        "cplx10": guess("cplx10", "cplx", 10, 104),
        "cplx4": guess("cplx4", "cplx", 4, 112),
        "cplx12": guess("cplx12", "cplx", 12, 105),
        "real9": guess("real9", "real", 9, 106),
        "real5": guess("real5", "real", 5, 107),
        "q4": guess("q4", "qutrit_ragged", 4, 108),
        "q6": guess("q6", "qutrit_ragged", 6, 109),
        "mixed3": guess("mixed3", "mixed", 3, 110),
        "mixed6": guess("mixed6", "mixed", 6, 111),
        "two2": guess("two2", "two", 2, 113),
    }
    M = lambda mpo, state: ["mpo", mpo, state]  # noqa: E731
    S = lambda state: ["mps", state]  # noqa: E731
    runs = [
        # two-site
        dict(targets=[M("heis", "real")], guess=g["real4"], bsz=2, max_bond=10),
        dict(targets=[M("rand3", "cplx")], guess=g["cplx6"], bsz=2, max_bond=12, transpose=True),
        dict(targets=[M("rand5", "real")], guess=g["real5"], bsz=2, max_bond=9, sweep_reverse=True),
        dict(targets=[M("rand5", "real")], guess=g["real5"], bsz=2, max_bond=9,
             sweep_sequence="LR"),
        dict(targets=[M("rand5", "real")], guess=g["real5"], bsz=2, max_bond=9,
             sweep_sequence="LR", sweep_reverse=True),
        dict(targets=[M("heis10", "cplx")], guess=g["cplx6"], bsz=2, max_bond=16, normalize=True),
        dict(targets=[M("rand_q", "qutrit_ragged")], guess=g["q4"], bsz=2, max_bond=8),
        dict(targets=[M("rand_mixed", "mixed")], guess=g["mixed3"], bsz=2, max_bond=7),
        dict(targets=[M("rand3", "cplx")], guess=g["cplx6"], bsz=2, max_bond=12, tol=1e-4,
             max_iterations=30),
        dict(targets=[M("heis", "real"), S("real_b")], guess=g["real4"], bsz=2, max_bond=10),
        dict(targets=[S("cplx"), S("cplx_b")], guess=g["cplx6"], bsz=2, max_bond=10,
             sweep_sequence="R"),
        dict(targets=[M("rand3", "cplx")], guess="zipup", max_bond=10, cutoff=1e-10),
        dict(targets=[M("heis", "real")], guess="zipup", cutoff=1e-3, max_iterations=4),
        dict(targets=[M("heis", "real")], guess=g["real8"], cutoff=1e-3, max_iterations=4),
        # one-site from a guess at max_bond
        dict(targets=[M("heis", "real")], guess=g["real8"], bsz=1, max_bond=8),
        dict(targets=[M("rand3", "cplx")], guess=g["cplx10"], bsz=1, max_bond=10,
             sweep_sequence="LR"),
        dict(targets=[M("rand5", "real")], guess=g["real9"], bsz=1, max_bond=9,
             sweep_reverse=True),
        dict(targets=[M("heis10", "cplx")], guess=g["cplx12"], max_bond=12, normalize=True,
             sweep_reverse=True, sweep_sequence="LR"),
        dict(targets=[M("rand_q", "qutrit_ragged")], guess=g["q6"], bsz=1, max_bond=6,
             transpose=True),
        dict(targets=[M("rand_mixed", "mixed")], guess=g["mixed6"], bsz=1, max_bond=6),
        dict(targets=[M("rand3", "cplx")], guess=g["cplx10"], bsz=1, max_bond=10, tol=1e-3,
             max_iterations=30, sweep_sequence="RRL"),
        dict(targets=[M("heis", "real"), S("real_b")], guess=g["real8"], bsz=1, max_bond=8),
        dict(targets=[S("cplx"), S("cplx_b")], guess=g["cplx10"], bsz=1, max_bond=10),
        dict(targets=[M("rand3", "cplx")], guess="zipup", max_bond=10, initial_bond_dim=10),
        # one-site bond expansion: by property
        dict(targets=[M("heis10", "cplx")], guess=g["cplx4"], bsz=1, max_bond=12, tol=1e-5,
             max_iterations=60, property=True),
        dict(targets=[M("rand3", "cplx"), S("cplx_b")], guess="zipup", bsz=1, max_bond=12,
             initial_bond_dim=4, tol=1e-5, max_iterations=60, property=True),
        # short chains
        dict(targets=[M("two", "two")], guess=g["two2"], bsz=2, max_bond=2),
        dict(targets=[M("two", "two"), S("two_b")], guess=g["two2"], bsz=1, max_bond=2),
        dict(targets=[M("two", "two")], guess="zipup", max_bond=2, cutoff=1e-10),
    ]

    def ref_target(t, transpose):
        if t[0] == "mps":
            return states[t[1]].copy()
        return states[t[2]].gate_with_op_lazy(mpos[t[1]], transpose=transpose)

    def np_target(t):
        if t[0] == "mps":
            return _lpr(states[t[1]])
        return (_lrud(mpos[t[1]]), _lpr(states[t[2]]))

    out_cases = []
    for run in runs:
        kw = {k: v for k, v in run.items() if k not in ("targets", "guess", "property")}
        tr = kw.get("transpose", False)
        tns = [ref_target(t, tr) for t in run["targets"]]
        rkw = {k: v for k, v in kw.items() if k != "transpose"}
        # the dispatcher's own default cutoff is 1e-10: pass the fit's default
        rkw.setdefault("cutoff", None)
        if run["guess"] == "zipup":
            tn_fit, np_guess = "zipup", "zipup"
        else:
            L = meta["guesses"][run["guess"]]["L"]
            np_guess = [store[f"{run['guess']}__guess{i}"] for i in range(L)]
            tn_fit = _to_mps(np_guess)
        q = qtn.tensor_network_1d_compress(tns, method="fit", tn_fit=tn_fit, **rkw)
        lpr = _lpr(q)
        bonds = [int(x.shape[2]) for x in lpr[:-1]]
        vec = np.asarray(q.to_dense()).reshape(-1)
        targets = [np_target(t) for t in run["targets"]]
        spectra, info = [], {}
        got = onp.fit(targets, guess=np_guess, spectra=spectra, info=info, **kw)
        check_tol_margin(info["tdiffs"], kw.get("tol", 0.0))
        exact = onp.target_dense(targets, tr)
        case = dict(run, bonds=bonds, sweeps=info["sweeps"])
        k = len(out_cases)
        if run.get("property"):
            f_ref = float(onp.fidelity(vec, exact))
            f_np = float(onp.fidelity(onp.dense(got), exact))
            assert f_np >= f_ref - PROPERTY_TOL, (run, f_np, f_ref)
            case["fidelity_ref"] = f_ref
        else:
            assert [x.shape[2] for x in got[:-1]] == bonds, (run, bonds)
            ov = onp.dense(got)
            scale = np.max(np.abs(vec))
            assert np.allclose(ov, vec, rtol=0, atol=1e-10 * scale), (run, np.max(np.abs(ov - vec)))
            svals = _bond_svals(q)
            for s_o, s_r in zip(onp.schmidt_values(got), svals):
                assert np.allclose(s_o, s_r, rtol=0, atol=1e-10 * s_r[0]), run
            for s, mb, cut, mode in spectra:
                check_svd_margin(s, mb, cut, mode)
            store[f"case{k}__vec"] = vec
            for i, s in enumerate(svals):
                store[f"case{k}__S{i}"] = s
        out_cases.append(case)
    meta["cases"] = out_cases
    meta["one_site_chain_raises"] = _one_site_chain()
    meta["property_tol"] = PROPERTY_TOL
    np.savez_compressed(os.path.join(OUT, "fit.npz"), **store)
    json.dump(meta, open(os.path.join(OUT, "fit.json"), "w"), indent=1)


if __name__ == "__main__":
    cases()
    print("golden fixtures written to", OUT)
    for f in ("fit.npz", "fit.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))
