"""Generate tests/golden/nonlocal.{npz,json} by running the UNMODIFIED
reference (quimb @ 97ceeae, numpy backend, through oracle/shims as
oracle/make_golden.py does): MatrixProductOperator.from_dense,
MatrixProductState.gate_nonlocal and gate_with_submpo (tn1d/core.py:
2339-2588, 4241-4345) with the 'direct', 'dm' and 'zipup' compressions, the
controlled MPO of Gate.build_mpo (circuit/gates.py:1123-1152) and a short
CircuitMPS run with gate_contract='auto-mps'.

Run in the build container only:   python oracle/make_golden_nonlocal.py
Inputs are stored as (l, p, r) MPS copies and dense gates; each case stores
the reference's bond sizes, per-bond singular values, dense output vector and
``info["cur_orthog"]``, all independent of the gauge.  Before writing, every
case is replayed on oracle/nonlocal_np.py and asserted equal; every
truncating cut of the replay is asserted to lie far above rounding noise (a
relative gap of at least 1e-6 at the kept rank, and a 'cutoff' threshold
that is not within 1e-3 of the discarded weight), so the pinned bond sizes
do not depend on rounding; and for every zip-up case the spanning tree of
quimb_b200.mpo_compress.ladder_tree_span is asserted equal to the
reference's get_tree_span of the sub-range network it builds.
"""

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden_sample import OUT, _lpr, _ragged_qutrit, qtn  # noqa: E402
from oracle.make_golden_mpo_compress import MIXED, _mixed_dims  # noqa: E402
from oracle import mpo_compress_np as mnp  # noqa: E402
from oracle import nonlocal_np as onp  # noqa: E402
from quimb_b200.mpo_compress import ladder_tree_span  # noqa: E402

import quimb as qu  # noqa: E402
from quimb.tensor.circuit.gates import Gate  # noqa: E402
from quimb.tensor.tn1d.compress import enforce_1d_like  # noqa: E402


# ------------------------------------------------------------------ checks ---
def _span_matches(p, mpo, where, sweep_reverse):
    """The reference's get_tree_span of the sub-range network gate_with_submpo
    hands to the zip-up compressor, against ladder_tree_span."""
    si, sf = min(where), max(where)
    N = sf - si + 1
    psi = p.copy()
    psi.canonicalize_((si, sf))
    A = _lpr(psi)[si:sf + 1]
    psi.add_tag("_KET")
    psi.gate_with_op_lazy_(mpo)
    tags = [psi.site_tag(s) for s in range(si, sf + 1)]
    _, sub = psi.partition(tags, which="any", inplace=True)
    sub = enforce_1d_like(sub, site_tags=tags)

    def node(tid):
        t = sub.tensor_map[tid]
        (i,) = [k for k in range(N) if tags[k] in t.tags]
        return i if "_KET" in t.tags else N + i

    gaps = [s - si for s in range(si, sf + 1) if s not in where]
    bw = []
    for i in range(N - 1):
        (t1,) = [t for t in sub.select_tensors(tags[i]) if "_KET" not in t.tags]
        (t2,) = [t for t in sub.select_tensors(tags[i + 1]) if "_KET" not in t.tags]
        bw.append(t1.bonds_size(t2))
    bond_a = [a.shape[2] for a in A[:-1]]
    root = 0 if sweep_reverse else N - 1
    tids = sub._get_tids_from_tags(tags[root])
    ref = [(node(a), node(b)) for a, b, _ in sub.get_tree_span(tids, inwards=True)]
    ours = ladder_tree_span(N, bond_a, bw, [a.shape[1] for a in A], root, gaps=gaps,
                            open_ends=(si > 0, sf < p.L - 1), rung_between=True)
    assert ref == ours, (where, ref, ours)


class _Cuts:
    """Records every truncating split the oracle makes and checks its margin."""

    def __init__(self):
        self.orig = mnp._split
        self.worst = np.inf

    def __enter__(self):
        mnp._split = self._split
        return self

    def __exit__(self, *exc):
        mnp._split = self.orig

    def _split(self, mat, method="svd", max_bond=None, cutoff=1e-10, cutoff_mode="rsum2",
               **kw):
        out = self.orig(mat, method=method, max_bond=max_bond, cutoff=cutoff,
                        cutoff_mode=cutoff_mode, **kw)
        if method == "eigh":
            s = np.sort(np.abs(np.linalg.eigvalsh(mat)))[::-1]
            n = out[0].shape[1]
        else:
            s = np.linalg.svd(mat, compute_uv=False)
            n = out[0].shape[1]
        self.check(s, n, cutoff, cutoff_mode)
        return out

    def check(self, s, n, cutoff, mode):
        if n >= s.size or s[0] == 0 or s[n] <= 1e-12 * s[0]:
            return                                   # nothing but noise is discarded
        gap = (s[n - 1] - s[n]) / s[0]
        assert gap > 1e-6, ("cut inside a near-degenerate pair", n, s[max(0, n - 2):n + 2])
        self.worst = min(self.worst, gap)
        if cutoff and cutoff > 0:
            p = 2 if mode == "rsum2" else 1
            tail = np.cumsum((s ** p)[::-1])[::-1]
            thr = cutoff * tail[0]
            for t in (tail[n], tail[n - 1]):
                assert abs(t - thr) > 1e-3 * thr, ("cut at the cutoff threshold", n, t, thr)


def _bond_svals(q):
    return [np.asarray(q.copy().singular_values(i)) for i in range(1, q.L)]


def _record(store, k, q, info):
    lpr = _lpr(q)
    vec = np.asarray(q.to_dense()).reshape(-1)
    store[f"case{k}__vec"] = vec
    svals = _bond_svals(q)
    for i, s in enumerate(svals):
        store[f"case{k}__S{i}"] = s
    return dict(bonds=[int(x.shape[2]) for x in lpr[:-1]],
                cur_orthog=list(info["cur_orthog"]) if info is not None else None), vec, svals


def _compare(run, got, vec, svals, bonds):
    assert [int(x.shape[2]) for x in got[:-1]] == bonds, (run, bonds,
                                                          [x.shape[2] for x in got[:-1]])
    ov = mnp.dense(got)
    scale = np.max(np.abs(vec))
    assert np.allclose(ov, vec, rtol=0, atol=1e-10 * scale), (run, np.max(np.abs(ov - vec)))
    for s_o, s_r in zip(mnp.schmidt_values(got), svals):
        assert np.allclose(s_o, s_r, rtol=0, atol=1e-10 * s_r[0]), run


# ------------------------------------------------------------------- cases ---
def _gates():
    rng = np.random.default_rng(11)
    g = {
        "U8": np.asarray(qu.rand_uni(8, seed=2)),
        "U4": np.asarray(qu.rand_uni(4, seed=3)),
        "U9": np.asarray(qu.rand_uni(9, seed=4)),
        "U12": np.asarray(qu.rand_uni(12, seed=5)),
        "U6": np.asarray(qu.rand_uni(6, seed=6)),
        "O8": np.linalg.qr(rng.standard_normal((8, 8)))[0],
        "O4": np.linalg.qr(rng.standard_normal((4, 4)))[0],
        "CX": np.asarray(Gate("CX", params=(), qubits=(0, 1)).array).reshape(4, 4),
        "RZZ": np.asarray(Gate("RZZ", params=(0.7,), qubits=(0, 1)).array).reshape(4, 4),
        "CCX": np.asarray(Gate("CCX", params=(), qubits=(0, 1, 2)).array).reshape(8, 8),
        "X": np.asarray(Gate("X", params=(), qubits=(0,)).array).reshape(2, 2),
        "H": np.asarray(Gate("H", params=(), qubits=(0,)).array).reshape(2, 2),
    }
    return {k: np.ascontiguousarray(v) for k, v in g.items()}


def cases():
    states = {
        "real": qtn.MPS_rand_state(8, 6, seed=3, dtype="float64"),
        "cplx": qtn.MPS_rand_state(8, 8, seed=5, dtype="complex128"),
        "qutrit_ragged": _ragged_qutrit(9),
        "mixed": _mixed_dims(MIXED, 31),
    }
    gates = _gates()
    store, meta = {}, {"states": {}, "gates": sorted(gates)}
    for name, p in states.items():
        for i, x in enumerate(_lpr(p)):
            store[f"{name}__site{i}"] = np.ascontiguousarray(x)
        meta["states"][name] = {"L": p.L}
    for name, G in gates.items():
        store[f"gate__{name}"] = G

    runs = []
    for method in ("direct", "dm", "zipup"):
        runs += [
            dict(state="cplx", gate="U8", where=[7, 2, 4], method=method, max_bond=6),
            dict(state="cplx", gate="U8", where=[7, 2, 4], method=method),
            dict(state="cplx", gate="U4", where=[0, 1], method=method, max_bond=6),
            dict(state="cplx", gate="U4", where=[6, 7], method=method, max_bond=4),
            dict(state="cplx", gate="U8", where=[0, 3, 7], method=method, max_bond=7),
            dict(state="cplx", gate="U8", where=[0, 3, 7], method=method, cutoff=0.0),
            dict(state="cplx", gate="U4", where=[5, 1], method=method, max_bond=7),
            dict(state="cplx", gate="U4", where=[5, 1], method=method, max_bond=7,
                 transpose=True),
            dict(state="real", gate="O8", where=[6, 1, 3], method=method, max_bond=5),
            dict(state="real", gate="CCX", where=[0, 3, 7], method=method),
            dict(state="real", gate="CX", where=[0, 2], method=method),
            dict(state="cplx", gate="RZZ", where=[1, 3], method=method),
            dict(state="cplx", gate="U8", where=[1, 6, 3], method=method, max_bond=6,
                 sweep_reverse=True),
            dict(state="qutrit_ragged", gate="U9", where=[4, 1], method=method, max_bond=6),
            dict(state="mixed", gate="U12", where=[0, 4, 2], method=method, max_bond=5),
            dict(state="mixed", gate="U6", where=[6, 1], method=method, max_bond=4),
            dict(state="real", gate="X", controls=[0, 2], where=[4], method=method),
            dict(state="cplx", gate="X", controls=[0, 2], where=[4], method=method,
                 max_bond=6),
            dict(state="cplx", gate="U4", controls=[3], where=[0, 6], method=method,
                 max_bond=7),
        ]
    out_cases = []
    cuts = _Cuts()
    for run in runs:
        p = states[run["state"]]
        G = gates[run["gate"]]
        kw = {k: v for k, v in run.items() if k not in ("state", "gate", "where", "controls")}
        where = tuple(run["where"])
        info = {}
        if run.get("controls"):
            gate = Gate.from_raw(G, qubits=where, controls=tuple(run["controls"]))
            mpo = gate.build_mpo()
            allsites = tuple(sorted(where + tuple(run["controls"])))
            dense_ref = np.asarray(mpo.to_dense([mpo.upper_ind(i) for i in allsites],
                                                [mpo.lower_ind(i) for i in allsites]))
            ours, _ = onp.controlled_mpo(G, where, run["controls"])
            assert np.allclose(_mpo_dense(ours), dense_ref), run
            if kw["method"] == "zipup":
                _span_matches(p, mpo, allsites, kw.get("sweep_reverse", False))
            q = p.gate_with_submpo(mpo, where=allsites, info=info, **kw)
            with cuts:
                got, c = onp.gate_controlled(_lpr(p), G, list(where), list(run["controls"]),
                                             **kw)
        else:
            dims = tuple(p.phys_dim(i) for i in where)
            if kw["method"] == "zipup":
                mpo = qtn.MatrixProductOperator.from_dense(G, dims=dims, sites=where, L=p.L)
                _span_matches(p, mpo, where, kw.get("sweep_reverse", False))
            q = p.gate_nonlocal(G, where, info=info, **kw)
            with cuts:
                got, c = onp.gate_nonlocal(_lpr(p), G, where, **kw)
        k = len(out_cases)
        case, vec, svals = _record(store, k, q, info)
        _compare(run, got, vec, svals, case["bonds"])
        assert tuple(case["cur_orthog"]) == (c, c), (run, info)
        out_cases.append(dict(run, **case))

    # the MPO itself: from_dense of every gate kind, as a dense operator
    for name, where, dims in (("CCX", (0, 3, 7), 2), ("U9", (4, 1), 3), ("U12", (0, 4, 2),
                                                                         (2, 3, 2))):
        m = qtn.MatrixProductOperator.from_dense(gates[name], dims=dims, sites=where)
        ours, sites = onp.from_dense(gates[name], dims, where)
        ref_bonds = [int(m.bond_size(a, b)) for a, b in zip(sites[:-1], sites[1:])]
        assert [w.shape[1] for w in ours[:-1]] == ref_bonds, (name, ref_bonds)
        meta.setdefault("from_dense", []).append(
            dict(gate=name, where=list(where), dims=dims, bonds=ref_bonds))

    circ = _circuit(gates)
    meta["circuit"] = circ.pop("meta")
    store.update(circ)
    meta["cases"] = out_cases
    meta["min_cut_gap"] = float(cuts.worst)
    np.savez_compressed(os.path.join(OUT, "nonlocal.npz"), **store)
    json.dump(meta, open(os.path.join(OUT, "nonlocal.json"), "w"), indent=1)


def _mpo_dense(W):
    """The dense operator of an (l, r, u, d) MPO, sites in order."""
    T = np.ones((1, 1, 1))
    for w in W:
        T = np.einsum("xal,lruv->xuavr", T, w).reshape(T.shape[0] * w.shape[2],
                                                      T.shape[1] * w.shape[3], w.shape[1])
    return T[..., 0]


def _circuit(gates):
    """CircuitMPS on 10 qubits: layers of H and random rotations, a Toffoli
    (dense 3-site gate, nonlocal), a doubly controlled X (sub-MPO), a
    long-range CX (swap + split) and a controlled rotation."""
    N = 10
    rng = np.random.default_rng(17)
    seq = []
    for q in range(N):
        seq.append(("H", (q,), (), ()))
    for q in range(N):
        seq.append(("RY", (q,), (), (float(rng.uniform(0, np.pi)),)))
    seq += [
        ("CCX", (0, 4, 9), (), ()),
        ("X", (6,), (1, 8), ()),
        ("CX", (2, 9), (), ()),
        ("RZZ", (3, 7), (), (0.4,)),
        ("CCX", (8, 2, 5), (), ()),
        ("RX", (5,), (0, 9), (0.9,)),
        ("CX", (7, 1), (), ()),
    ]
    for q in range(N):
        seq.append(("RZ", (q,), (), (float(rng.uniform(0, np.pi)),)))
    seq.append(("CCX", (3, 6, 1), (), ()))
    circ = qtn.CircuitMPS(N, max_bond=12, cutoff=1e-10)
    store, entries = {}, []
    for k, (name, qs, cs, params) in enumerate(seq):
        g = Gate(name, params=params, qubits=qs, controls=cs if cs else None)
        store[f"circ__gate{k}"] = np.ascontiguousarray(
            np.asarray(Gate(name, params=params, qubits=qs).array).reshape(2 ** len(qs), -1))
        entries.append(dict(name=name, qubits=list(qs), controls=list(cs)))
        circ.apply_gate(g)
    psi = circ.psi
    vec = np.asarray(psi.to_dense()).reshape(-1)
    store["circ__vec"] = vec
    bonds = [int(x.shape[2]) for x in _lpr(psi)[:-1]]
    # the oracle replays the same gate list
    sites = [np.zeros((1, 2, 1), dtype=complex) for _ in range(N)]
    for s in sites:
        s[0, 0, 0] = 1.0
    glist = [(store[f"circ__gate{k}"], e["qubits"], e["controls"]) if e["controls"] else
             (store[f"circ__gate{k}"], e["qubits"]) for k, e in enumerate(entries)]
    got = onp.apply_circuit(sites, glist, contract="auto-mps", max_bond=12, cutoff=1e-10)
    assert [int(x.shape[2]) for x in got[:-1]] == bonds, (bonds, [x.shape[2] for x in got])
    ov = mnp.dense(got)
    assert np.allclose(ov, vec, rtol=0, atol=1e-10), np.max(np.abs(ov - vec))
    store["meta"] = dict(N=N, max_bond=12, cutoff=1e-10, gates=entries, bonds=bonds)
    return store


if __name__ == "__main__":
    cases()
    print("golden fixtures written to", OUT)
    for f in ("nonlocal.npz", "nonlocal.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))
