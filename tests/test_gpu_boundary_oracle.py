"""GPU tier: boundary-MPS contraction (quimb_b200/boundary.py) and compressed
contraction (quimb_b200/compressed.py) against their numpy restatements
(oracle/boundary_np.py, oracle/compressed_np.py) at sizes the reference
fixtures do not reach: boundary bonds of 64-128 and bond dimensions of 4,
where the contractions, QRs and SVDs take their large-matrix routes.

Tolerance rule.  A truncated contraction is a deterministic function of the
input only while every kept rank is decided away from rounding.  Each
oracle run records the relative gap at every cut; the tests assert the
smallest one is at least 1e-6 (the seeds are chosen so) and then hold the
device to the oracle at 1e-8 relative: a perturbation of the singular values
of order 1e-15 cannot move a cut that stands 1e-6 clear, and the truncation
error it can move is bounded by the gap times the product's conditioning.
Ranks, ``n_compress`` and ``max_bond_seen`` must be identical.  Single
precision networks are widened on entry, so they are held to the float64
oracle on the same (upcast) inputs at the same tolerance."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import boundary_np as bnp
from oracle import compressed_np as cnp
from oracle import contract_np as cpn
from quimb_b200 import _lib, linalg
from quimb_b200 import boundary as bd
from quimb_b200 import compressed as cq
from quimb_b200 import contract as qc
from quimb_b200 import ops, tree
from tests import decomp_oracle as do
from tests import route_oracle as ro

pytestmark = pytest.mark.gpu

MIN_GAP = 1e-6
TOL = 1e-8


def _rand(rng, shape, dtype, shift=0.0):
    x = rng.standard_normal(shape) + shift
    if np.dtype(dtype).kind == "c":
        x = x + 1j * rng.standard_normal(shape)
    return x.astype(dtype)


def _peps(Lx, Ly, D, d, seed, dtype):
    """A PEPS grid in quimb's site convention (up, right, down, left, phys)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(Lx):
        row = []
        for j in range(Ly):
            nb = (i < Lx - 1) + (j < Ly - 1) + (i > 0) + (j > 0)
            row.append(_rand(rng, (D,) * nb + (d,), dtype))
        out.append(row)
    return out


def _flat(Lx, Ly, D, seed, dtype="float64", shift=0.0):
    """A flat 2D network: one tensor per site, bonds of size D."""
    rng = np.random.default_rng(seed)
    ts = []
    for i in range(Lx):
        for j in range(Ly):
            inds = [f"v{i},{j}"] * (i < Lx - 1) + [f"h{i},{j}"] * (j < Ly - 1)
            inds += [f"v{i - 1},{j}"] * (i > 0) + [f"h{i},{j - 1}"] * (j > 0)
            ts.append((_rand(rng, (D,) * len(inds), dtype, shift), tuple(inds), (i, j), None))
    return ts


def _device(ts):
    return [(qb.asarray(a), inds, coo, layer) for a, inds, coo, layer in ts]


_ORIG_COMPRESS = {m: m.compress_between for m in (bnp, bd, cq)}


def _record_bonds(monkeypatch, module):
    """Bond size after every compress_between of ``module``'s sweep."""
    seen = []
    inner = _ORIG_COMPRESS[module]

    def rec(ta, tb, *args, **kw):
        inner(ta, tb, *args, **kw)
        shared = [ix for ix in ta.inds if ix in tb.inds]
        seen.append(int(np.prod([ta.data.shape[ta.inds.index(ix)] for ix in shared])))
    monkeypatch.setattr(module, "compress_between", rec)
    return seen


# ------------------------------------------------------------ route recorder --
# Every contraction, QR and SVD the cases of this module launch is recorded by
# shape, stride and dtype and mapped through the library's own route
# functions; test_route_coverage (last in the module) asserts the union.
ROUTES = set()
_CONTRACT_USERS = (qc, tree, ops)


def _contract_key(a, la, b, lb, lc, kw):
    ext = dict(zip(la, a.shape))
    ext.update(zip(lb, b.shape))
    out = kw.get("out")
    cs = list(out.shape) if out is not None else [ext[l] for l in lc]
    cst = list(out.stride()) if out is not None else list(np.cumprod(([1] + cs[::-1])[:-1])[::-1])
    r = qc.route_pair(list(a.shape), list(a.stride()), la, list(b.shape), list(b.stride()), lb,
                      cs, [int(v) for v in cst], lc, _lib._TORCH2QB[a.dtype],
                      ptrs=(a.data_ptr(), b.data_ptr(), out.data_ptr() if out is not None
                            else 0x10000000))
    return ro.route_key(str(a.dtype).split(".")[-1], r)


@pytest.fixture(autouse=True)
def _route_recorder(monkeypatch):
    inner_cp = qc.contract_pair

    def cp(a, la, b, lb, lc, *args, **kw):
        key = _contract_key(a, la, b, lb, lc, kw)
        if key is not None:
            ROUTES.add(("contract",) + key)
        return inner_cp(a, la, b, lb, lc, *args, **kw)
    for mod in _CONTRACT_USERS:
        monkeypatch.setattr(mod, "contract_pair", cp)

    inner_qr, inner_svd, inner_trunc = linalg.qr, linalg.svd, linalg.svd_trunc
    inner_fallback = linalg._qr_complex_via_svd

    def qr(x, *args, **kw):
        x = ops.asarray(x)
        ROUTES.update(do.qr_keys_of(linalg.route_qr(x.shape, x.t.dtype)))
        return inner_qr(x, *args, **kw)

    def svd(x, *args, **kw):
        x = ops.asarray(x)
        ROUTES.update(do.svd_keys_of(linalg.route_svd(x.shape, x.t.dtype)))
        return inner_svd(x, *args, **kw)

    def svd_trunc(x, cutoff=-1.0, cutoff_mode=4, max_bond=-1, absorb=0, *args, **kw):
        x = ops.asarray(x)
        ROUTES.update(do.svd_keys_of(linalg.route_svd(x.shape, x.t.dtype, absorb)))
        return inner_trunc(x, cutoff, cutoff_mode, max_bond, absorb, *args, **kw)

    def fallback(x, *args, **kw):
        ROUTES.add(("qr", "complex_via_svd"))
        return inner_fallback(x, *args, **kw)
    monkeypatch.setattr(linalg, "qr", qr)
    monkeypatch.setattr(linalg, "svd", svd)
    monkeypatch.setattr(linalg, "svd_trunc", svd_trunc)
    monkeypatch.setattr(linalg, "_qr_complex_via_svd", fallback)
    yield


def _min_gap(trace):
    return min([r["gap"] for r in trace] + [np.inf])


# ------------------------------------------------------------ exact regime --
@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_boundary_exact_regime_matches_exact_contraction(dtype):
    """cutoff=0 and a bond larger than any the sweep can form: the QR-only
    shortcut keeps everything, so the value is the exact contraction
    whatever gauge moves were made.  The untruncated boundary carries
    redundant bonds, so the complex QRs meet rank-deficient input and take
    the SVD fallback."""
    ts = _flat(5, 5, 4, seed=3, dtype=dtype, shift=1.0)
    exact = cpn.array_contract([t[0] for t in ts], [t[1] for t in ts], (), optimize="greedy")
    v = bd.contract_boundary(_device(ts), 5, 5, max_bond=4096, cutoff=0.0)
    assert abs(v - exact) <= 1e-12 * abs(exact), (v, exact)


# -------------------------------------------------------- truncated regime --
PEPS_OPTS = [dict(), dict(sequence=("ymin", "ymax")), dict(sequence="xmax"),
             dict(canonize=False), dict(cutoff=1e-3)]


@pytest.mark.parametrize("dtype", ["float64", "complex128", "float32", "complex64"])
def test_boundary_peps_norm_matches_oracle(monkeypatch, dtype):
    arrays = _peps(5, 5, 4, 2, seed=0, dtype=dtype)
    ts, Lx, Ly = bnp.peps_norm_tensors(arrays)
    dts, _, _ = bd.peps_norm_tensors([[qb.asarray(a) for a in row] for row in arrays])
    for o in PEPS_OPTS:
        kw = dict(dict(max_bond=64, cutoff=0.0, layer_tags=("KET", "BRA")), **o)
        ranks = _record_bonds(monkeypatch, bnp)
        ref, obc = bnp.contract_boundary(ts, Lx, Ly, **kw)
        ref_ranks = list(ranks)
        ranks.clear()
        gap = _min_gap(obc.trace)
        assert gap >= MIN_GAP, (dtype, o, gap)
        bc = bd.BoundaryContractor2D(dts, Lx, Ly)
        dev_ranks = _record_bonds(monkeypatch, bd)
        v = bc.contract_boundary(**kw)
        assert (bc.n_compress, bc.max_bond_seen) == (obc.n_compress, obc.max_bond_seen), o
        assert dev_ranks == ref_ranks, o
        assert abs(v - ref) <= TOL * abs(ref), (dtype, o, v, ref, gap)


def test_boundary_flat_chi128_matches_oracle(monkeypatch):
    ts = _flat(6, 6, 4, seed=5)
    for o in (dict(), dict(sequence="xmax")):
        kw = dict(max_bond=128, cutoff=0.0, **o)
        ref_ranks = _record_bonds(monkeypatch, bnp)
        ref, obc = bnp.contract_boundary(ts, 6, 6, **kw)
        assert _min_gap(obc.trace) >= MIN_GAP
        bc = bd.BoundaryContractor2D(_device(ts), 6, 6)
        dev_ranks = _record_bonds(monkeypatch, bd)
        v = bc.contract_boundary(**kw)
        assert (bc.n_compress, bc.max_bond_seen) == (obc.n_compress, obc.max_bond_seen)
        assert dev_ranks == ref_ranks, o
        assert abs(v - ref) <= TOL * abs(ref), (o, v, ref)


def test_boundary_without_final_contract_matches_oracle():
    arrays = _peps(5, 5, 4, 2, seed=0, dtype="complex128")
    ts, Lx, Ly = bnp.peps_norm_tensors(arrays)
    kw = dict(max_bond=64, cutoff=0.0, layer_tags=("KET", "BRA"), final_contract=False,
              max_separation=2)
    obc, _ = bnp.contract_boundary(ts, Lx, Ly, **kw)
    ref = obc.close()
    bc = bd.contract_boundary(_device(ts), Lx, Ly, **kw)
    rest = [t for c in sorted(bc.sites) for t in bc.sites[c]]
    assert len(rest) == len(obc.tensors()) > 2
    v, _ = cpn.tensor_contract([t.data.to_numpy() for t in rest], [t.inds for t in rest])
    assert abs(v - ref) <= TOL * abs(ref)


def test_two_sided_on_one_process_is_bitwise_single_process():
    arrays = _peps(5, 5, 4, 2, seed=0, dtype="float64")
    dts, Lx, Ly = bd.peps_norm_tensors([[qb.asarray(a) for a in row] for row in arrays])
    for kw in (dict(max_bond=64, cutoff=0.0), dict(max_bond=48, cutoff=1e-3)):
        a = bd.contract_boundary(dts, Lx, Ly, layer_tags=("KET", "BRA"), **kw)
        b = bd.contract_boundary_two_sided(dts, Lx, Ly, layer_tags=("KET", "BRA"), **kw)
        assert a == b, (kw, a, b)


# ---------------------------------------------------- compressed contraction --
def _reg3(n, D, seed):
    """A random 3-regular graph network (configuration model, resampled until
    simple), one tensor per vertex, bonds of size D."""
    rng = np.random.default_rng(seed)
    while True:
        stubs = rng.permutation(np.repeat(np.arange(n), 3)).reshape(-1, 2)
        edges = {tuple(sorted(e)) for e in stubs.tolist()}
        if len(edges) == len(stubs) and all(a != b for a, b in edges):
            break
    inputs = [[] for _ in range(n)]
    for k, (a, b) in enumerate(sorted(edges)):
        inputs[a].append(f"e{k}")
        inputs[b].append(f"e{k}")
    arrays = [_rand(rng, (D,) * 3, "float64") for _ in range(n)]
    return arrays, inputs, []


COMPRESSED_RUNS = [
    dict(max_bond=8, cutoff=0.0), dict(max_bond=12, cutoff=0.0),
    dict(max_bond=10, cutoff=1e-6), dict(max_bond=8, cutoff=0.0, compress_late=False),
    dict(max_bond=10, cutoff=0.0, compress_span=2),
    dict(max_bond=10, cutoff=0.0, compress_matrices=False),
    dict(max_bond=8, cutoff=0.0, equalize_norms=True),
    dict(max_bond=12, cutoff=0.0, compress_min_size=256),
    dict(max_bond=16, cutoff=0.05, equalize_norms=True, compress_opts={"cutoff_mode": "abs"}),
    dict(max_bond=16, cutoff=2e-3, equalize_norms=True, compress_opts={"cutoff_mode": "sum2"}),
    dict(max_bond=lambda d: 8, cutoff=0.0),
    dict(max_bond=8, cutoff=0.0, compress_exclude={3, 7}),
]


def _compressed_case(name):
    if name == "reg40":
        return _reg3(40, 4, seed=2)
    ts = _flat(6, 6, 4, seed=7)
    return [t[0] for t in ts], [list(t[1]) for t in ts], []


@pytest.mark.parametrize("name", ["reg40", "flat66"])
def test_compressed_matches_oracle(monkeypatch, name):
    arrays, inputs, output = _compressed_case(name)
    seq = cnp.greedy_sequence(arrays, inputs, output)
    dev = [qb.asarray(a) for a in arrays]
    for kw in COMPRESSED_RUNS:
        ref_ranks = _record_bonds(monkeypatch, bnp)
        ref, oinfo = cnp.contract_compressed(arrays, inputs, output, seq, **kw)
        gap = _min_gap(oinfo["trace"])
        assert gap >= MIN_GAP, (name, kw, gap)
        info = {}
        dev_ranks = _record_bonds(monkeypatch, cq)
        got = qb.contract_compressed(dev, inputs, output, seq, info=info, **kw).to_numpy()
        assert (info["n_compress"], info["max_bond_seen"]) == (
            oinfo["n_compress"], oinfo["max_bond_seen"]), (name, kw)
        assert dev_ranks == ref_ranks and len(ref_ranks) == oinfo["n_compress"], (name, kw)
        assert np.abs(got - ref).max() <= TOL * np.abs(ref).max(), (name, kw, got, ref)


def test_compressed_strip_exponent_with_open_outputs_matches_oracle():
    """Open output indices: the mantissa has unit Frobenius norm and the
    exponent is the reference's, with and without equalized norms."""
    ts = _flat(5, 5, 4, seed=11)
    arrays = [t[0] for t in ts]
    inputs = [list(t[1]) for t in ts]
    # cut two bonds open: they become output indices of the corner tensors
    inputs[0] = [ix if ix != "h0,0" else "o1" for ix in inputs[0]]
    inputs[-1] = [ix if ix != "v3,4" else "o2" for ix in inputs[-1]]
    output = ["o1", "o2"]
    seq = cnp.greedy_sequence(arrays, inputs, output)
    dev = [qb.asarray(a) for a in arrays]
    for kw in (dict(max_bond=24, cutoff=0.0), dict(max_bond=24, cutoff=0.0, equalize_norms=False),
               dict(max_bond=32, cutoff=0.05, compress_opts={"cutoff_mode": "abs"})):
        (mant, ex), oinfo = cnp.contract_compressed(arrays, inputs, output, seq,
                                                    strip_exponent=True, **kw)
        assert _min_gap(oinfo["trace"]) >= MIN_GAP
        gm, gex = qb.contract_compressed(dev, inputs, output, seq, strip_exponent=True, **kw)
        gm = gm.to_numpy()
        assert abs(np.linalg.norm(gm) - 1.0) <= 1e-12
        assert abs(gex - ex) <= 1e-9, (kw, gex, ex)
        assert np.abs(gm - mant).max() <= TOL, kw


# ------------------------------------------- one config-5-sized inward step --
def _config5_band(Ly=4, chi=128, D=8, d=2, seed=4):
    """A width-``Ly`` band of BASELINE config 5 (PEPS norm, D=8, d=2,
    complex64): row 0 is a synthetic chi=128 boundary line whose tensors
    carry the ket and bra bonds down into row 1; rows 1 and 2 are two-layer
    PEPS rows.  Scaled so every tensor has entries of order one."""
    rng = np.random.default_rng(seed)
    arrays = _peps(3, Ly, D, d, seed, "complex64")
    ts, Lx, _ = bnp.peps_norm_tensors(arrays)
    band = [t for t in ts if t[2][0] > 0]
    for j in range(Ly):
        inds = [f"b{j - 1}"] * (j > 0) + [f"Kv0,{j}", f"Bv0,{j}"] + [f"b{j}"] * (j < Ly - 1)
        shape = [chi] * (j > 0) + [D, D] + [chi] * (j < Ly - 1)
        band.append((_rand(rng, shape, "complex64") / np.sqrt(chi), tuple(inds), (0, j), None))
    return band, Lx, Ly


def test_config5_inward_step_matches_oracle(monkeypatch):
    """One contract_boundary_from step at config-5 size: the boundary bonds
    reach chi * D = 1024 before compression back to 128, and the QRs of the
    middle boundary tensors are complex matrices of 16384 (chi d D^2) to
    131072 rows by 1024 columns, whose real embeddings take the TSQR route.
    The band is then closed exactly and compared with the oracle's (whose
    step takes about 80 s on 16 host cores)."""
    ts, Lx, Ly = _config5_band()
    kw = dict(max_bond=128, cutoff=0.0, layer_tags=("KET", "BRA"))
    ref_ranks = _record_bonds(monkeypatch, bnp)
    obc = bnp.Boundary2D(ts, Lx, Ly)
    obc.contract_boundary_from((0, 1), (0, Ly - 1), "xmin", **kw)
    ref = obc.close()
    gap = _min_gap(obc.trace)
    assert gap >= MIN_GAP, gap
    assert max(r["shape"][0] for r in obc.trace) >= 128 * 2 * 8 * 8
    bc = bd.BoundaryContractor2D(_device(ts), Lx, Ly)
    dev_ranks = _record_bonds(monkeypatch, bd)
    bc.contract_boundary_from((0, 1), (0, Ly - 1), "xmin", **kw)
    assert (bc.n_compress, bc.max_bond_seen) == (obc.n_compress, obc.max_bond_seen)
    assert dev_ranks == ref_ranks
    rest = [t for c in sorted(bc.sites) for t in bc.sites[c]]
    v, _ = cpn.tensor_contract([t.data.to_numpy() for t in rest], [t.inds for t in rest])
    assert abs(v - ref) <= TOL * abs(ref), (v, ref, gap)


# --------------------------------------------------------------- coverage --
def test_route_coverage():
    """The cases above together reach the large-matrix routes: a large-tile
    DMMA launch (the 128x128 tile, split-K or stream-K), aggregated QR,
    TSQR, the complex QR's SVD fallback on rank-deficient input and more than
    one Jacobi stream group.  Needs the rest of the module to have run."""
    producers = ("test_config5_inward_step_matches_oracle", "test_boundary_peps_norm_matches_oracle")
    if not any(k[0] == "qr" for k in ROUTES):
        pytest.skip(f"run with the rest of the module: the routes come from {producers}")
    contract = {k[1:] for k in ROUTES if k[0] == "contract"}
    print("routes seen:", sorted(map(str, ROUTES)))
    assert any(k[1] in ("splitk", "streamk") or (k[1] == "plain" and k[2] == 0)
               for k in contract), contract
    assert ("qr", "tsqr") in ROUTES
    assert ("qr", "aggregated", "m>4096") in ROUTES or ("qr", "aggregated", "m<=4096") in ROUTES
    assert ("qr", "complex_via_svd") in ROUTES
    assert any(k[:2] == ("svd", "groups") and k[2] in (2, 4) for k in ROUTES), ROUTES
