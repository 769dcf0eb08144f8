"""CPU tier of PEPS local expectations: the numpy oracle against what the
unmodified reference computed, the plaquette bookkeeping against the
reference's docstring answers, and the host layer (environments, the
reduced density matrices, descriptor packing of ``qb_plaquette_expec``) run
against a numpy emulation of the C ABI.  The raw-kernel tests need the device
and are not repeated here."""

import ctypes

import numpy as np
import pytest

from oracle import peps_expec_np as pe
from tests import test_gpu_peps_expec as gpu
from tests.abi_emulator import _NP, _addr, _flat, emulated_abi
from tests.conftest import load_golden
from tests.test_observables_cpu import _emulated_rdm_reduce
from quimb_b200 import _lib


def _emulated_plaquette_expec(emu, dtype, n, desc, desc_dev, rho, rho_elems, G, g_elems, out,
                              stream):
    """numpy version of qb_plaquette_expec (csrc/plaquette.cu), same contract."""
    if dtype not in (_lib.QB_F64, _lib.QB_C128):
        return emu._fail(-1, "qb_plaquette_expec: dtype must be QB_F64 or QB_C128")
    if n < 0:
        return emu._fail(-2, "qb_plaquette_expec: n_terms < 0")
    if n == 0:
        return 0
    align = 15 if dtype == _lib.QB_C128 else 7
    if any(not _addr(p) or _addr(p) & a for p, a in
           ((desc, 7), (desc_dev, 7), (rho, align), (G, align), (out, align))):
        return emu._fail(-4, "qb_plaquette_expec: null or misaligned pointer")
    table = _flat(desc, n * _lib.QB_PLAQ_DESC_WORDS, np.int64).reshape(n, -1)
    r = _flat(rho, rho_elems, _NP[dtype])
    g = _flat(G, g_elems, _NP[dtype])
    res = []
    for row in table:
        ro, go, ns, nt, p0, p1 = (int(v) for v in row[:6])
        dims = [int(v) for v in row[6:6 + ns]] if 1 <= ns <= 6 else []
        pos = (p0,) if nt == 1 else (p0, p1)
        D = int(np.prod(dims)) if dims else 0
        ok = dims and min(dims) >= 1 and D <= 64 and nt in (1, 2) and 0 <= p0 < ns
        ok = ok and (nt == 1 or p0 < p1 < ns)
        dg = int(np.prod([dims[s] for s in pos])) if ok else 0
        if not (ok and 0 <= ro <= rho_elems - D * D and 0 <= go <= g_elems - dg * dg):
            return emu._fail(-3, "qb_plaquette_expec: invalid descriptor")
        res.append(gpu._einsum_expec(r[ro:ro + D * D].reshape(D, D), dims,
                                     g[go:go + dg * dg].reshape(dg, dg), pos))
    emu._tick("qb_plaquette_expec")
    _flat(desc_dev, n * _lib.QB_PLAQ_DESC_WORDS, np.int64)[...] = table.ravel()
    _flat(out, 2 * n, _NP[dtype])[...] = np.array(res, dtype=_NP[dtype]).ravel()
    return 0


@pytest.fixture
def emulator():
    with emulated_abi() as emu:
        emu.qb_rdm_reduce = lambda *a: _emulated_rdm_reduce(emu, *a)
        emu.qb_rdm_workspace = emu._real.qb_rdm_workspace
        emu.qb_plaquette_expec = lambda *a: _emulated_plaquette_expec(emu, *a)
        yield emu


# ----------------------------------------------------------------- oracle ---
def test_oracle_matches_reference():
    data, meta = load_golden("peps_expec")
    for rec in meta["runs"]:
        st = meta["states"][rec["state"]]
        arrays, terms, keys = gpu.golden_state(data, meta, rec["state"])
        got, trace = pe.compute_local_expectation(arrays, terms, **rec["kw"])
        assert pe.min_gap(trace) == pytest.approx(rec["min_gap"], rel=1e-6, abs=1e-12)
        tol = gpu._ref_tol(st)
        if rec["kw"].get("return_all"):
            for where, (e, n) in zip(keys, rec["values"]):
                gpu._close(got[where][0], complex(*e), tol)
                if n is not None:
                    gpu._close(got[where][1], complex(*n), tol)
        else:
            gpu._close(got, complex(*rec["value"]), tol)


def test_oracle_dense_and_normalize():
    data, meta = load_golden("peps_expec")
    for name, st in meta["states"].items():
        arrays, terms, _ = gpu.golden_state(data, meta, name)
        wide = [[pe._widen(a) for a in row] for row in arrays]
        gpu._close(pe.dense_expectation(wide, terms), complex(*st["exact"]), 1e-5)
        gpu._close(pe.dense_expectation(wide, terms, True), complex(*st["exact_normalized"]),
                   1e-5)
        for rec in st["normalize"]:
            out, _ = pe.normalize(arrays, rec["max_bond"], cutoff=0.0)
            tol = gpu._ref_tol(st)
            for i, row in enumerate(out):
                for j, x in enumerate(row):
                    want = data[f"{name}__norm{rec['max_bond']}_site{i}_{j}"]
                    np.testing.assert_allclose(x, want, rtol=tol, atol=tol * np.abs(want).max())


# ------------------------------------------------------------ bookkeeping ---
def test_plaquette_sizes_docstring():
    import quimb_b200 as qb
    H2 = {}
    for i in range(10):
        for j in range(10):
            if j + 1 < 10:
                H2[(i, j), (i, j + 1)] = None
            if i + 1 < 10:
                H2[(i, j), (i + 1, j)] = None
    assert qb.calc_plaquette_sizes(H2.keys()) == ((1, 2), (2, 1))
    assert qb.calc_plaquette_sizes(H2.keys(), autogroup=False) == ((2, 2),)
    H2[(1, 1), (2, 2)] = None
    assert qb.calc_plaquette_sizes(H2.keys()) == ((2, 2),)
    H2[(1, 1), (1, 3)] = None
    H2[(1, 1), (3, 1)] = None
    assert qb.calc_plaquette_sizes(H2.keys()) == ((1, 3), (2, 2), (3, 1))
    assert qb.calc_plaquette_sizes(H2.keys(), autogroup=False) == ((3, 3),)
    assert qb.plaquette_to_sites([(3, 4), (2, 2)]) == ((3, 4), (3, 5), (4, 4), (4, 5))


def test_plaquette_map_docstring():
    import quimb_b200 as qb
    plaquettes = [((0, 0), (2, 2)), ((0, 0), (1, 2)), ((1, 0), (1, 2)),
                  ((0, 0), (2, 1)), ((0, 1), (2, 1))]
    got = qb.calc_plaquette_map(plaquettes)
    want = {((0, 0), (0, 1)): ((0, 0), (1, 2)),
            ((0, 0), (1, 0)): ((0, 0), (2, 1)),
            ((0, 0), (1, 1)): ((0, 0), (2, 2)),
            ((0, 1), (1, 0)): ((0, 0), (2, 2)),
            ((0, 1), (1, 1)): ((0, 1), (2, 1)),
            ((1, 0), (1, 1)): ((1, 0), (1, 2))}
    assert {k: v for k, v in got.items() if not pe.is_lone_coo(k)} == want
    assert got == pe.calc_plaquette_map(plaquettes)


# ------------------------------------------------------------- host layer ---
def test_emu_golden(emulator):
    gpu.test_golden_matches_reference()
    assert emulator.calls["qb_plaquette_expec"] == len(load_golden("peps_expec")[1]["runs"])
    assert emulator.calls["qb_rdm_reduce"] > 0


def test_emu_golden_normalize(emulator):
    gpu.test_golden_normalize()


def test_emu_dense_state(emulator):
    gpu.test_dense_state_without_truncation()


@pytest.mark.parametrize("fc", ["x", "y"])
def test_emu_matches_oracle(emulator, fc):
    gpu.check_against_oracle(4, 4, 2, 2, 5, np.complex128, 3, dict(field=0.3, nnn=0.5,
                                                                   long=0.2), fc)


def test_emu_complex_term_on_real_state(emulator):
    """A complex G on a real PEPS: its real and imaginary parts are two
    descriptors of the same launch."""
    import quimb_b200 as qb
    arrays = pe.rand_peps(3, 3, 2, 2, 9, np.float64)
    Y = pe.spin("Y")
    terms = {(1, 1): Y, ((0, 0), (0, 1)): np.kron(Y, pe.spin("X"))}
    dev = [[qb.asarray(a) for a in row] for row in arrays]
    n0 = emulator.calls["qb_plaquette_expec"]
    got = qb.peps_compute_local_expectation(dev, terms, 16, cutoff=0.0, return_all=True)
    want, _ = pe.compute_local_expectation(arrays, terms, 16, cutoff=0.0, return_all=True)
    assert emulator.calls["qb_plaquette_expec"] == n0 + 1
    for where in want:
        gpu._close(got[where][0], want[where][0], 1e-10)


def test_emu_one_launch_per_call(emulator):
    import quimb_b200 as qb
    arrays = pe.rand_peps(3, 4, 2, 2, 3, np.float64)
    terms = pe.heis_terms(3, 4, field=0.2, nnn=0.3)
    dev = [[qb.asarray(a) for a in row] for row in arrays]
    n0 = emulator.calls["qb_plaquette_expec"]
    qb.peps_compute_local_expectation(dev, terms, 8, normalized=True)
    assert emulator.calls["qb_plaquette_expec"] == n0 + 1


def test_emu_argument_errors(emulator):
    import quimb_b200 as qb
    arrays = [[qb.asarray(a) for a in row] for row in pe.rand_peps(3, 3, 2, 2, 1, np.float64)]
    h = pe.heis2()
    n0 = qb.launch_count()
    for bad in ({(3, 0): np.eye(2)}, {((0, 1), (0, 0)): h}, {((0, 0), (0, 1), (0, 2)): h},
                {((0, 0), (3, 0)): h}, {(0, -1): np.eye(2)}):
        with pytest.raises(KeyError):
            qb.peps_compute_local_expectation(arrays, bad, 4)
    for bad in ({(0, 0): np.ones((2, 3))}, {((0, 0), (0, 1)): np.eye(2)},
                {(0, 0): np.eye(3)}):
        with pytest.raises(ValueError):
            qb.peps_compute_local_expectation(arrays, bad, 4)
    d3 = [[qb.asarray(a) for a in row] for row in pe.rand_peps(3, 3, 2, 3, 1, np.float64)]
    with pytest.raises(NotImplementedError):
        qb.peps_compute_local_expectation(d3, {((0, 0), (1, 1)): np.eye(9)}, 4)
    with pytest.raises(NotImplementedError):
        qb.peps_compute_local_expectation(arrays, {(0, 0): np.eye(2)}, 4, mode="full-bond")
    with pytest.raises(NotImplementedError):
        qb.peps_compute_local_expectation(arrays, {(0, 0): np.eye(2)}, 4, equalize_norms=True)
    assert qb.launch_count() == n0


def test_emu_environments_leave_contractor_unchanged(emulator):
    """compute_environments works on a copy: the contractor's tensors and the
    earlier snapshots keep their contents through later sweeps."""
    import quimb_b200 as qb
    arrays = pe.rand_peps(4, 3, 2, 2, 2, np.float64)
    bc = qb.BoundaryContractor2D(*qb.peps_norm_tensors(
        [[qb.asarray(a) for a in row] for row in arrays]))

    def contents(sites):
        return {c: [(t.data.to_numpy().copy(), t.inds) for t in ts] for c, ts in sites.items()}

    def same(a, b):
        assert a.keys() == b.keys()
        for c in a:
            assert len(a[c]) == len(b[c])
            for (x, ix), (y, iy) in zip(a[c], b[c]):
                assert ix == iy and np.array_equal(x, y)

    before = contents(bc.sites)
    envs = bc.compute_x_environments(3, layer_tags=("KET", "BRA"))
    same(contents(bc.sites), before)
    assert envs["xmin", 0] == {} and envs["xmax", 3] == {}
    assert sorted(envs["xmin", 1]) == [(0, j) for j in range(3)]
    assert all(len(ts) == 2 for ts in envs["xmin", 1].values())
    assert sorted(envs["xmin", 3]) == [(2, j) for j in range(3)]
    snaps = {k: contents(v) for k, v in envs.items()}
    bc.compute_x_environments(3, layer_tags=("KET", "BRA"))
    bc.compute_plaquette_environments(2, 2, 3, layer_tags=("KET", "BRA"))
    for k, v in envs.items():
        same(contents(v), snaps[k])
    same(contents(bc.sites), before)
    dense = bc.compute_environments("ymin", dense=True)
    assert all(len(env) <= 1 for env in dense.values())


def test_emu_single_precision_rejects_before_widening(emulator):
    """Bad keys on a float32 PEPS raise before the widening launch."""
    import quimb_b200 as qb
    arrays = [[qb.asarray(a) for a in row]
              for row in pe.rand_peps(3, 3, 2, 2, 1, np.float32)]
    n0 = qb.launch_count()
    with pytest.raises(KeyError):
        qb.peps_compute_local_expectation(arrays, {((0, 1), (0, 0)): pe.heis2()}, 4)
    with pytest.raises(ValueError):
        qb.peps_compute_local_expectation(arrays, {(0, 0): np.eye(3)}, 4)
    assert qb.launch_count() == n0


def test_emu_normalize_rejects_nonpositive_real_norm(emulator, monkeypatch):
    import quimb_b200 as qb
    from quimb_b200 import peps_expec as px
    arrays = [[qb.asarray(a) for a in row] for row in pe.rand_peps(3, 3, 2, 2, 1, np.float64)]
    monkeypatch.setattr(px, "contract_boundary", lambda *a, **k: -0.5)
    with pytest.raises(ValueError):
        qb.peps_normalize(arrays, 4)


def test_emu_rejects_bad_dtype_in_kernel(emulator):
    arr = ctypes.c_int64 * 12
    assert emulator.qb_plaquette_expec(_lib.QB_F32, 1, arr(), 8, 8, 1, 8, 1, 8, None) == -1
