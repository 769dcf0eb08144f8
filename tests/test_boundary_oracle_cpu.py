"""CPU tier: the numpy restatements of boundary-MPS contraction
(oracle/boundary_np.py) and compressed contraction (oracle/compressed_np.py)
against every run of the unmodified reference stored in
tests/golden/boundary.*, compressed.* and compressed2.*.  The GPU tier holds
the device compositions to these oracles at sizes the fixtures cannot reach,
so the oracles must first reproduce the reference exactly where it ran."""

import numpy as np
import pytest

from oracle import boundary_np as bnp
from oracle import compressed_np as cnp
from tests.conftest import load_golden


def _tol(dtype):
    # the complex64 fixture is the reference's single-precision arithmetic;
    # the oracle widens on entry, as the device composition does
    return 2e-5 if "complex64" in dtype or "float32" in dtype else 1e-10


@pytest.mark.parametrize("name", ["peps44", "peps35", "peps53_c64", "flat55", "flat64"])
def test_boundary_oracle_matches_reference(golden_boundary, name):
    data, meta = golden_boundary
    m = meta[name]
    ts = [(data[f"{name}__t{k}"], r["inds"], tuple(r["site"]), r["layer"])
          for k, r in enumerate(m["tensors"])]
    tol = _tol(m["dtype"])
    assert len(m["runs"]) == 8
    for run in m["runs"]:
        v, bc = bnp.contract_boundary(ts, m["Lx"], m["Ly"], layer_tags=m["layers"], **run["kw"])
        ref = complex(*run["value"])
        assert abs(v - ref) <= tol * abs(ref), (name, run["kw"], v, ref)
        assert bc.n_compress > 0 and bc.trace
    exact = complex(*m["exact"])
    v, _ = bnp.contract_boundary(ts, m["Lx"], m["Ly"], layer_tags=m["layers"],
                                 max_bond=4096, cutoff=0.0)
    assert abs(v - exact) <= tol * abs(exact)


@pytest.mark.parametrize("name", ["flat44", "flat53_c", "norm33", "reg10"])
def test_compressed_oracle_matches_reference(name):
    data, meta = load_golden("compressed")
    m = meta[name]
    arrays = [data[f"{name}__t{k}"] for k in range(len(m["inputs"]))]
    assert [list(s) for s in cnp.greedy_sequence(arrays, m["inputs"], m["output"])] == m["seq"]
    assert len(m["runs"]) == 8
    for run in m["runs"]:
        v, info = cnp.contract_compressed(arrays, m["inputs"], m["output"], m["seq"], **run["kw"])
        ref = data[run["key"]]
        assert v.shape == ref.shape
        assert np.abs(v - ref).max() <= 1e-10 * np.abs(ref).max(), (name, run["kw"])
    exact = data[f"{name}__exact"]
    v, info = cnp.contract_compressed(arrays, m["inputs"], m["output"], m["seq"],
                                      max_bond=4096, cutoff=0.0)
    assert info["n_compress"] == 0
    assert np.abs(v - exact).max() <= 1e-10 * np.abs(exact).max()


@pytest.mark.parametrize("name", ["peps33_open", "peps34_open_c", "flat55", "reg12"])
def test_compressed_oracle_rescaling_matches_reference(name):
    data, meta = load_golden("compressed2")
    m = meta[name]
    arrays = [data[f"{name}__t{k}"] for k in range(len(m["inputs"]))]
    for run in m["runs"]:
        kw = dict(run["kw"])
        if "cutoff_mode" in kw:
            kw["compress_opts"] = {"cutoff_mode": kw.pop("cutoff_mode")}
        v, info = cnp.contract_compressed(arrays, m["inputs"], m["output"], m["seq"], **kw)
        if run["exponent"] is not None:
            v, ex = v
            assert abs(ex - run["exponent"]) <= 1e-10, (name, kw)
            assert abs(np.linalg.norm(v) - 1.0) <= 1e-12
        ref = data[run["key"]]
        assert np.abs(v - ref).max() <= 1e-10 * np.abs(ref).max(), (name, kw)
        assert [r["rank"] for r in info["trace"]] == run["ranks"]
        assert (info["n_compress"], info["max_bond_seen"]) == (
            run["n_compress"], run["max_bond_seen"])
        assert min([r["gap"] for r in info["trace"]] + [np.inf]) >= 1e-6
    # open outputs: the fixture pins strip_exponent where max-abs and Frobenius
    # scaling differ
    if m["output"]:
        strips = [r for r in m["runs"] if r["exponent"] is not None]
        assert strips and any(np.abs(data[r["key"]]).max() < 0.9 for r in strips)


def test_cut_gap_rule():
    s = np.array([4.0, 2.0, 1.0, 0.5])
    assert bnp.cut_gap(s, 2) == pytest.approx(0.25)
    assert bnp.cut_gap(s, 4) == np.inf
    # a relative cutoff right next to a singular value leaves no margin
    assert bnp.cut_gap(s, 2, cutoff=0.2501, cutoff_mode="rel") == pytest.approx(1e-4)
    assert bnp.cut_gap(s, 3, cutoff=0.6, cutoff_mode="abs") == pytest.approx(0.1 / 4)


def test_peps_norm_tensors_matches_reference_network(golden_boundary):
    """The oracle's PEPS norm network (conjugated bra layer) gives the
    reference's value of <psi|psi>."""
    data, meta = golden_boundary
    arrays = [[data[f"peps44_site__{i}_{j}"] for j in range(4)] for i in range(4)]
    ts, Lx, Ly = bnp.peps_norm_tensors(arrays)
    run = meta["peps44"]["runs"][0]
    v, _ = bnp.contract_boundary(ts, Lx, Ly, layer_tags=("KET", "BRA"), **run["kw"])
    ref = complex(*run["value"])
    assert abs(v - ref) <= 1e-10 * abs(ref)
