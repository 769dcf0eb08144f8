"""GPU tier: compressed contraction along a fixed sequence (SURVEY 8f rank 3)
against the values of the UNMODIFIED reference's
``_contract_compressed_tid_sequence`` (compress_mode='basic',
tree_gauge_distance=0) stored in tests/golden/compressed.* by
oracle/make_golden.py: four small networks (flat 2D real / complex, a PEPS
norm with multibonds, a random 3-regular graph), eight option sets each."""

import numpy as np
import pytest

import quimb_b200 as qb
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden_compressed():
    return load_golden("compressed")


@pytest.mark.parametrize("name", ["flat44", "flat53_c", "norm33", "reg10"])
def test_contract_compressed_matches_reference(golden_compressed, name):
    data, meta = golden_compressed
    m = meta[name]
    arrays = [data[f"{name}__t{k}"] for k in range(len(m["inputs"]))]
    exact = data[f"{name}__exact"]
    for run in m["runs"]:
        kw = dict(run["kw"])
        info = {}
        out = qb.contract_compressed([qb.asarray(a) for a in arrays], m["inputs"], m["output"],
                                     m["seq"], info=info, **kw)
        ref = data[run["key"]]
        got = out.to_numpy()
        assert got.shape == ref.shape
        scale = max(np.abs(ref).max(), 1e-300)
        # same sequence of truncations -> same value up to rounding (the SVD
        # gauge does not enter the contracted value)
        assert np.abs(got - ref).max() <= 1e-9 * scale, (name, kw)
        assert info["n_compress"] >= 0
    # a generous bond leaves the contraction exact
    out = qb.contract_compressed([qb.asarray(a) for a in arrays], m["inputs"], m["output"],
                                 m["seq"], max_bond=4096, cutoff=0.0)
    assert np.abs(out.to_numpy() - exact).max() <= 1e-10 * max(np.abs(exact).max(), 1e-300)


def test_contract_compressed_paths_and_errors(golden_compressed):
    data, meta = golden_compressed
    m = meta["flat44"]
    arrays = [qb.asarray(data[f"flat44__t{k}"]) for k in range(len(m["inputs"]))]
    n = len(arrays)
    # an SSA path describing the same sequence
    alias, ssa, nxt = {i: i for i in range(n)}, [], n
    for a, b in m["seq"]:
        ia = [k for k, v in alias.items() if v == a][-1]
        ib = [k for k, v in alias.items() if v == b][-1]
        ssa.append((ia, ib))
        alias = {k: v for k, v in alias.items() if v not in (a, b)}
        alias[nxt] = b
        nxt += 1
    seq = qb.path_to_sequence(ssa, n)
    assert [tuple(s) for s in seq] == [tuple(s) for s in m["seq"]]
    v1 = qb.contract_compressed(arrays, m["inputs"], m["output"], seq, max_bond=4, cutoff=0.0)
    mant, ex = qb.contract_compressed(arrays, m["inputs"], m["output"], seq, max_bond=4,
                                      cutoff=0.0, strip_exponent=True, equalize_norms=True)
    ref = data[meta["flat44"]["runs"][0]["key"]]
    assert abs(v1.item() - ref) <= 1e-9 * abs(ref)
    assert abs(mant.item() * 10.0 ** ex - ref) <= 1e-9 * abs(ref)
    with pytest.raises(NotImplementedError):
        qb.contract_compressed(arrays, m["inputs"], m["output"], seq, max_bond=4,
                               tree_gauge_distance=1)


@pytest.mark.parametrize("name", ["peps33_open", "peps34_open_c", "flat55", "reg12"])
def test_contract_compressed_rescaling_matches_reference(name):
    """tests/golden/compressed2.* (oracle/make_golden_compressed2.py): the
    reference divides tensors by their Frobenius norm, so with equalize_norms
    an absolute ('abs', 'sum2') cutoff keeps what that norm decides, and a
    stripped mantissa of an open output has unit Frobenius norm.  Every cut
    of these runs lies at a relative gap >= 1e-6, so the kept ranks and the
    value are the reference's to rounding."""
    data, meta = load_golden("compressed2")
    m = meta[name]
    arrays = [qb.asarray(data[f"{name}__t{k}"]) for k in range(len(m["inputs"]))]
    for run in m["runs"]:
        kw = dict(run["kw"])
        if "cutoff_mode" in kw:
            kw["compress_opts"] = {"cutoff_mode": kw.pop("cutoff_mode")}
        info = {}
        out = qb.contract_compressed(arrays, m["inputs"], m["output"], m["seq"], info=info, **kw)
        ref = data[run["key"]]
        assert (info["n_compress"], info["max_bond_seen"]) == (
            run["n_compress"], run["max_bond_seen"]), (name, kw)
        if run["exponent"] is not None:
            out, ex = out
            assert abs(ex - run["exponent"]) <= 1e-10, (name, kw, ex, run["exponent"])
        got = out.to_numpy()
        assert got.shape == ref.shape
        assert np.abs(got - ref).max() <= 1e-9 * np.abs(ref).max(), (name, kw)
