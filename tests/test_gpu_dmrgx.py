"""GPU tier: DMRG-X (``quimb_b200.DMRGX``) and the <psi|H.H|psi>
environments it runs on (``mps.env2_*_step``, ``mps_expec2``, the bra-site
``norm_step`` / ``norm_step_right``).

Checked against what the unmodified reference computed (tests/golden/dmrgx.*:
pinned sweeps step by step, property runs by final energy, variance and
state) and against the numpy oracle (oracle/dmrgx_np.py)."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import dmrg_np as dm
from oracle import dmrgx_np as onp
from quimb_b200 import linalg, mps
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------- helpers ---
def _np(x):
    return np.asarray(x.to_numpy() if hasattr(x, "to_numpy") else x)


def _dev(xs):
    return [qb.asarray(np.ascontiguousarray(a)) for a in xs]


def rand_mps(L, chi, dtype, seed, d=2):
    rng = np.random.default_rng(seed)
    bonds = [1] + [min(chi, d ** i, d ** (L - i)) for i in range(1, L)] + [1]
    out = []
    for i in range(L):
        shape = (bonds[i], d, bonds[i + 1])
        x = rng.standard_normal(shape)
        if np.dtype(dtype).kind == "c":
            x = x + 1j * rng.standard_normal(shape)
        out.append((x / np.sqrt(bonds[i] * d)).astype(dtype))
    return out


def rand_fields(L, dh, seed):
    return list(np.random.default_rng(seed).uniform(-dh, dh, L))


def computational(bits, dtype="float64"):
    out = []
    for c in bits:
        a = np.zeros((1, 2, 1), dtype)
        a[0, int(c), 0] = 1.0
        out.append(a)
    return out


def case_inputs(data, case):
    name, L = case["name"], case["L"]
    mpo = [data[f"{name}__mpo{i}"] for i in range(L)]
    p0 = [data[f"{name}__p0_{i}"] for i in range(L)]
    return mpo, p0


def dense_state(sites):
    return onp.mps_dense([_np(s) for s in sites])


def fidelity(x, y):
    return abs(np.vdot(x, y)) ** 2 / (np.vdot(x, x).real * np.vdot(y, y).real)


def spectrum(fields, psi):
    """Eigenvalues of the MBL chain in the S^z sector of ``psi`` (H conserves
    total S^z; the sector is read off the largest amplitude)."""
    L = len(fields)
    nup = bin(int(np.argmax(np.abs(psi)))).count("1")
    basis = [s for s in range(2 ** L) if bin(s).count("1") == nup]
    index = {s: k for k, s in enumerate(basis)}
    H = np.zeros((len(basis), len(basis)))
    for k, s in enumerate(basis):
        bits = [(s >> (L - 1 - i)) & 1 for i in range(L)]     # site 0 = highest bit
        sz = [0.5 - b for b in bits]                           # |0> = up
        H[k, k] = sum(sz[i] * sz[i + 1] for i in range(L - 1)) + \
            sum(h * z for h, z in zip(fields, sz))
        for i in range(L - 1):
            if bits[i] != bits[i + 1]:
                t = s ^ (1 << (L - 1 - i)) ^ (1 << (L - 2 - i))
                H[index[t], k] += 0.5
    return np.linalg.eigvalsh(H)


def run_case(case, mpo, p0, dmrgx_cls=None):
    d = (dmrgx_cls or qb.DMRGX)(_dev(mpo), _dev(p0), case["chi"], seed=0)
    d.opts.update(case["opts"])
    run = case.get("sweeps") or case.get("run")
    if isinstance(run, dict):
        assert d.solve(**run)
    else:
        for direction, canonize in run:
            (d.sweep_right if direction == "R" else d.sweep_left)(canonize=canonize)
    return d


# ------------------------------------------------------------ environments ---
def check_env_steps(dtype, L=6, chi=8, seed=0):
    rng = np.random.default_rng(seed)
    fields = rand_fields(L, 4.0, seed)
    mpo = onp.mpo_mbl(fields)
    k = rand_mps(L, chi, dtype, seed + 1)
    b = rand_mps(L, chi // 2, dtype, seed + 2)
    i = L // 2
    A, B, W = k[i], b[i], mpo[i].astype(dtype)
    a, r = A.shape[0], A.shape[2]
    E2 = rng.standard_normal((a, 5, 5, a)).astype(dtype)
    E2r = rng.standard_normal((r, 5, 5, r)).astype(dtype)
    Eo = rng.standard_normal((B.shape[0], a)).astype(dtype)
    Eor = rng.standard_normal((B.shape[2], r)).astype(dtype)
    if np.dtype(dtype).kind == "c":
        E2 = E2 + 1j * rng.standard_normal(E2.shape)
        Eo = Eo + 1j * rng.standard_normal(Eo.shape)
    dA, dB, dW = qb.asarray(A), qb.asarray(B), qb.asarray(W)
    for got, ref in [
        (mps.env2_left_step(qb.asarray(E2), dA, dW), onp.env2_left(E2, A, W)),
        (mps.env2_right_step(qb.asarray(E2r), dA, dW), onp.env2_right(E2r, A, W)),
        (mps.norm_step(qb.asarray(Eo), dA, dB), onp.ovl_left(Eo, A, B)),
        (mps.norm_step_right(qb.asarray(Eor), dA, dB), onp.ovl_right(Eor, A, B)),
    ]:
        ref = np.asarray(ref)
        np.testing.assert_allclose(_np(got), ref, rtol=0, atol=1e-12 * np.max(np.abs(ref)))
    # the default bra is the ket: the existing norm steps are unchanged
    E = rng.standard_normal((a, a)).astype(dtype)
    np.testing.assert_allclose(_np(mps.norm_step(qb.asarray(E), dA)),
                               onp.ovl_left(E, A, A), rtol=0, atol=1e-12)
    # <H^2> of the whole chain
    got = mps.mps_expec2(_dev(k), _dev(mpo), shape="lpr").item()
    ref = onp.mps_expec2(k, mpo)
    assert abs(got - ref) <= 1e-12 * abs(ref)


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_env_steps_and_expec2(dtype):
    check_env_steps(dtype)


def check_expec2_golden():
    data, meta = load_golden("dmrgx")
    for case in meta["cases"]:
        if case["kind"] != "pinned":
            continue
        mpo, p0 = case_inputs(data, case)
        got = qb.mps_expec2(_dev(p0), _dev(mpo), shape="lpr").item()
        assert abs(got - case["en2_p0"]) <= 1e-11 * abs(case["en2_p0"]), case["name"]


def test_expec2_golden():
    check_expec2_golden()


def test_dmrg2_ground_state_variance():
    mpo = dm.mpo_heis(10)
    d = qb.DMRG2(mpo, [8, 16, 32], cutoffs=1e-12, mpo_shape="lrdu", seed=2)
    d.solve(tol=1e-11, max_sweeps=10)
    sites = d.state
    e = qb.mps_expec(sites, mpo, shape="lpr", mpo_shape="lrdu").item()
    e2 = qb.mps_expec2(sites, mpo, shape="lpr", mpo_shape="lrdu").item()
    assert abs(e - d.energy) < 1e-9
    assert e2 - e ** 2 < 1e-10


# --------------------------------------------------------------- dense Heff ---
def check_dense_heff(dtype, L=6, chi=8, seed=3):
    fields = rand_fields(L, 4.0, seed)
    mpo = onp.mpo_mbl(fields)
    k = rand_mps(L, chi, dtype, seed)
    i = L // 2
    W = [w.astype(dtype) for w in mpo]
    Lenv = np.ones((1, 1, 1), dtype)
    for j in range(i):
        Lenv = onp.env_left(Lenv, k[j], W[j])
    Renv = np.ones((1, 1, 1), dtype)
    for j in range(L - 1, i, -1):
        Renv = onp.env_right(Renv, k[j], W[j])
    d = qb.DMRGX(_dev(mpo), _dev(k), chi)
    d.lenv, d.renv = {i: qb.asarray(Lenv)}, {i: qb.asarray(Renv)}
    H = _np(d.dense_heff(i))
    ref = onp.dense_heff(Lenv, W[i], Renv)
    scale = np.max(np.abs(ref))
    np.testing.assert_allclose(H, ref, rtol=0, atol=1e-12 * scale)
    np.testing.assert_allclose(H, H.conj().T, rtol=0, atol=1e-12 * scale)


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_dense_heff(dtype):
    check_dense_heff(dtype)


# ------------------------------------------------------------ pinned cases ---
def check_pinned(name):
    data, meta = load_golden("dmrgx")
    case = next(c for c in meta["cases"] if c["name"] == name)
    mpo, p0 = case_inputs(data, case)
    d = run_case(case, mpo, p0)
    np.testing.assert_allclose(np.array(d.local_energies), data[f"{name}__local"],
                               rtol=0, atol=1e-10)
    np.testing.assert_allclose(np.array(d.total_energies), data[f"{name}__total"],
                               rtol=0, atol=1e-10)
    assert abs(d.energies[0] - case["energy0"]) < 1e-11
    assert fidelity(dense_state(d.state), data[f"{name}__state"]) > 1 - 1e-10
    assert d.state[0].dtype == np.dtype(case["dtype"])


PINNED = ["pin_real", "pin_wide", "pin_complex", "pin_thresh1"]
PROPERTY = ["explicit", "bigger", "thresh1", "partial", "complex"]


@pytest.mark.parametrize("name", PINNED)
def test_pinned(name):
    check_pinned(name)


# ---------------------------------------------------------- property cases ---
def check_property(name):
    data, meta = load_golden("dmrgx")
    case = next(c for c in meta["cases"] if c["name"] == name)
    mpo, p0 = case_inputs(data, case)
    d = run_case(case, mpo, p0)
    psi = dense_state(d.state)
    run = case["run"]
    energy = d.energy if isinstance(run, dict) else d.total_energies[-1][-1]
    variance = (d.variance if isinstance(run, dict) else
                qb.mps_expec2(d.state, d.ham, shape="lpr").item().real - energy ** 2)
    assert abs(energy - case["energy"]) < 1e-8
    assert variance < case["tol"]
    assert abs(np.vdot(psi, psi).real - 1.0) < 1e-10
    # a state of variance v lies within sqrt(v) of an eigenvalue: the window
    # is 1e-10 unless the reference itself stopped at a larger variance
    window = max(1e-10, np.sqrt(max(case["variance"], 0.0)))
    ev = spectrum(case["fields"], psi)
    assert np.sum(np.abs(ev - energy) < window) == 1
    # both runs stop once their variance is below tol, so two states of
    # variance v near one eigenstate may differ by O(v / gap^2): the bound is
    # 1e-8 unless the reference stopped at a variance above 1e-10
    assert fidelity(psi, data[f"{name}__state"]) > 1 - max(1e-8, 1e2 * case["variance"])
    assert d.state[0].dtype == np.dtype(case["dtype"])


@pytest.mark.parametrize("name", PROPERTY)
def test_property(name):
    check_property(name)


# ------------------------------------------------------------ larger chain ---
def test_large_chain_device_eigh(monkeypatch):
    """L = 24 from a computational state, bonds up to 32 (D = 2048): the local
    eigensolves run on the multi-group Jacobi route.  The oracle checks the
    result without a dense H: <H> and <H^2> of the final state, and one
    oracle local step (dense LAPACK eigh at D = 2048, overlap and variance
    selection) at the middle site, which must return the same eigenvalue."""
    routes = []
    inner = linalg.svd

    def svd(x, *a, **k):
        x = qb.asarray(x)
        routes.append(linalg.route_svd(x.shape, x.t.dtype))
        return inner(x, *a, **k)
    monkeypatch.setattr(linalg, "svd", svd)
    L = 24
    fields = rand_fields(L, 8.0, 24)
    mpo = onp.mpo_mbl(fields)
    p0 = computational("011010011010110100101101")
    d = qb.DMRGX(_dev(mpo), _dev(p0), 32)
    d.solve(tol=1e-10, sweep_sequence="R", max_sweeps=4)
    assert d.max_bond() == 32
    big = [r for r in routes if r["kernel_shape"] == (2048, 2048)]
    assert big and all(r["groups"] >= 2 and not r["complex_embed"] for r in big)

    k = [_np(a) for a in d.state]
    en, en2 = onp.mps_expec(k, mpo), onp.mps_expec2(k, mpo)
    assert abs(en - d.energy) < 1e-9
    assert abs((en2 - en ** 2) - d.variance) < 1e-9
    assert d.variance < 1e-8

    # one oracle step at the middle site, from the device's state
    i = L // 2
    for j in range(L - 1, i, -1):
        onp.right_canonize_site(k, j)
    assert k[i].shape[0] * k[i].shape[1] * k[i].shape[2] == 2048
    o = onp.DMRGX(mpo, k, 32)
    o.target, o.old = d.energy, list(k)
    E3, E4, E2 = np.ones((1, 1, 1)), np.ones((1, 1, 1, 1)), np.ones((1, 1))
    for j in range(i):
        E3 = onp.env_left(E3, k[j], mpo[j])
        E4 = onp.env2_left(E4, k[j], mpo[j])
        E2 = onp.ovl_left(E2, k[j], k[j])
    o.lenv, o.lenv2, o.lovl = {i: E3}, {i: E4}, {i: E2}
    E3, E4, E2 = np.ones((1, 1, 1)), np.ones((1, 1, 1, 1)), np.ones((1, 1))
    for j in range(L - 1, i, -1):
        E3 = onp.env_right(E3, k[j], mpo[j])
        E4 = onp.env2_right(E4, k[j], mpo[j])
        E2 = onp.ovl_right(E2, k[j], k[j])
    o.renv, o.renv2, o.rovl = {i: E3}, {i: E4}, {i: E2}
    loc, tot = o._update(i, "right")
    assert abs(loc - d.energy) < 1e-8
    assert abs(tot - d.energy) < 1e-8


# ------------------------------------------------------------------ errors ---
def check_errors():
    fields = rand_fields(6, 4.0, 1)
    mpo = onp.mpo_mbl(fields)
    p0 = computational("010101")
    with pytest.raises(NotImplementedError, match="bsz"):
        qb.DMRGX(_dev(mpo), _dev(p0), 4, bsz=2)
    full = onp.mpo_mbl(fields)
    W = np.zeros((5, 5, 2, 2))
    W[:, :, :, :] = full[1]
    cyc = [W.copy() for _ in range(6)]
    with pytest.raises(NotImplementedError, match="open-boundary"):
        qb.DMRGX(_dev(cyc), _dev(p0), 4)
    # a two-site state whose one bond makes D = 2 * 4097 at site 0
    rng = np.random.default_rng(4)
    big = [rng.standard_normal((1, 2, 4097)), rng.standard_normal((4097, 2, 1))]
    d = qb.DMRGX(_dev(onp.mpo_mbl([0.5, -0.5])), _dev(big), 4097)
    with pytest.raises(NotImplementedError, match="8192"):
        d.sweep_right(canonize=False)


def test_errors():
    check_errors()
