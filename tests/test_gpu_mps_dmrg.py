"""GPU tier: MPS norm / expectation, device Lanczos and DMRG2 against the
oracle and the reference-generated golden values."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import dmrg_np as dm

pytestmark = pytest.mark.gpu


def _ref_sites(data, prefix, L):
    return [data[f"{prefix}__{i}"] for i in range(L)]


def test_mps_norm_expec_match_reference_golden(golden_mps):
    data, meta = golden_mps
    sites = _ref_sites(data, "mps12", 12)          # quimb layout 'lrp'
    n2 = qb.mps_norm2(sites, shape="lrp").item()
    assert n2 == pytest.approx(meta["mps12_norm2"], rel=1e-12)
    mpo = [np.asarray(data[f"heis6__{i}"]) for i in range(6)]
    # 12-site Heisenberg MPO from the reference's 6-site tensors (bulk is uniform)
    mpo12 = [mpo[0]] + [mpo[1]] * 10 + [mpo[5]]
    e = qb.mps_expec(sites, mpo12, shape="lrp", mpo_shape="lrud").item()
    assert e == pytest.approx(meta["mps12_expec_heis"], rel=1e-11)
    csites = _ref_sites(data, "cmps8", 8)
    n2c = qb.mps_norm2(csites, shape="lrp").item()
    assert np.real(n2c) == pytest.approx(meta["cmps8_norm2"], rel=1e-12)
    assert abs(np.imag(n2c)) < 1e-12 * abs(n2c)
    mpo8 = [mpo[0]] + [mpo[1]] * 6 + [mpo[5]]
    ec = qb.mps_expec(csites, mpo8, shape="lrp").item()
    assert np.real(ec) == pytest.approx(meta["cmps8_expec_heis"], rel=1e-11)


@pytest.mark.parametrize("L,chi", [(10, 16), (30, 64)])
def test_mps_norm_vs_oracle(L, chi):
    sites = dm.mps_rand(L, chi, seed=L)
    ref = dm.mps_norm2(sites)
    out = qb.mps_norm2(sites, shape="lpr").item()
    assert out == pytest.approx(ref, rel=1e-12)
    mpo = dm.mpo_heis(L)
    # oracle MPO layout W[wl, wr, pu(bra), pd(ket)] -> 'lrdu'
    e = qb.mps_expec(sites, mpo, shape="lpr", mpo_shape="lrdu").item()
    assert e == pytest.approx(dm.mps_expec(sites, mpo), rel=1e-11)


def test_env_steps_vs_oracle():
    rng = np.random.default_rng(0)
    E = rng.standard_normal((6, 5, 6)); A = rng.standard_normal((6, 2, 7))
    W = rng.standard_normal((5, 4, 2, 2))
    ref = dm.env_step_left(E, A, W)
    Wq = np.transpose(W, (0, 1, 3, 2))             # -> (l, r, u=ket, d=bra)
    out = qb.env_left_step(qb.asarray(E), qb.asarray(A), qb.asarray(Wq))
    np.testing.assert_allclose(out.to_numpy(), ref, atol=1e-12)
    E2 = rng.standard_normal((7, 4, 7))
    ref = dm.env_step_right(E2, A, W)
    out = qb.env_right_step(qb.asarray(E2), qb.asarray(A), qb.asarray(Wq))
    np.testing.assert_allclose(out.to_numpy(), ref, atol=1e-12)


def test_effective_hamiltonian_matvec_vs_oracle():
    from quimb_b200.dmrg import EffHam2
    rng = np.random.default_rng(1)
    a, s, t, b, w = 9, 2, 2, 8, 5
    L = rng.standard_normal((a, w, a)); R = rng.standard_normal((b, w, b))
    W1 = rng.standard_normal((w, w, 2, 2)); W2 = rng.standard_normal((w, w, 2, 2))
    x = rng.standard_normal(a * s * t * b)
    ref = dm.EffHam2(L, W1, W2, R, (a, s, t, b))._matvec(x)
    tq = lambda W: qb.asarray(np.transpose(W, (0, 1, 3, 2)))  # noqa: E731
    H = EffHam2(qb.asarray(L), tq(W1), tq(W2), qb.asarray(R), (a, s, t, b))
    out = H.matvec(qb.asarray(x))
    np.testing.assert_allclose(out.to_numpy(), ref, rtol=1e-12, atol=1e-11)


def test_lanczos_vs_dense():
    rng = np.random.default_rng(2)
    n = 600
    M = rng.standard_normal((n, n)); M = 0.5 * (M + M.T)
    Md = qb.asarray(M)
    mv = lambda v: qb.tensordot(Md, v, axes=1)  # noqa: E731
    v0 = qb.asarray(rng.standard_normal(n))
    theta, x, info = qb.eigh_lanczos(mv, v0, ncv=20, tol=1e-10, return_info=True)
    w = np.linalg.eigvalsh(M)
    assert theta == pytest.approx(w[0], abs=1e-8)
    xv = x.to_numpy()
    assert np.linalg.norm(M @ xv - theta * xv) < 1e-6
    assert abs(np.linalg.norm(xv) - 1) < 1e-12
    thi, _ = qb.eigh_lanczos(mv, v0, which="LA", ncv=20, tol=1e-10)
    assert thi == pytest.approx(w[-1], abs=1e-8)
    # tiny problems: the Krylov space is the whole space
    M4 = M[:4, :4]
    th4, _ = qb.eigh_lanczos(lambda v: qb.tensordot(qb.asarray(M4), v, axes=1),
                             qb.asarray(np.ones(4)), ncv=4, tol=1e-12)
    assert th4 == pytest.approx(np.linalg.eigvalsh(M4)[0], abs=1e-10)


def test_dmrg2_energies_match_reference_golden(golden_mps):
    _, meta = golden_mps
    run = meta["dmrg2_runs"][0]                      # L = 10, exact known
    mpo = dm.mpo_heis(run["L"])
    d = qb.DMRG2(mpo, run["bond_dims"], cutoffs=run["cutoffs"], mpo_shape="lrdu", seed=3)
    d.solve(tol=run["tol"], max_sweeps=8)
    assert d.energy == pytest.approx(run["exact"], abs=1e-7)
    assert d.energy == pytest.approx(run["energies"][-1], abs=1e-6)
    # state is normalised and right/left canonical pieces are isometries
    n2 = qb.mps_norm2(d.state, shape="lpr").item()
    assert n2 == pytest.approx(1.0, abs=1e-10)


def test_dmrg2_L20_vs_reference_and_oracle(golden_mps):
    _, meta = golden_mps
    run = meta["dmrg2_runs"][1]
    mpo = dm.mpo_heis(run["L"])
    d = qb.DMRG2(mpo, run["bond_dims"], cutoffs=run["cutoffs"], mpo_shape="lrdu", seed=5)
    d.solve(tol=run["tol"], max_sweeps=8)
    assert d.energy == pytest.approx(run["energies"][-1], abs=20 * run["tol"])
    o = dm.DMRG2(mpo, run["bond_dims"], cutoffs=run["cutoffs"], seed=5)
    o.solve(tol=run["tol"], max_sweeps=8)
    assert d.energy == pytest.approx(o.energy, abs=20 * run["tol"])
    assert d.max_bond() <= run["bond_dims"][-1]


def test_dmrg2_parity_mode_arpack_driver():
    mpo = dm.mpo_heis(8)
    d = qb.DMRG2(mpo, [8, 16], cutoffs=1e-10, mpo_shape="lrdu", seed=1)
    d.opts["local_eig_backend"] = "SCIPY"
    d.solve(tol=1e-8, max_sweeps=6)
    H = dm.mpo_to_dense(mpo)
    assert d.energy == pytest.approx(np.linalg.eigvalsh(H)[0], abs=1e-7)


def test_dmrg2_complex128_dtype_preserved():
    """dtype preservation (reference: test_dmrg.py:290-300): a complex state
    stays complex, the energy is the real ground-state energy."""
    mpo = dm.mpo_heis(8)
    d = qb.DMRG2(mpo, [8, 16], cutoffs=1e-10, mpo_shape="lrdu", seed=4, dtype="complex128")
    d.solve(tol=1e-8, max_sweeps=6)
    assert all(a.dtype == np.complex128 for a in d.state)
    e0 = np.linalg.eigvalsh(dm.mpo_to_dense(mpo))[0]
    assert d.energy == pytest.approx(e0, abs=1e-7)


def test_lanczos_complex_hermitian():
    rng = np.random.default_rng(7)
    n = 300
    M = rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n)); M = 0.5 * (M + M.conj().T)
    Md = qb.asarray(M)
    theta, x = qb.eigh_lanczos(lambda v: qb.tensordot(Md, v, axes=1),
                               qb.asarray(rng.standard_normal(n) + 1j * rng.standard_normal(n)),
                               ncv=16, tol=1e-10)
    assert theta == pytest.approx(np.linalg.eigvalsh(M)[0], abs=1e-8)
    xv = x.to_numpy()
    assert np.linalg.norm(M @ xv - theta * xv) < 1e-6


@pytest.mark.parametrize("dtype,exchange", [("float64", "auto"), ("complex128", "auto"),
                                            ("float64", "p2p")],
                         ids=["float64", "complex128", "float64-p2p"])
def test_bond_sharded_eigensolve_two_ranks_one_gpu(dtype, exchange):
    """SURVEY 8e: the local eigensolve row-sharded over 2 ranks (both on this
    GPU) reproduces the unsharded DMRG2 and exact diagonalisation; replicated
    parts stay bit-identical.  'auto' stages the gloo collectives through the
    host; 'p2p' runs the float64 gathers and reductions in the peer-memory
    kernels over CUDA IPC (other dtypes never take them)."""
    import time

    from tests.test_gpu_p2p import run_process_group, torchrun_cmd
    t0 = time.time()
    rc, out, err = run_process_group(
        torchrun_cmd("dist_dmrg_worker.py", 2, "--backend", "gloo", "--same-gpu",
                     "--dtype", dtype, "--exchange", exchange), timeout=300)
    print(f"sharded DMRG2 ({dtype}, {exchange}): {time.time() - t0:.1f} s wall")
    assert rc == 0 and "DIST_DMRG_OK" in out, out[-2000:] + err[-2000:]


def test_environments_and_moving_environment_vs_oracle():
    L, chi = 9, 6
    sites = dm.mps_rand(L, chi, seed=11)
    mpo = dm.mpo_heis(L)
    dev = [qb.asarray(s) for s in sites]
    H = [qb.asarray(w) for w in mpo]
    # norm environments: <psi|psi> from any cut
    le = qb.compute_left_environments(dev, shape="lpr")
    re = qb.compute_right_environments(dev, shape="lpr")
    assert sorted(le) == list(range(1, L)) and sorted(re) == list(range(0, L - 1))
    n2 = dm.mps_norm2(sites)
    for i in range(1, L - 1):
        # <psi|psi> = sum L_i[a', a] conj(A_i)[a', p, b'] A_i[a, p, b] R_i[b', b]
        A = sites[i]
        val = np.einsum("xa,xpy,apb,yb->", le[i].to_numpy(), A.conj(), A, re[i].to_numpy(),
                        optimize=True)
        assert abs(val - n2) <= 1e-11 * abs(n2)
    # energy environments against the oracle's step functions
    leh = qb.compute_left_environments(dev, H, shape="lpr", mpo_shape="lrdu")
    E = np.ones((1, 1, 1))
    for i in range(L - 1):
        E = dm.env_step_left(E, sites[i], mpo[i])
        np.testing.assert_allclose(leh[i + 1].to_numpy(), E, rtol=1e-11, atol=1e-12)
    reh = qb.compute_right_environments(dev, H, shape="lpr", mpo_shape="lrdu")
    E = np.ones((1, 1, 1))
    for i in range(L - 1, 0, -1):
        E = dm.env_step_right(E, sites[i], mpo[i])
        np.testing.assert_allclose(reh[i - 1].to_numpy(), E, rtol=1e-11, atol=1e-12)
    # moving window: every position reproduces <psi|H|psi>
    from quimb_b200.mps import mpo_lrud
    Hl = [mpo_lrud(w, "lrdu", i, L) for i, w in enumerate(H)]
    expec = dm.mps_expec(sites, mpo)
    for begin in ("left", "right"):
        me = qb.MovingEnvironment(dev, Hl, begin=begin, bsz=2)
        order = list(range(L - 1)) if begin == "left" else list(range(L - 2, -1, -1))
        for i in order + order[::-1]:
            me.move_to(i)
            Le, Re = (t.to_numpy() for t in me())
            A, B = sites[i], sites[i + 1]
            # oracle MPO layout is (l, r, bra, ket)
            val = np.einsum("xwa,apm,mqb,wvPp,vuQq,xPn,nQy,yub->", Le, A, B, mpo[i],
                            mpo[i + 1], A.conj(), B.conj(), Re, optimize=True)
            assert abs(val - expec) <= 1e-10 * abs(expec), (begin, i)


@pytest.mark.parametrize("ncv", [2, 3, 4, 8, 20, 64])
def test_lanczos_thick_restart_all_basis_sizes(ncv):
    """Thick-restart Lanczos with per-step residual monitoring: every basis
    size converges to the dense answer ('SA' and 'LA'), clustered spectra
    included; the residual reported is the true |H x - theta x|."""
    rng = np.random.default_rng(ncv)
    n = 400
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    # close (but, for the 2- and 3-vector bases, not pathological) low cluster
    low = [-5.0, -4.999, -4.99] if ncv >= 8 else [-5.0, -4.5, -4.2]
    lam = np.concatenate([low, np.linspace(-4, 6, n - 3)])
    H = (q * lam) @ q.T
    Hd = qb.asarray(H)
    count = [0]

    def mv(v):
        count[0] += 1
        return qb.tensordot(Hd, v, axes=((1,), (0,)))

    v0 = qb.asarray(rng.standard_normal(n))
    for which, ref in (("SA", lam.min()), ("LA", lam.max())):
        count[0] = 0
        theta, x, info = qb.eigh_lanczos(mv, v0, which=which, ncv=ncv, tol=1e-9,
                                         maxiter=4000, return_info=True)
        assert info["converged"] and info["nmatvec"] == count[0]
        assert abs(theta - ref) < 1e-8, (which, ncv, theta, ref)
        xv = x.to_numpy()
        assert abs(np.linalg.norm(xv) - 1) < 1e-12
        assert np.linalg.norm(H @ xv - theta * xv) <= 2e-9 * max(1, abs(theta))
    # a converged start vector stops after the ARPACK-like minimum of matvecs
    count[0] = 0
    theta, x, info = qb.eigh_lanczos(mv, qb.asarray(q[:, 0].copy()), ncv=max(ncv, 4), tol=1e-6,
                                     return_info=True)
    assert abs(theta - lam[0]) < 1e-9 and info["nmatvec"] <= 4


@pytest.mark.parametrize("method,tol", [("svd:eig", 1e-8), ("svd:rand", 1e-5)])
def test_dmrg2_other_bond_compress_methods(method, tol):
    """bond_compress_method (dmrg.py:84-102 opts): the Gram-matrix SVD gives
    the same energies as the Jacobi SVD; the randomized range finder is an
    approximation near the cut (GEMM-bound alternative at large chi)."""
    mpo = dm.mpo_heis(14)
    ref = qb.DMRG2(mpo, [8, 16, 32], cutoffs=1e-10, mpo_shape="lrdu", seed=2)
    ref.solve(tol=1e-7, max_sweeps=8)
    d = qb.DMRG2(mpo, [8, 16, 32], cutoffs=1e-10, mpo_shape="lrdu", seed=2)
    d.opts["bond_compress_method"] = method
    d.solve(tol=1e-7, max_sweeps=8)
    assert abs(d.energy - ref.energy) < tol * abs(ref.energy)
    with pytest.raises(ValueError):
        d.opts["bond_compress_method"] = "cholesky"
        d.sweep("R", max_bond=8, cutoff=0.0, method="cholesky")


def test_dmrg1_matches_reference_and_oracle(golden_mps):
    """One-site DMRG (quimb's DMRG1): energies of the reference's own runs
    (tests/golden/mps_dmrg.json: dmrg1_runs), the numpy oracle and exact
    diagonalisation; bonds grow only through expand_bond_dimension."""
    from quimb_b200.dmrg import DMRG1
    _, meta = golden_mps
    for r in meta["dmrg1_runs"]:
        mpo = dm.mpo_heis(r["L"])
        d = DMRG1(mpo, r["bond_dims"], cutoffs=1e-10, mpo_shape="lrdu", seed=1)
        assert d.solve(tol=r["tol"], max_sweeps=12)
        assert abs(d.energy - r["energies"][-1]) < 50 * r["tol"]
        assert abs(d.energy - r["exact"]) < 1e-6
        assert d.max_bond() <= r["bond_dims"][-1]
        o = dm.DMRG1(mpo, r["bond_dims"], cutoffs=1e-10, seed=1)
        o.solve(tol=r["tol"], max_sweeps=12)
        assert abs(d.energy - o.energy) < 50 * r["tol"]
    # complex dtype is preserved, sweeps in both directions
    mpo = dm.mpo_heis(8)
    d = DMRG1(mpo, [4, 8, 16], cutoffs=1e-10, mpo_shape="lrdu", seed=3, dtype="complex128")
    d.solve(tol=1e-8, max_sweeps=10, sweep_sequence="RL")
    assert d.state[0].dtype == np.complex128
    assert abs(d.energy - np.linalg.eigvalsh(dm.mpo_to_dense(mpo))[0]) < 1e-7


def test_chain_plans_replay_as_cuda_graphs():
    """Norm, expectation and the environment chain as persistent device plans
    (SURVEY 8f rank 2): captured once, replayed with new site data, zero
    host-side launches per replay, values equal to the eager path / oracle."""
    L, chi = 14, 24
    mpo = dm.mpo_heis(L)
    s1 = dm.mps_rand(L, chi, seed=4)
    s2 = dm.mps_rand(L, chi, seed=5)
    plan_n = qb.ChainPlan(s1, shape="lpr", kind="norm")
    plan_e = qb.ChainPlan(s1, mpo, shape="lpr", mpo_shape="lrdu", kind="expec")
    plan_r = qb.ChainPlan(s1, mpo, shape="lpr", mpo_shape="lrdu", kind="right_envs")
    plan_l = qb.ChainPlan(s1, shape="lpr", kind="left_envs")
    for sites in (s1, s2):
        dev = [qb.asarray(a) for a in sites]
        n0 = qb.launch_count()
        n2 = plan_n(dev).item()
        ex = plan_e(dev).item()
        envs = plan_r(dev)
        lenv = plan_l(dev)
        assert qb.launch_count() == n0          # graph replays only
        assert abs(n2 - dm.mps_norm2(sites)) <= 1e-11 * abs(n2)
        assert abs(ex - dm.mps_expec(sites, mpo)) <= 1e-10 * max(1.0, abs(ex))
        eager = qb.compute_right_environments(dev, [qb.asarray(w) for w in mpo], "lpr", "lrdu")
        for k, E in eager.items():
            np.testing.assert_allclose(envs[k].to_numpy(), E.to_numpy(), rtol=1e-12, atol=1e-13)
        eager_l = qb.compute_left_environments(dev, None, "lpr")
        for k, E in eager_l.items():
            np.testing.assert_allclose(lenv[k].to_numpy(), E.to_numpy(), rtol=1e-12, atol=1e-13)
    with pytest.raises(ValueError):
        plan_n.update(3, np.zeros((2, 2, 2)))
