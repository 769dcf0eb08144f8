"""GPU tier: parity at the sizes BASELINE.json names (chi = 1024, d = 2,
w = 5) -- not through properties but against numpy / LAPACK on the same
inputs.  Each case costs a few seconds of host BLAS; together they pin the
"within 1e-10 fp64 of the reference path" target of the north star where the
bench and the DMRG sweep actually run.

  * the two GEMM shapes of the MPS-norm step (tn1d/core.py:502-557 through
    tensor_contract, tensor_core.py:224-358) and the DMRG  L . x  step
    (5120 x 1024 x 4096; tensor_core.py:12393-12417),
  * qb_svd on 2048 x 2048 and qb_qr_stab on 2048 x 1024 against LAPACK
    (decomp.py:1058-1118, :2198-2216),
  * one complete two-site update of DMRG2 at chi = 1024 (dmrg.py:803-870):
    matvec against the numpy restatement, the Lanczos eigenpair through its
    residual under the numpy operator, the truncated split against LAPACK's
    SVD + the reference's truncation rule, the environment step against numpy.
"""

import numpy as np
import pytest
import torch

import quimb_b200 as qb
from quimb_b200 import _lib
from oracle import decomp_np as dn
from oracle import dmrg_np as dm

pytestmark = pytest.mark.gpu


def _rel(out, ref):
    return float(np.abs(out - ref).max() / max(np.abs(ref).max(), 1e-300))


@pytest.mark.parametrize("case", ["norm_ket", "norm_bra", "dmrg_Lx"])
def test_contraction_at_baseline_shapes_vs_numpy(case):
    rng = np.random.default_rng(11)
    chi, d, w = 1024, 2, 5
    if case == "norm_ket":
        # T[a, p, b'] = sum_b E[a, b] A[b, p, b']        (1024 x 1024 x 2048)
        E = rng.standard_normal((chi, chi))
        A = rng.standard_normal((chi, d, chi))
        ref = np.tensordot(E, A, axes=((1,), (0,)))
        out = qb.tensordot(qb.asarray(E), qb.asarray(A), axes=((1,), (0,)))
    elif case == "norm_bra":
        # E'[a', b'] = sum_{a, p} A[a, p, a'] T[a, p, b']  (1024 x 2048 x 1024)
        A = rng.standard_normal((chi, d, chi))
        T = rng.standard_normal((chi, d, chi))
        ref = np.tensordot(A, T, axes=((0, 1), (0, 1)))
        out = qb.tensordot(qb.asarray(A), qb.asarray(T), axes=((0, 1), (0, 1)))
    else:
        # T1[a', w, s, t, b] = sum_a L[a', w, a] x[a, s, t, b]  (5120 x 1024 x 4096)
        L = rng.standard_normal((chi, w, chi))
        x = rng.standard_normal((chi, d, d, chi))
        ref = np.tensordot(L, x, axes=((2,), (0,)))
        out = qb.tensordot(qb.asarray(L), qb.asarray(x), axes=((2,), (0,)))
    assert out.shape == ref.shape
    assert _rel(out.to_numpy(), ref) < 1e-11


def test_svd_2048_vs_lapack():
    rng = np.random.default_rng(12)
    n = 2048
    x = rng.standard_normal((n, n))
    U, s, VH = (t.to_numpy() for t in qb.linalg.svd(qb.asarray(x)))
    s_ref = np.linalg.svd(x, compute_uv=False)
    assert np.abs(s - s_ref).max() < 1e-11 * s_ref[0]
    assert np.abs(U.T @ U - np.eye(n)).max() < 1e-11
    assert np.abs(VH @ VH.T - np.eye(n)).max() < 1e-11
    assert np.abs((U * s) @ VH - x).max() < 1e-10 * s_ref[0]


def test_qr_stab_2048x1024_vs_lapack():
    rng = np.random.default_rng(13)
    m, n = 2048, 1024
    x = rng.standard_normal((m, n))
    Q, _, R = qb.qr_stabilized(qb.asarray(x))
    q, r = Q.to_numpy(), R.to_numpy()
    qr_ref, _, rr_ref = dn.qr_stabilized(x)
    assert np.abs(q.T @ q - np.eye(n)).max() < 1e-12
    assert np.abs(q @ r - x).max() < 1e-11 * np.abs(x).max() * np.sqrt(n)
    assert np.all(np.diag(r) >= 0) and np.abs(np.tril(r, -1)).max() == 0.0
    # the stabilised factorisation is unique: compare factor by factor
    scale = np.abs(rr_ref).max()
    assert np.abs(r - rr_ref).max() < 1e-10 * scale
    assert np.abs(q - qr_ref).max() < 1e-9


def test_dmrg2_two_site_update_at_chi1024_vs_numpy():
    """One full-size update (a = b = 1024, d = 2, w = 5) of the Heisenberg
    chain: every arithmetic piece of dmrg.py:803-870 against numpy."""
    from quimb_b200.dmrg import EffHam2
    from quimb_b200.mps import env_left_step
    L, chi = 22, 1024
    mpo = dm.mpo_heis(L)
    d = qb.DMRG2(mpo, chi, cutoffs=0.0, mpo_shape="lrdu", seed=3)
    d.opts["local_eig_tol"] = 1e-3
    d.right_canonize()
    d._init_right_envs()
    d.lenv = {0: d._ones_env()}
    site = 10
    for i in range(site):
        if i > 0:
            d.lenv[i] = env_left_step(d.lenv[i - 1], d._k[i - 1], d.ham[i - 1])
        d._update_local_state(i, "right", max_bond=chi, cutoff=0.0)
    d.lenv[site] = env_left_step(d.lenv[site - 1], d._k[site - 1], d.ham[site - 1])
    A, B = d._k[site], d._k[site + 1]
    assert A.shape == (chi, 2, chi) and B.shape == (chi, 2, chi)
    dims = (chi, 2, 2, chi)
    H = EffHam2(d.lenv[site], d.ham[site], d.ham[site + 1], d.renv[site + 1], dims)
    Ln, Rn = d.lenv[site].to_numpy(), d.renv[site + 1].to_numpy()
    W1, W2 = d.ham[site].to_numpy(), d.ham[site + 1].to_numpy()   # (l, r, u, d)

    def matvec_np(v):
        x = v.reshape(dims)
        T = np.tensordot(Ln, x, axes=((2,), (0,)))                  # a' w s t b
        T = np.einsum("awstb,wvsp->avptb", T, W1, optimize=True)    # a' w1 s' t b
        T = np.einsum("avptb,vutq->aupqb", T, W2, optimize=True)    # a' w2 s' t' b
        return np.tensordot(T, Rn, axes=((1, 4), (1, 2))).reshape(-1)  # a' s' t' b'

    # (a) matvec
    rng = np.random.default_rng(14)
    v = rng.standard_normal(chi * 4 * chi)
    ref = matvec_np(v)
    out = H.matvec(qb.asarray(v)).to_numpy()
    assert _rel(out, ref) < 1e-11
    # (b) eigenpair of the local problem, tight tolerance, through its residual
    from quimb_b200.contract import contract_pair
    v0 = qb.Array(contract_pair(A.t, [0, 1, 9], B.t, [9, 2, 3], [0, 1, 2, 3]))
    d.opts["local_eig_tol"] = 1e-9
    theta, gs, info = d._eigs(H, v0.reshape(-1))
    g = gs.to_numpy().reshape(-1)
    Hg = matvec_np(g)
    assert abs(np.linalg.norm(g) - 1.0) < 1e-12
    assert abs(g @ Hg - theta) < 1e-10 * abs(theta)
    assert np.linalg.norm(Hg - theta * g) < 1e-6 * abs(theta)
    e0 = v0.to_numpy().reshape(-1)
    assert theta < (e0 @ matvec_np(e0)) / (e0 @ e0)
    # (c) truncated split of the optimised tensor, reference rule on LAPACK's SVD
    mat = g.reshape(2 * chi, 2 * chi)
    left, _, right = qb.array_split(qb.asarray(mat), method="svd", absorb="right",
                                    max_bond=chi, cutoff=0.0, cutoff_mode="sum2")
    l, r = left.to_numpy(), right.to_numpy()
    Ur, sr, Vr = np.linalg.svd(mat, full_matrices=False)
    assert l.shape == (2 * chi, chi) and r.shape == (chi, 2 * chi)
    assert np.abs(l.T @ l - np.eye(chi)).max() < 1e-11
    assert np.abs(np.linalg.norm(r, axis=1) - sr[:chi]).max() < 1e-11 * sr[0]
    assert np.abs(l @ r - (Ur[:, :chi] * sr[:chi]) @ Vr[:chi]).max() < 1e-10 * sr[0]
    # (d) environment step with the new left site
    Anew = qb.asarray(l.reshape(chi, 2, chi))
    E = env_left_step(d.lenv[site], Anew, d.ham[site]).to_numpy()
    An = l.reshape(chi, 2, chi)
    T = np.tensordot(Ln, An, axes=((2,), (0,)))                      # a' w p b
    T = np.einsum("awpb,wvpq->avqb", T, W1, optimize=True)           # a' w1 p' b
    Eref = np.tensordot(An, T, axes=((0, 1), (0, 2)))                # b' w1 b
    assert E.shape == Eref.shape
    assert _rel(E, Eref) < 1e-11


def test_cfg1_4096_cubed_default_dmma_and_int8_engine():
    """BASELINE configs[0] at full size: two rank-4 chi=64 tensors sharing two
    indices = a 4096^3 GEMM.  `engine=auto` runs float64 on the DMMA kernel
    (one launch, plus a reduce when split-K is chosen); the int8-split engine,
    requested explicitly, takes 5 launches (row maxima + split of each
    operand, GEMM).  Both at fp64 level against numpy."""
    rng = np.random.default_rng(15)
    a = rng.standard_normal((64, 64, 64, 64))
    b = rng.standard_normal((64, 64, 64, 64))
    A, B = qb.asarray(a), qb.asarray(b)
    ref = np.tensordot(a, b, axes=((2, 3), (0, 1)))
    n0 = qb.launch_count()
    out = qb.tensordot(A, B, axes=((2, 3), (0, 1)))
    assert qb.launch_count() - n0 <= 2
    assert _rel(out.to_numpy(), ref) < 1e-12
    n0 = qb.launch_count()
    out8 = qb.contract_pair(A.t, [0, 1, 2, 3], B.t, [2, 3, 4, 5], [0, 1, 4, 5],
                            engine=_lib.QB_ENGINE_OZAKI)
    assert qb.launch_count() - n0 == 5
    assert _rel(out8.cpu().numpy(), ref) < 1e-12
    # permuted operands (the index permutation is folded into the split gather)
    ref2 = np.tensordot(a.transpose(0, 2, 1, 3), b.transpose(3, 1, 2, 0), axes=((1, 3), (3, 2)))
    out2 = qb.tensordot(A.transpose(0, 2, 1, 3), B.transpose(3, 1, 2, 0), axes=((1, 3), (3, 2)))
    assert _rel(out2.to_numpy(), ref2) < 1e-12
    out28 = qb.contract_pair(A.t.permute(0, 2, 1, 3), [0, 1, 2, 3],
                             B.t.permute(3, 1, 2, 0), [4, 5, 3, 1], [0, 2, 4, 5],
                             engine=_lib.QB_ENGINE_OZAKI)
    assert _rel(out28.cpu().numpy(), ref2) < 1e-12
