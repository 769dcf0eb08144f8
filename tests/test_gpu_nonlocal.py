"""GPU tier: multi-site, long-range and controlled gates as sub-MPOs
(``quimb_b200.nonlocal_gates``) and the 'auto-mps' / 'nonlocal' circuit
driver.

Checked against what the unmodified reference computed
(tests/golden/nonlocal.*: bond sizes, per-bond singular values, the dense
output and the orthogonality centre, all gauge-independent), against the
numpy oracle (oracle/nonlocal_np.py) at L = 40, chi = 128, and against the
uncompressed ``tebd.mpo_apply`` product of the same operator written as a
full-length MPO when nothing is truncated."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import mpo_compress_np as mnp
from oracle import nonlocal_np as onp
from quimb_b200 import nonlocal_gates as nl
from tests.conftest import load_golden
from tests.test_gpu_mpo_compress import overlap
from tests.test_gpu_mps_sample import rand_mps

pytestmark = pytest.mark.gpu

METHODS = ("direct", "dm", "zipup")

CX = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1], [0, 0, 1, 0]], dtype=float)
X = np.array([[0, 1], [1, 0]], dtype=float)
H = np.array([[1, 1], [1, -1]], dtype=float) / 2 ** 0.5
CCX = np.eye(8)
CCX[6:, 6:] = X


def rzz(theta):
    return np.diag(np.exp(-0.5j * theta * np.array([1, -1, -1, 1])))


def rand_unitary(n, dtype, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, n))
    if np.dtype(dtype).kind == "c":
        x = x + 1j * rng.standard_normal((n, n))
    q, r = np.linalg.qr(x)
    return (q * np.sign(np.diag(r))).astype(dtype)


# ----------------------------------------------------------------- helpers ---
def _np(x):
    return np.asarray(x.to_numpy() if hasattr(x, "to_numpy") else x)


def _dev(A):
    return [qb.asarray(a) for a in A]


def _kwargs(case):
    return {k: v for k, v in case.items()
            if k not in ("state", "gate", "where", "controls", "bonds", "cur_orthog")}


def _inputs(data, meta, case):
    L = meta["states"][case["state"]]["L"]
    A = [np.ascontiguousarray(data[f"{case['state']}__site{i}"]) for i in range(L)]
    return A, np.ascontiguousarray(data[f"gate__{case['gate']}"])


def check_golden_case(data, meta, case):
    A, G = _inputs(data, meta, case)
    k = meta["cases"].index(case)
    info = {}
    if case.get("controls"):
        out = qb.mps_gate_controlled(_dev(A), G, case["where"], case["controls"], info=info,
                                     **_kwargs(case))
    else:
        out = qb.mps_gate_nonlocal(_dev(A), G, case["where"], info=info, **_kwargs(case))
    got = [_np(x) for x in out]
    assert [x.shape[2] for x in got[:-1]] == case["bonds"]
    assert list(info["cur_orthog"]) == case["cur_orthog"]
    vec = data[f"case{k}__vec"]
    np.testing.assert_allclose(mnp.dense(got), vec, rtol=0, atol=1e-10 * np.max(np.abs(vec)))
    for i, s in enumerate(mnp.schmidt_values(got)):
        ref = data[f"case{k}__S{i}"]
        np.testing.assert_allclose(s, ref, rtol=0, atol=1e-10 * ref[0])


def circuit_gates(data, meta):
    out = []
    for k, e in enumerate(meta["circuit"]["gates"]):
        G = data[f"circ__gate{k}"]
        out.append((G, e["qubits"], e["controls"]) if e["controls"] else (G, e["qubits"]))
    return out


def zero_state(n):
    out = []
    for _ in range(n):
        x = np.zeros((1, 2, 1), dtype=np.complex128)
        x[0, 0, 0] = 1
        out.append(x)
    return out


class CutGaps:
    """The smallest relative gap s[n-1] - s[n] (over s[0]) at every truncating
    split the oracle makes, noise-level tails excepted."""

    def __init__(self):
        self.orig = mnp._split
        self.worst = np.inf

    def __enter__(self):
        mnp._split = self._split
        return self

    def __exit__(self, *exc):
        mnp._split = self.orig

    def _split(self, mat, method="svd", **kw):
        out = self.orig(mat, method=method, **kw)
        s = (np.sort(np.abs(np.linalg.eigvalsh(mat)))[::-1] if method == "eigh"
             else np.linalg.svd(mat, compute_uv=False))
        n = out[0].shape[1]
        if n < s.size and s[n] > 1e-12 * s[0]:
            self.worst = min(self.worst, (s[n - 1] - s[n]) / s[0])
        return out


def check_against_oracle(L, chi, G, where, dtype, method, seed, **kw):
    """The device result against the oracle at ``max_bond = chi``: equal
    bonds, Schmidt values to 1e-10 of the largest, normalised fidelity within
    1e-12 of 1.  Every truncating cut of the oracle lies in a relative gap of
    at least 1e-8, far from rounding."""
    A = rand_mps(L, chi, 2, dtype, seed)
    with CutGaps() as cuts:
        want, c = onp.gate_nonlocal(A, G, where, method=method, max_bond=chi, **kw)
    assert cuts.worst > 1e-8, cuts.worst
    info = {}
    out = qb.mps_gate_nonlocal(_dev(A), G, where, method=method, max_bond=chi, info=info,
                               **kw)
    assert info["cur_orthog"] == (c, c)
    got = [_np(x) for x in out]
    assert [x.shape[2] for x in got] == [x.shape[2] for x in want]
    for s, r in zip(mnp.schmidt_values(got), mnp.schmidt_values(want)):
        np.testing.assert_allclose(s, r, rtol=0, atol=1e-10 * r[0])
    f = abs(overlap(got, want)) ** 2 / (overlap(got, got).real * overlap(want, want).real)
    assert abs(f - 1) < 1e-12, f


def full_mpo(sub, present, L, d=2):
    """A sub-MPO on ``present`` (sorted) written as an (l, r, u, d) MPO on all
    L sites: identities elsewhere, bonds carried past the gaps."""
    out, k, D = [], 0, 1
    for s in range(L):
        if k < len(present) and s == present[k]:
            w = _np(sub[k])
            D = w.shape[1]
            k += 1
        else:
            w = np.einsum("ab,ud->abud", np.eye(D), np.eye(d)).astype(_np(sub[0]).dtype)
        out.append(np.ascontiguousarray(w))
    return out


# ------------------------------------------------------------------ tests ---
def test_golden_matches_reference():
    data, meta = load_golden("nonlocal")
    for case in meta["cases"]:
        check_golden_case(data, meta, case)


def test_circuit_matches_reference():
    """CircuitMPS (gate_contract='auto-mps') with Toffolis, a doubly
    controlled X, a controlled rotation and long-range CX gates."""
    data, meta = load_golden("nonlocal")
    c = meta["circuit"]
    sites = _dev(zero_state(c["N"]))
    qb.tebd.apply_circuit(sites, circuit_gates(data, meta), contract="auto-mps",
                          max_bond=c["max_bond"], cutoff=c["cutoff"])
    got = [_np(x) for x in sites]
    assert [x.shape[2] for x in got[:-1]] == c["bonds"]
    # The last Toffoli's 'direct' sweep canonicalises rank-deficient complex
    # product sites (condition up to 1e16), where the device complex QR takes
    # its SVD route; that route's vectors of close singular values are
    # orthonormal only to ~2e-7 (DESIGN 4.15), which bounds the agreement here.
    np.testing.assert_allclose(mnp.dense(got), data["circ__vec"], rtol=0, atol=1e-6)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_scale_two_site_long_range(method, dtype):
    check_against_oracle(40, 128, rand_unitary(4, dtype, 3), (27, 5), dtype, method, seed=7)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_scale_three_site(method, dtype):
    check_against_oracle(40, 128, rand_unitary(8, dtype, 4), (22, 9, 14), dtype, method,
                         seed=8)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("where", [(1, 5, 3), (6, 2), (0, 7)])
def test_untruncated_equals_mpo_apply(method, where):
    """cutoff = 0 and no max_bond: the uncompressed product of the same
    operator as a full-length MPO (``mpo_apply`` contracts the MPO's upper
    index, i.e. ``transpose=True`` here)."""
    L = 8
    A = rand_mps(L, 6, 2, np.complex128, 3)
    G = rand_unitary(2 ** len(where), np.complex128, 5)
    sub, present = qb.mpo_from_dense(G, 2, where)
    psi = _dev(A)
    full = qb.tebd.mpo_apply(_dev(full_mpo(sub, present, L)), psi)
    got = qb.mps_gate_with_submpo(psi, sub, where, method=method, cutoff=0.0, transpose=True)
    ff = qb.tebd.mps_overlap(full, full).real
    for x, y in ((got, full), (got, got)):
        assert abs(qb.tebd.mps_overlap(x, y) - ff) <= 1e-12 * ff


@pytest.mark.parametrize("name", ["CX", "RZZ", "CX_far", "C2X"])
def test_mpo_from_dense_is_unitary(name):
    """U U^dagger = 1 on the dense product of the MPO's sites."""
    if name == "C2X":
        mpo, sites = nl._controlled_mpo(X, (2,), [4], [0, 2], np.complex128,
                                        qb.asarray(np.zeros(1)).device)
        want_bonds = [2, 2]
    else:
        G = {"CX": CX, "RZZ": rzz(0.3), "CX_far": CX}[name]
        mpo, sites = qb.mpo_from_dense(G, 2, (5, 1) if name == "CX_far" else (0, 1))
        want_bonds = [2]
    W = [_np(w) for w in mpo]
    assert [w.shape[1] for w in W[:-1]] == want_bonds
    T = np.ones((1, 1, 1))
    for w in W:
        T = np.einsum("xal,lruv->xuavr", T, w).reshape(T.shape[0] * w.shape[2],
                                                      T.shape[1] * w.shape[3], w.shape[1])
    U = T[..., 0]
    np.testing.assert_allclose(U @ U.conj().T, np.eye(U.shape[0]), rtol=0, atol=1e-13)
    if name == "CX_far":
        # sites (5, 1): the gate's first index is site 5, the MPO's first site 1
        np.testing.assert_allclose(U, CX.reshape(2, 2, 2, 2).transpose(1, 0, 3, 2)
                                   .reshape(4, 4), atol=1e-13)
    if name == "C2X":
        want = np.eye(8)
        want[6:, 6:] = X
        np.testing.assert_allclose(U, want, atol=1e-13)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("sweep_reverse", [False, True])
def test_canonical_form_and_info(method, sweep_reverse):
    L = 10
    A = rand_mps(L, 8, 2, np.complex128, 5)
    where = (7, 2, 4)
    info = {}
    out = qb.mps_gate_nonlocal(_dev(A), rand_unitary(8, np.complex128, 6), where,
                               method=method, max_bond=6, sweep_reverse=sweep_reverse,
                               info=info)
    c = 7 if sweep_reverse else 2
    assert info["cur_orthog"] == (c, c)
    for i, x in enumerate(out):
        if i == c:
            continue
        x = _np(x)
        l, d, r = x.shape
        m = x.reshape(l * d, r) if i < c else x.reshape(l, d * r)
        g = m.conj().T @ m if i < c else m @ m.conj().T
        np.testing.assert_allclose(g, np.eye(g.shape[0]), rtol=0, atol=1e-12)
    assert tuple(qb.mps_calc_current_orthog_center(list(out))) == (c, c)


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
@pytest.mark.parametrize("method", METHODS)
def test_single_precision_keeps_dtype(dtype, method):
    L = 8
    A = rand_mps(L, 6, 2, dtype, 8)
    G = rand_unitary(8, dtype, 9)
    out = qb.mps_gate_nonlocal(_dev(A), G, (6, 1, 3), method=method, max_bond=6)
    assert all(x.dtype == np.dtype(dtype) for x in out)
    wide = np.complex128 if np.dtype(dtype).kind == "c" else np.float64
    want, _ = onp.gate_nonlocal([a.astype(wide) for a in A], G.astype(wide), (6, 1, 3),
                                method=method, max_bond=6)
    got = [_np(x).astype(wide) for x in out]
    f = abs(overlap(got, want)) ** 2 / (overlap(got, got).real * overlap(want, want).real)
    assert abs(f - 1) < 1e-4, f


@pytest.mark.parametrize("method", METHODS)
def test_inputs_unchanged(method):
    """The caller's list and arrays are left as they were; sites outside the
    canonicalised span are the caller's objects."""
    L = 9
    psi = _dev(rand_mps(L, 8, 2, np.complex128, 12))
    info = {}
    qb.mps_canonicalize(psi, 3, info)
    before = list(psi)
    A = [_np(x) for x in psi]
    out = qb.mps_gate_nonlocal(psi, rand_unitary(8, np.complex128, 13), (6, 3, 4),
                               method=method, max_bond=5, info=info)
    assert all(x is y for x, y in zip(psi, before))
    for x, a in zip(psi, A):
        assert np.array_equal(_np(x), a)
    for i in (0, 1, 2, 7, 8):
        assert out[i] is psi[i]
    for i in (3, 4, 5, 6):
        assert out[i] is not psi[i]


def test_apply_circuit_auto_mps_at_scale():
    """24 qubits: layers of rotations, Toffolis, doubly controlled gates and
    CNOTs spanning up to 23 sites, against the oracle driver."""
    rng = np.random.default_rng(21)
    N = 24
    gates = []
    for q in range(N):
        gates.append((H, (q,)))
    for layer in range(2):
        for q in range(N):
            th = rng.uniform(0, np.pi)
            gates.append((np.array([[np.cos(th / 2), -np.sin(th / 2)],
                                    [np.sin(th / 2), np.cos(th / 2)]]), (q,)))
        gates += [(CCX, (0, 11, 23)), (CX, (3, 20)), (CX, (22, 1)), (X, (12,), (2, 17)),
                  (CCX, (15, 5, 9)), (rzz(0.37), (4, 18)), (CX, (0, 23))]
    opts = dict(max_bond=32, cutoff=1e-10)
    with CutGaps() as cuts:
        want = onp.apply_circuit(zero_state(N), gates, contract="auto-mps", **opts)
    sites = _dev(zero_state(N))
    qb.tebd.apply_circuit(sites, gates, contract="auto-mps", **opts)
    got = [_np(x) for x in sites]
    assert [x.shape[2] for x in got] == [x.shape[2] for x in want]
    f = abs(overlap(got, want)) ** 2 / (overlap(got, got).real * overlap(want, want).real)
    assert abs(f - 1) < 1e-10, (f, cuts.worst)


@pytest.mark.parametrize("contract", ["auto-mps", "nonlocal"])
def test_apply_circuit_modes_agree_untruncated(contract):
    """Without truncation every contract mode gives the same state."""
    N = 7
    gates = [(H, (q,)) for q in range(N)] + [(CX, (0, 5)), (rzz(0.8), (6, 2)),
                                             (CX, (3, 4)), (H, (5,)), (CX, (1, 6))]
    base = _dev(zero_state(N))
    qb.tebd.apply_circuit(base, gates, cutoff=0.0)
    sites = _dev(zero_state(N))
    qb.tebd.apply_circuit(sites, gates, contract=contract, cutoff=0.0)
    v, u = mnp.dense([_np(x) for x in sites]), mnp.dense([_np(x) for x in base])
    np.testing.assert_allclose(v, u, rtol=0, atol=1e-12)


def test_argument_errors():
    L = 6
    psi = _dev(rand_mps(L, 4, 2, np.float64, 16))
    U4 = rand_unitary(4, np.float64, 1)
    mpo, _ = qb.mpo_from_dense(U4, 2, (1, 4))
    for m in ("zipup-first", "zipup-oversample"):
        with pytest.raises(NotImplementedError, match="KeyError"):
            qb.mps_gate_with_submpo(psi, mpo, (1, 4), method=m)
    for m in ("fit", "src", "srcmps", "sdc", "src-oversample", "lazy", "projector"):
        with pytest.raises(NotImplementedError, match=m):
            qb.mps_gate_nonlocal(psi, U4, (1, 4), method=m)
    with pytest.raises(ValueError):
        qb.mps_gate_nonlocal(psi, U4, (1, 4), method="nope")
    with pytest.raises(NotImplementedError):
        qb.mps_gate_with_submpo(psi, mpo, (1, 4), equalize_norms=True)
    with pytest.raises(TypeError, match="positive"):
        qb.mps_gate_with_submpo(psi, mpo, (1, 4), positive=1)
    with pytest.raises(ValueError):
        qb.mps_gate_with_submpo(psi, mpo, (1, 2, 4))          # one MPO site short
    with pytest.raises(ValueError):
        qb.mps_gate_nonlocal(psi, U4, (1, 1))                 # repeated site
    with pytest.raises(ValueError):
        qb.mps_gate_nonlocal(psi, U4, (1, 6))                 # out of range
    with pytest.raises(ValueError):
        qb.mpo_from_dense(np.eye(8), 2, (0, 1))               # size does not fit
    with pytest.raises(ValueError):
        qb.mps_gate_controlled(psi, X, (2,), (2, 3))          # target is a control
    with pytest.raises(ValueError):
        qb.tebd.apply_circuit(psi, [(CCX, (0, 2, 4))])        # default mode: two sites max
    with pytest.raises(ValueError):
        qb.tebd.apply_circuit(psi, [(X, (4,), (0,))])         # controls need auto-mps
    with pytest.raises(ValueError):
        qb.tebd.apply_circuit(psi, [(X, (4,))], contract="nope")
