"""GPU tier: MPO application with compression, the variational fit,
successive compression and non-local gates (quimb_b200/mpo_compress.py,
fit.py, successive.py, nonlocal_gates.py) against their numpy oracles
(oracle/mpo_compress_np.py, fit_np.py, successive_np.py, nonlocal_np.py)
at bond dimensions of 256 to 1024.  At the chi = 128 of the per-module tests
these algorithms mostly run the 64x64 DMMA tile; here their contractions
reach the 128x128 tile (classic and stream-K launches, affine operand feeds)
and their splits the Jacobi SVD of matrices of thousands of rows.  Inputs
are random MPS (``rand_mps``: bonds min(chi, d^i, d^(L-i)) less a few) on
chains long enough that at least three consecutive bonds sit at chi, under
random MPOs of bond 5.

Tolerance rule.  A truncated compression is a deterministic function of its
input only while every kept rank is decided away from rounding.  Each case
records the singular values of every truncating SVD its oracle makes and
asserts that the relative gap (s[n-1] - s[n]) / s[0] at each kept rank n is
at least 1e-6 (the seeds are chosen so; tails below 1e-12 s[0] are rounding
and exempt).  'dm' cuts are eigenvalue cuts of reduced density matrices and
are held to ``check_dm_margin`` instead, the two-site fit's cuts also to
``fit_np.check_svd_margin``.  The device must then give identical bond
sizes, Schmidt values within 1e-9 s_0 of the oracle's at every bond and a
normalised fidelity within 1e-10 of 1.  Randomised methods get the oracle's
seed, and 'srcmps' the oracle's sampling MPS.

Every contraction, QR and SVD the cases launch is recorded by shape,
strides and dtype and mapped through the library's own route functions
(``route_pair``, ``schedule_pair``, ``feed_pair``, ``route_svd``,
``route_qr``).  Each case prints the large routes it reached;
``test_route_coverage`` (last in the module) pins their union, so a planner
change that moves these algorithms off the large tile fails here."""

import numpy as np
import pytest

import quimb_b200 as qb
from oracle import decomp_np as dnp
from oracle import fit_np as fnp
from oracle import mpo_compress_np as mnp
from oracle import nonlocal_np as nnp
from oracle import successive_np as snp
from quimb_b200 import _lib, linalg
from quimb_b200 import contract as qc
from quimb_b200 import fit as qfit
from quimb_b200 import mpo_compress, mps, ops, tebd, tree
from tests import decomp_oracle as do
from tests import route_oracle as ro
from tests.test_gpu_fit import full_mps
from tests.test_gpu_mpo_compress import check_dm_margin, overlap, rand_mpo
from tests.test_gpu_mps_sample import rand_mps
from tests.test_gpu_nonlocal import rand_unitary

pytestmark = pytest.mark.gpu

MIN_GAP = 1e-6
S_TOL = 1e-9
F_TOL = 1e-10
D_W = 5          # MPO bond
SVD_ROWS = 1000  # a Jacobi SVD this tall or taller counts as a large split


# ------------------------------------------------------------ route recorder --
ROUTES = {}      # test id -> set of route keys
_CONTRACT_USERS = (qc, ops, tree, tebd, mps, mpo_compress, qfit)


def _contract_key(a, la, b, lb, lc, kw):
    """(dtype, route, cfg, layout) as ``route_oracle.route_key``, with the
    stream-K schedule and, for the large real tile, the operand feeds."""
    ext = dict(zip(la, a.shape))
    ext.update(zip(lb, b.shape))
    out = kw.get("out")
    cs = list(out.shape) if out is not None else [ext[l] for l in lc]
    cst = list(out.stride()) if out is not None else ro.strides(cs)
    args = (list(a.shape), list(a.stride()), la, list(b.shape), list(b.stride()), lb,
            cs, [int(v) for v in cst], lc, _lib._TORCH2QB[a.dtype])
    ptrs = (a.data_ptr(), b.data_ptr(), out.data_ptr() if out is not None else 0x10000000)
    key = ro.route_key(str(a.dtype).split(".")[-1], qc.route_pair(*args, ptrs=ptrs))
    if key is None:
        return None
    if key[1] == "streamk":
        key += (qc.schedule_pair(*args, ptrs=ptrs),)
    if key[1] in ("plain", "streamk") and key[2] == 0 and key[3] >= 0:
        f = qc.feed_pair(*args, ptrs=ptrs)
        key += ("A:" + str(f["A"]), "B:" + str(f["B"]))
    return ("contract",) + key


def _svd_keys(route):
    keys = do.svd_keys_of(route)
    if route["kernel_shape"][0] >= SVD_ROWS:
        keys.append(("svd", f"rows>={SVD_ROWS}"))
    return keys


@pytest.fixture(autouse=True)
def _route_recorder(monkeypatch, request):
    seen = ROUTES.setdefault(request.node.name, set())
    inner_cp = qc.contract_pair

    def cp(a, la, b, lb, lc, *args, **kw):
        key = _contract_key(a, la, b, lb, lc, kw)
        if key is not None:
            seen.add(key)
        return inner_cp(a, la, b, lb, lc, *args, **kw)
    for mod in _CONTRACT_USERS:
        monkeypatch.setattr(mod, "contract_pair", cp)

    inner_qr, inner_svd, inner_trunc = linalg.qr, linalg.svd, linalg.svd_trunc

    def qr(x, *args, **kw):
        x = ops.asarray(x)
        seen.update(do.qr_keys_of(linalg.route_qr(x.shape, x.t.dtype)))
        return inner_qr(x, *args, **kw)

    def svd(x, *args, **kw):
        x = ops.asarray(x)
        seen.update(_svd_keys(linalg.route_svd(x.shape, x.t.dtype)))
        return inner_svd(x, *args, **kw)

    def svd_trunc(x, cutoff=-1.0, cutoff_mode=4, max_bond=-1, absorb=0, *args, **kw):
        x = ops.asarray(x)
        seen.update(_svd_keys(linalg.route_svd(x.shape, x.t.dtype, absorb)))
        return inner_trunc(x, cutoff, cutoff_mode, max_bond, absorb, *args, **kw)
    monkeypatch.setattr(linalg, "qr", qr)
    monkeypatch.setattr(linalg, "svd", svd)
    monkeypatch.setattr(linalg, "svd_trunc", svd_trunc)
    yield
    print(f"\n{request.node.name} large routes:", sorted(map(str, filter(_large, seen))))


def _large(key):
    """The routes this module is about: the 128x128 tile (cfg 0, any launch)
    and Jacobi SVDs of at least SVD_ROWS rows."""
    if key[0] == "contract":
        return key[2] in ("plain", "splitk", "streamk") and key[3] == 0
    return key == ("svd", f"rows>={SVD_ROWS}")


# ------------------------------------------------------------ oracle checks --
def _record_cuts(monkeypatch):
    """(singular values, kept rank) of every truncating SVD the oracles make."""
    cuts = []
    inner = dnp.svd_truncated

    def rec(x, *args, **kw):
        info = {}
        out = inner(x, *args, info=info, **kw)
        cuts.append((info["svals"], info["n_keep"]))
        return out
    monkeypatch.setattr(dnp, "svd_truncated", rec)
    return cuts


def min_cut_gap(cuts):
    """Smallest relative gap at a kept rank, rounding-level tails exempt."""
    gap = np.inf
    for s, n in cuts:
        if n < s.size and s[n] > 1e-12 * s[0]:
            gap = min(gap, (s[n - 1] - s[n]) / s[0])
    return gap


def _np(x):
    return np.asarray(x.to_numpy() if hasattr(x, "to_numpy") else x)


def _dev(xs):
    return [qb.asarray(x) for x in xs]


def check_result(out, want, cuts, what):
    """Identical bonds, Schmidt values to S_TOL s_0, fidelity within F_TOL of 1;
    every oracle cut at least MIN_GAP clear."""
    gap = min_cut_gap(cuts)
    assert gap >= MIN_GAP, (what, gap)
    got = [_np(x) for x in out]
    bonds = [x.shape[2] for x in want[:-1]]
    assert [x.shape[2] for x in got[:-1]] == bonds, what
    for i, (s, r) in enumerate(zip(mnp.schmidt_values(got), mnp.schmidt_values(want))):
        np.testing.assert_allclose(s, r, rtol=0, atol=S_TOL * r[0], err_msg=f"{what} bond {i}")
    f = abs(overlap(got, want)) ** 2 / (overlap(got, got).real * overlap(want, want).real)
    assert abs(f - 1) < F_TOL, (what, f)
    print(f"\n{what}: bonds up to {max(bonds)}, min cut gap {gap:.2e}, 1 - F = {1 - f:.1e}")


def _ladder(L, chi, d, dtype, seed):
    A = rand_mps(L, chi, d, dtype, seed)
    W = rand_mpo(L, D_W, d, dtype, seed + 1)
    return A, W


# ---------------------------------------------------------------- the cases --
# L = 2 log2(chi) + 2 puts three bonds of the d = 2 input at chi.
# (chi, dtype, method, seed)
GATE_CASES = [
    (256, "complex128", "direct", 7),
    (256, "complex128", "dm", 7),
    (256, "complex128", "zipup", 7),
    (256, "complex128", "zipup-first", 7),
    (512, "complex128", "zipup", 7),
    (512, "complex128", "dm", 7),
    (512, "float64", "direct", 8),
    (1024, "float64", "zipup", 7),
    (1024, "float64", "dm", 7),
]


def _chain(chi):
    return 2 * int(np.log2(chi)) + 2


@pytest.mark.parametrize("chi,dtype,method,seed", GATE_CASES,
                         ids=[f"{c[2]}-{c[1]}-chi{c[0]}" for c in GATE_CASES])
def test_gate_with_mpo(monkeypatch, chi, dtype, method, seed):
    A, W = _ladder(_chain(chi), chi, 2, dtype, seed)
    cuts = _record_cuts(monkeypatch)
    spectra = []
    want = mnp.gate_with_mpo(A, W, method=method, max_bond=chi,
                             spectra=spectra if method == "dm" else None)
    for w, nrm in spectra:
        check_dm_margin(w, nrm, chi, 1e-10)
    out = qb.mps_gate_with_mpo(_dev(A), _dev(W), method=method, max_bond=chi)
    check_result(out, want, cuts, f"{method} {dtype} chi={chi}")


@pytest.mark.parametrize("bsz", [1, 2])
def test_fit(monkeypatch, bsz):
    """Two-site from a random start of bond chi / 2, one-site from a guess at
    full bond; two sweeps.  The two-site fit's first sweep grows the bonds to
    chi, its second truncates (2 chi)-wide blocks back to chi."""
    chi, dtype, seed = 256, "complex128", 7
    L = _chain(chi)
    A, W = _ladder(L, chi, 2, dtype, seed)
    guess = None if bsz == 2 else full_mps(L, chi, 2, dtype, seed + 2)
    kw = dict(max_bond=chi, bsz=bsz, max_iterations=2, seed=seed + 3, cutoff=0.0,
              initial_bond_dim=chi // 2)
    cuts = _record_cuts(monkeypatch)
    spectra = []
    want = fnp.fit([(W, A)], guess=guess, spectra=spectra, **kw)
    for s, mb, cut, mode in spectra:
        fnp.check_svd_margin(s, mb, cut, mode)
    out = qb.mps_fit([(_dev(W), _dev(A))], guess=None if guess is None else _dev(guess), **kw)
    check_result(out, want, cuts, f"fit bsz={bsz} {dtype} chi={chi}")


SUCCESSIVE = ["src", "srcmps", "sdc", "src-oversample"]


@pytest.mark.parametrize("method", SUCCESSIVE)
def test_successive(monkeypatch, method):
    chi, dtype, seed = 256, "complex128", 7
    L = _chain(chi)
    A, W = _ladder(L, chi, 2, dtype, seed)
    F = None
    if method.startswith("srcmps"):
        k = chi if method == "srcmps" else qb.successive.oversample_bond(chi, None)
        F = qb.fit.random_guess_host([2] * L, k, dtype, seed + 2)
    cuts = _record_cuts(monkeypatch)
    want = snp.gate_with_mpo_successive(A, W, chi, method=method, seed=seed, tn_fit=F)
    out = qb.mps_gate_with_mpo_successive(_dev(A), _dev(W), chi, method=method, seed=seed,
                                          tn_fit=None if F is None else _dev(F))
    check_result(out, want, cuts, f"{method} {dtype} chi={chi}")


def test_nonlocal(monkeypatch):
    """A three-site gate spanning the chi-sized middle of the chain, zip-up
    over the sub-range ladder (gap sites carry the identity)."""
    chi, dtype, seed = 256, "complex128", 8
    L = _chain(chi)
    A = rand_mps(L, chi, 2, dtype, seed)
    G = rand_unitary(8, dtype, 4)
    where = (11, 6, 9)
    cuts = _record_cuts(monkeypatch)
    want, c = nnp.gate_nonlocal(A, G, where, method="zipup", max_bond=chi)
    info = {}
    out = qb.mps_gate_nonlocal(_dev(A), G, where, method="zipup", max_bond=chi, info=info)
    assert info["cur_orthog"] == (c, c)
    check_result(out, want, cuts, f"nonlocal zipup {dtype} chi={chi}")


# --------------------------------------------------------------- coverage --
# The large routes the cases above reach on an H100 SXM (132 SMs), as the
# recorder reported them: contraction keys are ("contract", dtype, launch,
# cfg, layout[, stream-K schedule][, A feed, B feed]), layout and feeds for
# real operands only.
PINNED = {
    ('contract', 'complex128', 'plain', 0, -1),
    ('contract', 'complex128', 'splitk', 0, -1),
    ('contract', 'complex128', 'streamk', 0, -1, 'pair'),
    ('contract', 'complex128', 'streamk', 0, -1, 'segments'),
    ('contract', 'float64', 'plain', 0, 0, 'A:affine', 'B:affine'),
    ('contract', 'float64', 'plain', 0, 0, 'A:affine', 'B:table'),
    ('contract', 'float64', 'plain', 0, 0, 'A:table', 'B:table'),
    ('contract', 'float64', 'plain', 0, 2, 'A:table', 'B:table'),
    ('contract', 'float64', 'splitk', 0, -1),
    ('contract', 'float64', 'streamk', 0, 0, 'pair', 'A:affine', 'B:affine'),
    ('contract', 'float64', 'streamk', 0, 0, 'pair', 'A:affine', 'B:table'),
    ('contract', 'float64', 'streamk', 0, 0, 'pair', 'A:table', 'B:table'),
    ('contract', 'float64', 'streamk', 0, 0, 'segments', 'A:affine', 'B:table'),
    ('contract', 'float64', 'streamk', 0, 0, 'segments', 'A:table', 'B:affine'),
    ('contract', 'float64', 'streamk', 0, 0, 'segments', 'A:table', 'B:table'),
    ('contract', 'float64', 'streamk', 0, 2, 'pair', 'A:affine', 'B:affine'),
    ('contract', 'float64', 'streamk', 0, 2, 'segments', 'A:affine', 'B:affine'),
    ('contract', 'float64', 'streamk', 0, 2, 'segments', 'A:affine', 'B:table'),
    ('contract', 'float64', 'streamk', 0, 2, 'segments', 'A:table', 'B:affine'),
    ('contract', 'float64', 'streamk', 0, 2, 'segments', 'A:table', 'B:table'),
    ('svd', 'rows>=1000'),
}


def test_route_coverage():
    """Needs the rest of the module to have run.  The union of the cases'
    routes includes the 128x128 tile's classic launch of real operands with
    both operands on the affine feed, its stream-K launch (segments and 2-CTA
    pair schedules) for both dtypes and a Jacobi SVD of at least SVD_ROWS
    rows, and its large part is exactly PINNED."""
    if not any(k for name, keys in ROUTES.items() if name != "test_route_coverage"
               for k in keys):
        pytest.skip("run with the rest of the module: the routes come from its cases")
    union = set().union(*ROUTES.values())
    print("\nall routes seen:", sorted(map(str, union)))
    large = set(filter(_large, union))
    print("large routes seen:", sorted(map(str, large)))
    r = qc.route_pair([8, 8], [8, 1], [0, 1], [8, 8], [8, 1], [1, 2], [8, 8], [8, 1], [0, 2])
    if r["sms"] != 132:
        pytest.skip(f"this device has {r['sms']} SMs; the pinned routes are for 132")
    assert ("contract", "float64", "plain", 0, 0, "A:affine", "B:affine") in large
    for dt in ("float64", "complex128"):
        for sched in ("segments", "pair"):
            assert any(k[1:3] == (dt, "streamk") and k[5] == sched for k in large), (dt, sched)
    assert ("svd", f"rows>={SVD_ROWS}") in large
    assert large == PINNED, (sorted(map(str, large - PINNED)), sorted(map(str, PINNED - large)))
