"""Oracles of the decomposition tests (QR, SVD, truncated SVD, eigh).

Exact dyadic constructions
--------------------------
A normalised Sylvester-Hadamard block of order 4^j has entries +-2^-j and is
orthogonal.  Block-diagonal products of such blocks over different partitions
of the rows (each with a random signed row permutation) give dense orthogonal
matrices whose entries are integers in units of a small power of two.  From
them:

* QR: A = Q0 R0 with R0 dyadic, upper triangular, positive diagonal and
  strictly row-diagonally dominant (kappa(R0) <= 11).  Full column rank makes
  (Q0, R0) THE stabilised QR of A.
* SVD: A = Q1 diag(s) V^T with Q1 the first n columns of an m x m factor, V an
  n x n factor and dyadic s: the singular values are exact, and so are the
  singular subspaces.

Every product is formed in float64 under an asserted bound: with all factors
integers in units 2^-J, every partial sum of every product is an integer in
units of the product's unit whose magnitude is below |F1| |F2| ... < 2^53, so
float64 arithmetic is exact in any summation order (``exact_product``).

Bounds
------
eps = 2^-52, n = the number of columns, ``C`` below.  All are relative to the
2-norm of the input (s1) and are what a backward-stable factorisation meets:

* backward error   |A - Q R|_F, |A - U S V^T|_F  <= C n eps |A|_F
* orthogonality    |Q^T Q - I|_max               <= C n eps
* singular values  |s_i - s_i*|                  <= C n eps s1        (Weyl)
* QR factors       |R - R0|_max / |R0|_max, |Q - Q0|_max <= C n eps kappa(R0)
* singular vectors |sin angle(u_i, u_i*)|        <= C n eps s1 / gap_i, and the
  same for the subspace of an exact cluster against the rest.

A matrix scaled by 2^k is judged in its own units.  When the scaled matrix
is stored with subnormal entries, it is compared against the oracle of the
matrix as stored (scaling it back up is exact), with a floor of about one
subnormal unit in the last place (2^-1074) per output entry.
"""

import numpy as np
from scipy.linalg import hadamard

EPS = 2.0 ** -52
TINY = 2.0 ** -1074
C = 16.0
LIM = 2.0 ** 53


def bound(n):
    return C * max(n, 1) * EPS


# -------------------------------------------------------------- dyadic blocks
def _pow4_parts(n, rng, cap=64):
    """A partition of n into powers of four (each <= cap), in random order."""
    parts = []
    left = n
    while left:
        b = cap
        while b > left:
            b //= 4
        parts.append(b)
        left -= b
    rng.shuffle(parts)
    return parts


def hadamard_unit(order):
    """Normalised Sylvester-Hadamard block of order 4^j as integers (+-1) and
    its unit 2^-j: H = ints * 2^-j, H^T H = I."""
    j = int(round(np.log(order) / np.log(4)))
    assert 4 ** j == order, order
    return hadamard(order).astype(np.int64), j


def _apply_layer(X, J, rng, cap):
    """One factor applied to X (ints in units 2^-J, m x k): block-diagonal
    Hadamard blocks over a random partition of the m rows into powers of four,
    then the rows signed and permuted.  Returns (ints, unit exponent); blocks
    of smaller order are scaled up to the common unit.  Asserts the exactness
    bound of the product."""
    m = X.shape[0]
    parts = _pow4_parts(m, rng, cap)
    jmax = max(hadamard_unit(b)[1] for b in parts)
    Y = np.empty_like(X)
    o = 0
    for b in parts:
        h, j = hadamard_unit(b)
        blk = X[o:o + b]
        mag = np.abs(h).astype(np.float64) @ np.abs(blk).astype(np.float64)
        assert mag.max(initial=0.0) * 2.0 ** (jmax - j) < LIM, "dyadic product would not be exact"
        Y[o:o + b] = (h @ blk) << (jmax - j)
        o += b
    perm = rng.permutation(m)
    sign = rng.choice(np.array([-1, 1], dtype=np.int64), size=m)
    return Y[perm] * sign[:, None], J + jmax


def exact_product(*factors):
    """Product of (ints, J) factors, formed in float64.  Asserts that every
    partial sum is an integer below 2^53 in units of the product, which makes
    the float64 result exact whatever the summation order."""
    ints = [f[0].astype(np.float64) for f in factors]
    J = sum(f[1] for f in factors)
    mag = np.abs(ints[0])
    for x in ints[1:]:
        mag = mag @ np.abs(x)
    assert mag.max(initial=0.0) < LIM, "dyadic product would not be exact"
    p = ints[0]
    for x in ints[1:]:
        p = p @ x
    return p, J


def isometry(m, k, rng, layers=2, cap=64):
    """m x k matrix with orthonormal columns, (ints, J): the first k columns
    of a product of `layers` signed, permuted block-Hadamard factors over
    different partitions (dense once layers >= 2)."""
    X = np.zeros((m, k), dtype=np.int64)
    X[np.arange(k), np.arange(k)] = 1
    J = 0
    for _ in range(layers):
        X, J = _apply_layer(X, J, rng, cap)
    return X, J


def to_float(f):
    ints, J = f
    return np.ldexp(np.asarray(ints, dtype=np.float64), -J)


# ----------------------------------------------------------------- QR oracle
def qr_case(m, n, rng, layers=2):
    """(A, Q0, R0, kappa): A = Q0 R0 exactly, R0 upper triangular with a
    positive diagonal in [4, 8] and at most three off-diagonal entries of
    magnitude <= 1 per row (units of 1/4): kappa_inf(R0) <= 11."""
    k = min(m, n)
    Q0 = isometry(m, k, rng, layers)
    R = np.zeros((k, n), dtype=np.int64)
    R[np.arange(k), np.arange(k)] = rng.integers(16, 33, size=k)   # 4 .. 8 in units of 1/4
    for i in range(k):
        cols = np.arange(i + 1, n)
        if cols.size:
            pick = rng.choice(cols, size=min(3, cols.size), replace=False)
            R[i, pick] = rng.integers(-4, 5, size=pick.size)
    A, J = exact_product(Q0, (R, 2))
    Rf = np.ldexp(R.astype(np.float64), -2)
    kappa = np.linalg.cond(Rf[:, :k]) if k else 1.0
    return np.ldexp(A, -J), to_float(Q0), Rf, kappa


# ---------------------------------------------------------------- SVD oracle
def spectrum(kind, n, rng):
    """Dyadic singular values, descending, as (ints, unit exponent)."""
    if kind == "separated":
        s = np.arange(2 * n, n, -1, dtype=np.int64)              # distinct, gap 1
        return s, 0
    if kind == "clusters":
        base = np.repeat(np.arange(1, n + 1)[::-1], 3)[:n]      # triples
        return np.sort(base)[::-1].astype(np.int64) * 4, 0
    if kind == "zeros":
        r = max(1, n // 2)
        s = np.zeros(n, dtype=np.int64)
        s[:r] = np.arange(2 * r, r, -1)
        return s, 0
    if kind == "graded":
        e = np.round(np.linspace(0, 40, n)).astype(np.int64)    # 2^0 .. 2^-40
        return np.left_shift(np.int64(1), 40 - e), 40
    if kind == "gap":
        r = max(1, n // 3)
        s = np.full(n, 1, dtype=np.int64)
        s[:r] = 1 << 20                                          # 1 | 2^-20
        s[:r] += np.arange(r)[::-1]
        return s, 20
    raise ValueError(kind)


def svd_case(m, n, kind, rng):
    """(A, U0, s, V0): A = U0 diag(s) V0^T exactly (m >= n), U0 m x n and V0
    n x n with dyadic entries, s exact and descending."""
    cap = 16 if kind == "graded" else 64
    U0 = isometry(m, n, rng, 2, cap)
    Vf = isometry(n, n, rng, 2, cap)
    si, js = spectrum(kind, n, rng)
    A, J = exact_product(U0, (np.diag(si), js), (Vf[0].T, Vf[1]))
    return np.ldexp(A, -J), to_float(U0), np.ldexp(si.astype(np.float64), -js), to_float(Vf)


def gaps(s):
    """Distance of each singular value to the rest of the spectrum (0 inside
    an exact cluster: there the cluster's subspace is compared instead)."""
    g = np.full(s.size, np.inf)
    for i in range(s.size):
        d = np.abs(s - s[i])
        d[i] = np.inf
        d[d == 0] = np.inf
        g[i] = d.min()
    return g


def clusters(s):
    """Index ranges of equal singular values."""
    out, i = [], 0
    while i < s.size:
        j = i + 1
        while j < s.size and s[j] == s[i]:
            j += 1
        out.append((i, j))
        i = j
    return out


def subspace_sin(X, Y):
    """Largest sine of the principal angles between the column spans of the
    orthonormal X and Y (same column count)."""
    if X.shape[1] == 0:
        return 0.0
    proj = X - Y @ (Y.T @ X)
    return float(np.linalg.norm(proj, 2))


# ------------------------------------------------------------ checks (numpy)
def check_orthonormal_cols(Q, n, what="Q"):
    k = Q.shape[1]
    err = np.abs(Q.T @ Q - np.eye(k)).max(initial=0.0)
    assert err <= bound(n), f"{what}: |Q^T Q - I| = {err:.3g} > {bound(n):.3g}"


def check_qr(A, Q, R, n=None, kappa=None, Q0=None, R0=None, scale=1.0, floor=None):
    """Stabilised QR against the bounds; Q0 / R0 (exact factors of A / scale)
    when known."""
    n = A.shape[1] if n is None else n
    assert np.all(np.isfinite(Q)) and np.all(np.isfinite(R))
    k = min(A.shape)
    assert np.all(np.tril(R[:, :k], -1) == 0), "R is not upper triangular"
    assert np.all(np.diag(R) >= 0), "diag(R) < 0: not stabilised"
    nrm = np.linalg.norm(A)
    floor = C * n * TINY if floor is None else floor
    err = np.linalg.norm(A - Q @ R)
    assert err <= bound(n) * nrm + floor, f"|A - QR| / |A| = {err / max(nrm, TINY):.3g}"
    check_orthonormal_cols(Q, n)
    if R0 is not None:
        tol = bound(n) * kappa
        eR = np.abs(R - R0 * scale).max() / (np.abs(R0).max() * scale)
        eQ = np.abs(Q - Q0).max()
        assert eR <= tol, f"|R - R0| / |R0| = {eR:.3g} > {tol:.3g}"
        assert eQ <= tol, f"|Q - Q0| = {eQ:.3g} > {tol:.3g}"


def check_svd(A, U, s, VH, s_exact=None, U0=None, V0=None, scale=1.0, floor=None):
    """Thin SVD (U m x k, s k, VH k x n) against the bounds; the exact
    factors (of A / scale) when known."""
    n = max(A.shape)
    assert np.all(np.isfinite(U)) and np.all(np.isfinite(s)) and np.all(np.isfinite(VH))
    assert np.all(np.diff(s) <= 0) and np.all(s >= 0), "s not sorted / negative"
    nrm = np.linalg.norm(A)
    floor = C * n * TINY if floor is None else floor
    err = np.linalg.norm(A - (U * s) @ VH)
    assert err <= bound(n) * nrm + floor, f"|A - USV| / |A| = {err / max(nrm, TINY):.3g}"
    check_orthonormal_cols(U, n, "U")
    check_orthonormal_cols(VH.T, n, "V")
    if s_exact is None:
        return
    s1 = s_exact[0] * scale
    es = np.abs(s - s_exact * scale).max()
    assert es <= bound(n) * s1 + floor, f"|s - s*| / s1 = {es / max(s1, TINY):.3g}"
    if U0 is None:
        return
    for i, j in clusters(s_exact):
        if s_exact[i] == 0.0:
            continue      # the null space is any completion
        rest = np.concatenate([s_exact[:i], s_exact[j:]])
        # the vectors on the longer side are also separated from its null
        # space (singular value 0)
        k = s_exact.size
        for X, X0, r in ((U[:, i:j], U0[:, i:j],
                          np.append(rest, 0.0) if A.shape[0] > k else rest),
                         (VH[i:j].T, V0[:, i:j],
                          np.append(rest, 0.0) if A.shape[1] > k else rest)):
            gap = np.abs(r - s_exact[i]).min(initial=np.inf) * scale
            tol = bound(n) * s1 / gap if np.isfinite(gap) else bound(n)
            if tol < 0.5:
                sn = subspace_sin(X, X0)
                assert sn <= tol, f"singular subspace {i}:{j}: sin = {sn:.3g} > {tol:.3g}"


def keep_rule(s, cutoff, cutoff_mode, max_bond=-1):
    """(n_keep, truncation error) of the reference rule on exact values."""
    from oracle.decomp_np import number_svals_to_keep
    nk = s.size
    if cutoff > 0.0:
        nk = number_svals_to_keep(s, cutoff, cutoff_mode)
    if max_bond > 0:
        nk = min(nk, max_bond)
    err = float(np.sqrt(np.sum(s[nk:] ** 2)))
    return nk, err


# -------------------------------------------------------------- mpmath oracle
def mp_svd(A, dps=40):
    """Singular values of a float64 matrix at `dps` digits (mpmath)."""
    import mpmath
    if A.shape[0] < A.shape[1]:
        A = A.T
    with mpmath.workdps(dps):
        M = mpmath.matrix(A.tolist())
        s = mpmath.svd_r(M, compute_uv=False)
        return np.array(sorted((float(x) for x in s), reverse=True))


def mp_qr_r(A, dps=40):
    """R of the stabilised QR (diag >= 0) at `dps` digits, rounded once."""
    import mpmath
    with mpmath.workdps(dps):
        M = mpmath.matrix(A.tolist())
        _, R = mpmath.qr(M)
        k = min(A.shape)
        R = np.array([[float(R[i, j]) for j in range(A.shape[1])] for i in range(k)])
    sg = np.where(np.diag(R) < 0, -1.0, 1.0)
    return R * sg[:, None]


# --------------------------------------------------------------- route search
# shapes around every threshold: panel instantiations switch at 2048 / 4096 /
# 8192 / 16384 rows, TSQR above 16384, aggregation above 4096 rows or 48 MiB,
# Jacobi stream groups at 16 / 64 column blocks of 16 (n = 1030: 66 blocks,
# not divisible -> one group)
ROWS = (16, 48, 64, 100, 2048, 2049, 4096, 4097, 8192, 8193, 16384, 16385, 65536)
COLS = (1, 15, 16, 17, 31, 32, 33, 127, 128, 129, 512, 1024, 1030, 1600, 2048)
ABSORBS = (None, 100, 2, -1, -10, -11, 0, -12, 12, 1, 10, 11)
QR_KEYS = ([("qr", "panel", k) for k in range(4)]
           + [("qr", "aggregated", "m<=4096"), ("qr", "aggregated", "m>4096"),
              ("qr", "tsqr"), ("qr", "wide"), ("qr", "complex")])
SVD_KEYS = ([("svd", "groups", g) for g in (1, 2, 4)]
            + [("svd", "groups", "fallback")]
            + [("svd", "epilogue", e) for e in ("accumulate", "left", "right", "values")]
            + [("svd", "mirror"), ("svd", "transpose"), ("svd", "qr_first"),
               ("svd", "complex")])


def grid_shapes():
    shapes = set()
    for m in ROWS:
        for n in COLS:
            if n <= m and m * n * n <= (1 << 34):
                shapes.add((m, n))
                if m <= 2048:
                    shapes.add((n, m))     # wide
    return sorted(shapes, key=lambda s: (s[0] * s[1] * min(s), s))


def qr_keys_of(route):
    keys = []
    if route["complex_embed"]:
        return [("qr", "complex")]
    if route["path"] == "tsqr":
        keys.append(("qr", "tsqr"))
    if route["path"] == "wide":
        keys.append(("qr", "wide"))
    for k in route["kernels"]:
        for b in range(4):
            if k["panel_mask"] >> b & 1:
                keys.append(("qr", "panel", b))
        if k["wy_t"]:
            keys.append(("qr", "aggregated", "m<=4096" if k["shape"][0] <= 4096 else "m>4096"))
    return keys


def svd_keys_of(route):
    if route["complex_embed"]:
        return [("svd", "complex")]
    keys = [("svd", "epilogue", route["epilogue"])]
    if route["mirror"]:
        keys.append(("svd", "mirror"))
    if route["transpose"]:
        keys.append(("svd", "transpose"))
    if route["qr_first"]:
        keys.append(("svd", "qr_first"))
    g = route["groups"]
    keys.append(("svd", "groups", g))
    if g == 1 and route["nblk"] >= 16:
        keys.append(("svd", "groups", "fallback"))
    return keys


def search_routes(min_cols=1):
    """{key: (shape, dtype, absorb, route)}: the cheapest grid shape with at
    least `min_cols` columns and rows that reaches each QR / SVD route, as the
    library reports it."""
    import torch
    from quimb_b200 import linalg
    found = {}
    for shape in grid_shapes():
        if min(shape) < min_cols:
            continue
        for dt in (torch.float64, torch.complex128):
            if dt == torch.complex128 and max(shape) > 64:
                continue
            r = linalg.route_qr(shape, dt)
            for key in qr_keys_of(r):
                found.setdefault(key, (shape, dt, None, r))
            for absorb in ABSORBS if dt == torch.float64 else (None,):
                if max(shape) > 16384 and min(shape) > 64:
                    continue
                r = linalg.route_svd(shape, dt, absorb)
                for key in svd_keys_of(r):
                    found.setdefault(key, (shape, dt, absorb, r))
    return found
