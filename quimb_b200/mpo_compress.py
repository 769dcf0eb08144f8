"""Apply an MPO to an MPS on the device and compress the result to a bounded
bond dimension, without forming the full chi D_w product chain first.

Mirrors, at array level and for open-boundary (l, p, r) site lists,

  MatrixProductState.gate_with_mpo         tn1d/core.py:2446-2509
  tensor_network_1d_compress (dispatch)    tn1d/compress.py:3197-3356
    'direct'                               tn1d/compress.py:139-297
    'dm'                                   tn1d/compress.py:383-665
    'zipup'                                tn1d/compress.py:668-864
    'zipup-first' / 'zipup-oversample'     tn1d/compress.py:867-1073
  canonize_around_ / get_tree_span         tensor_core.py:7447-7626,
                                           networking.py:196-356

The network is the reference's two-layer ladder: MPS site i, A[l, p, r],
and MPO site i, W[wl, wr, u, d], joined by a rung.  By default the MPO's
lower index d meets the MPS and u becomes the output index; ``transpose``
swaps the two (``tebd.mpo_apply`` contracts u).

Every contraction is one ``contract_pair`` launch, every factorisation the
device QR, Jacobi SVD or ``eigh``; the only host arithmetic is each split's
truncation rule and the spanning tree of the zip-up gauge (control logic on
a graph of 2 L nodes).
"""

import collections
import math

import numpy as np

from . import ops, tebd
from .array import Array
from .contract import contract_pair
from .linalg import norm as _norm
from .mps import mpo_lrud
from .split import array_split, tensor_canonize_bond

METHODS = ("direct", "dm", "zipup", "zipup-first", "zipup-oversample")

# methods the reference offers that are not built here
_NOT_BUILT = ("fit", "src", "sdc", "srcmps", "projector", "autofit", "local-early",
              "local-late", "superorthogonal", "l2bp")

# the options the direct sweep's compress_between takes (split.tensor_compress_bond)
_BOND_OPTS = {"max_bond", "cutoff", "cutoff_mode", "absorb", "renorm", "reduced"}

_DEFAULT_CUTOFF_MODE = {"direct": "rsum2", "dm": "rsum1", "zipup": "rsum2",
                        "zipup-first": "rsum2", "zipup-oversample": "rsum2"}


def _check_method(method):
    if method in METHODS:
        return
    if any(method == m or method.startswith(m + "-") for m in _NOT_BUILT):
        raise NotImplementedError(f"mps_gate_with_mpo: method {method!r} is not implemented "
                                  f"(available: {', '.join(METHODS)})")
    raise ValueError(f"mps_gate_with_mpo: unknown method {method!r}")


def _cp(a, la, b, lb, lc):
    """One contraction of two Arrays (lazy conjugation folded into the loads),
    promoting a dtype mismatch first."""
    if a.dtype != b.dtype:
        dt = np.result_type(a.dtype, b.dtype)
        a, b = a.astype(dt, copy=False), b.astype(dt, copy=False)
    return Array(contract_pair(a.t, la, b.t, lb, lc, conj_a=a.cj, conj_b=b.cj))


# ---------------------------------------------------------------- the ladder ---
def _prepare(sites, mpo, mpo_shape, transpose):
    """MPS sites A[l, p, r] and MPO sites W[wl, wr, o, p] (o the output index,
    p the one that meets the MPS), one common dtype; views of the caller's
    arrays."""
    L = len(sites)
    if L == 0:
        raise ValueError("mps_gate_with_mpo: empty MPS")
    if len(mpo) != L:
        raise ValueError(f"mps_gate_with_mpo: the MPO has {len(mpo)} sites, the MPS {L}")
    A = [ops.asarray(a) for a in sites]
    for a in A:
        if a.ndim != 3:
            raise ValueError("mps_gate_with_mpo: sites must be (l, p, r) arrays")
        if np.dtype(a.dtype).kind not in "fc":
            raise TypeError(f"mps_gate_with_mpo: unsupported dtype {a.dtype}")
    if A[0].shape[0] != 1 or A[-1].shape[2] != 1:
        raise ValueError("mps_gate_with_mpo: open boundaries only (first left and last "
                         "right bond of dimension 1)")
    W = []
    for i in range(L):
        w = mpo_lrud(mpo[i], mpo_shape, i, L)
        W.append(w.transpose(0, 1, 3, 2) if transpose else w)
    for i in range(L):
        if W[i].shape[3] != A[i].shape[1]:
            raise ValueError(f"mps_gate_with_mpo: site {i} has physical dimension "
                             f"{A[i].shape[1]}, the MPO index meeting it {W[i].shape[3]}")
        if i and (A[i - 1].shape[2] != A[i].shape[0] or W[i - 1].shape[1] != W[i].shape[0]):
            raise ValueError(f"mps_gate_with_mpo: bond mismatch between sites {i - 1} and {i}")
    if W[0].shape[0] != 1 or W[-1].shape[1] != 1:
        raise ValueError("mps_gate_with_mpo: open-boundary MPO only")
    dt = np.result_type(*[x.dtype for x in A + W])
    A = [a.astype(dt, copy=False) for a in A]
    W = [w.astype(dt, copy=False) for w in W]
    return A, W, dt


def _flip(A, W):
    """The ladder read from the other end."""
    return ([a.transpose(2, 1, 0) for a in reversed(A)],
            [_flip_w(w) for w in reversed(W)])


def _flip_w(w):
    if isinstance(w, int):
        return w
    return w.transpose(1, 0) if w.ndim == 2 else w.transpose(1, 0, 2, 3)


def _flip_mps(A):
    return [a.transpose(2, 1, 0) for a in reversed(A)]


def ladder_tree_span(L, bond_a, bond_w, phys, root, gaps=(), open_ends=(False, False),
                     rung_between=False):
    """``get_tree_span`` (networking.py:196-356, defaults: weight_bonds,
    ndim_sort 'max', distance_sort 'min', inwards) of the MPS / MPO ladder
    fanning out from site ``root``: the ordered merges ``(n1, n2)``, node
    ``i`` the MPS tensor of site i and node ``L + i`` the MPO tensor.

    Models the network ``gate_with_mpo`` builds: MPS tensors first, then MPO
    tensors; index orders 'lrp' and 'lrud' without the end sites' outer
    bonds.  ``bond_a[i]`` / ``bond_w[i]`` are the bonds (i, i + 1) of the two
    layers, ``phys[i]`` the rung of site i.

    The sub-range network of ``gate_with_submpo`` (tn1d/core.py:2339-2442)
    differs in three ways: sites in ``gaps`` carry a two-index identity on
    the MPO layer instead of an MPO tensor (no rung; enforce_1d_like,
    compress.py:38-125), ``open_ends`` marks MPS end tensors that keep their
    bond to the rest of the chain as an outer index, and with
    ``rung_between`` the MPO tensors list their rung between their left and
    right bonds (the index order of ``MatrixProductOperator.from_dense``)."""
    gaps = frozenset(gaps)

    def ndim(n):
        i = n % L
        if n < L:
            return 3 - (i == 0 and not open_ends[0]) - (i == L - 1 and not open_ends[1])
        if i in gaps:
            return 2
        return 4 - (i == 0) - (i == L - 1)

    def neighbours(n):
        i, off = n % L, (0 if n < L else L)
        out = [off + i - 1] if i > 0 else []
        rung = [] if i in gaps else [n + L if n < L else n - L]
        if rung_between and n >= L:
            out += rung
            rung = []
        if i < L - 1:
            out.append(off + i + 1)
        return out + rung

    def size(n1, n2):
        if abs(n1 - n2) == L:
            return phys[n1 % L]
        i = min(n1, n2) % L
        return bond_a[i] if n1 < L else bond_w[i]

    region = [root, L + root]
    in_region = set(region)
    candidates, merges = [], {}
    distances = {n: 0 for n in region}
    connectivity = collections.defaultdict(lambda: 0)

    def check(s, nb):
        if nb in in_region:
            return
        if nb not in distances:
            merges[nb] = s
            distances[nb] = distances[s] + 1
            candidates.append(nb)
        connectivity[nb] += math.log2(size(s, nb))

    for s in region:
        for nb in neighbours(s):
            check(s, nb)
    seq = []
    while candidates:
        candidates.sort(key=lambda t: (connectivity[t], ndim(t), -distances[t]))
        s = candidates.pop()
        in_region.add(s)
        seq.append((s, merges[s]))
        for nb in neighbours(s):
            check(s, nb)
    seq.reverse()
    return seq


def _ladder_inds(L, n):
    i = n % L
    if n < L:
        return (("a", i - 1), ("p", i), ("a", i))
    return (("w", i - 1), ("w", i), ("o", i), ("p", i))


def _ladder_inds_gap(L, n, W):
    i = n % L
    if n >= L and W[i].ndim == 2:
        return (("w", i - 1), ("w", i))
    return _ladder_inds(L, n)


def _canonize_around(A, W, root, **span_opts):
    """``canonize_around_(site root)`` of the ladder: the QR moves of the
    spanning tree, inwards (tensor_canonize_bond, absorb='right'), on new
    lists.  A gap site of a sub-range ladder (``W[i]`` an int, the size of
    the bond passing it) enters as the identity matrix the reference threads
    through it; the gauge generally leaves a full matrix there."""
    L = len(A)
    gaps = [i for i, w in enumerate(W) if isinstance(w, int)]
    W = [ops.eye(w, dtype=A[0].dtype, device=A[0].device) if isinstance(w, int) else w
         for w in W]
    T = list(A) + list(W)
    seq = ladder_tree_span(L, [a.shape[2] for a in A[:-1]], [w.shape[1] for w in W[:-1]],
                           [a.shape[1] for a in A], root, gaps=gaps, **span_opts)
    for n1, n2 in seq:
        T[n1], T[n2] = tensor_canonize_bond(T[n1], _ladder_inds_gap(L, n1, W), T[n2],
                                            _ladder_inds_gap(L, n2, W), absorb="right")
    return T[:L], T[L:]


def _product_site(a, w):
    """A[a, p, b] W[w, v, o, p] -> site[(a w), o, (b v)]; at a gap site
    (``w`` the int size of the MPO bond passing it) the index expansion
    A[a, p, b] delta[w, v], placed without a contraction."""
    if isinstance(w, int):
        return _expand_site(a, w)
    t = _cp(a, [0, 1, 2], w, [3, 4, 5, 1], [0, 3, 5, 2, 4])
    l, wl, o, r, wr = t.shape
    return t.reshape(l * wl, o, r * wr)


def _expand_site(a, D):
    """site[(a w), p, (b v)] = A[a, p, b] delta[w, v]: one permute launch
    copies A, broadcast over w, onto the (w, v) diagonal of a zeroed buffer."""
    from . import _lib
    x = a.t
    l, p, r = x.shape
    out = ops.zeros((l, D, p, r, D), dtype=a.dtype, device=a.device).t
    if out.numel():
        src = x.unsqueeze(-1).expand(l, p, r, D)
        dst = out.diagonal(dim1=1, dim2=4)
        rc = _lib.load().qb_permute(_lib.desc(src), _lib.desc(dst), int(a.cj),
                                    _lib.stream_ptr())
        _lib.check(rc, "qb_permute")
    return Array(out.reshape(l * D, p, r * D))


def _seed(A):
    """The right boundary of a contraction carried in from the right:
    delta[b, k] over the ladder's last MPS bond, with a size-1 MPO bond
    (ones((1, 1, 1)) when that bond is closed)."""
    r = A[-1].shape[2]
    return Array(ops.eye(r, dtype=A[0].dtype, device=A[0].device).t.reshape(r, 1, r))


def _carry(a, w, R):
    """C[a, w, o, k] = sum R[b, v, k] A[a, p, b] W[w, v, o, p], with W the
    identity at a gap site (one launch) or a gauged gap matrix W[w, v]."""
    if isinstance(w, int):
        return _cp(a, [0, 1, 2], R, [2, 3, 4], [0, 3, 1, 4])
    T = _cp(a, [0, 1, 2], R, [2, 3, 4], [0, 1, 3, 4])                  # [a, p, v, k]
    if w.ndim == 2:
        return _cp(T, [0, 1, 3, 4], w, [5, 3], [0, 5, 1, 4])
    return _cp(T, [0, 1, 3, 4], w, [5, 3, 6, 1], [0, 5, 6, 4])


# ------------------------------------------------------------------ methods ---
def _direct(A, W, canonize, opts):
    """compress.py:139-297: contract site by site, QR each finished site into
    the next, then one compress_between sweep back (absorb='left',
    reduced='right')."""
    L = len(A)
    out = [_product_site(A[0], W[0])]
    for i in range(1, L):
        out.append(_product_site(A[i], W[i]))
        if canonize:
            tebd.left_canonize_site(out, i - 1)
    _direct_sweep(out, opts)
    return out


def _direct_sweep(out, opts):
    """_do_direct_sweep (compress.py:867-908) without its normalisation."""
    for i in range(len(out) - 1, 0, -1):
        tebd.right_compress_site(out, i, **opts)


def _zipup(A, W, canonize, rev, opts, span_opts=None):
    """compress.py:668-864 over the ladder read from the right (from the left
    when ``rev``): pseudo-canonical gauge around the starting end, then carry
    U s leftwards, splitting C = (U s) A W at every site (absorb='left').
    The result is right-canonical in the direction of the sweep.

    The ladder may be a sub-range of a longer chain: the MPS end bonds are
    then open outer indices (the first product keeps its left bond, the
    carry starts from delta over the last right bond), a gap site (``W[i]``
    an int) carries an identity, and ``span_opts`` describe the sub-range
    network to :func:`ladder_tree_span`."""
    L = len(A)
    opts = dict(opts)
    opts.setdefault("absorb", "left")
    if canonize:
        A, W = _canonize_around(A, W, 0 if rev else L - 1, **(span_opts or {}))
    if rev:
        A, W = _flip(A, W)
    ts = [None] * L
    Us = _seed(A)
    for i in range(L - 1, -1, -1):
        # C[a, w, o, k] = sum Us[b, v, k] A[a, p, b] W[w, v, o, p]
        C = _carry(A[i], W[i], Us)
        la, lw, o, k = C.shape
        if i == 0:
            ts[0] = C.reshape(la * lw, o, k)
            break
        left, _, right = array_split(C.reshape(la * lw, o * k), **opts)
        n = right.shape[0]
        ts[i] = ops.materialize(right).reshape(n, o, k)
        Us = ops.materialize(left).reshape(la, lw, n)
    return _flip_mps(ts) if rev else ts


def _dm(A, W, opts):
    """compress.py:383-665: left environments of the ket / bra double layer,
    then from the right one reduced density matrix per site, split by
    ``eigh``; U^dagger folded into the ket's right environment.  The bra's
    environment is the conjugate of the ket's and is never formed: it enters
    every contraction as a conjugation flag.  On a sub-range ladder (see
    :func:`_zipup`) the first environment traces over the open left bond and
    the right environment starts from delta over the open right bond."""
    L = len(A)
    opts = dict(opts)
    opts.setdefault("method", "eigh")
    opts.setdefault("positive", 1)
    opts.setdefault("absorb", None)
    # E[a, w, a', w'] (ket a, w; bra a', w') left of site i, for i = 1 .. L-1
    envs = [None] * L
    E = None
    for i in range(L - 1):
        a, w = A[i], W[i]
        if E is None:
            # the trace runs over the open left bond too, when there is one
            T = _product_site(a, w).reshape(-1, a.shape[2], w.shape[1])
            E = _cp(T, [0, 1, 2], T.conj(), [0, 3, 4], [1, 2, 3, 4])
        elif isinstance(w, int):
            # gap site: the identities of the two layers only relabel w
            X = _cp(E, [0, 1, 2, 3], a, [0, 4, 5], [1, 2, 3, 4, 5])             # [w, a', w', p, b]
            E = _cp(X, [1, 2, 3, 4, 5], a.conj(), [2, 4, 10], [5, 1, 10, 3])   # [b, w, b', w']
        else:
            X = _cp(E, [0, 1, 2, 3], a, [0, 4, 5], [1, 2, 3, 4, 5])             # [w, a', w', p, b]
            X = _cp(X, [1, 2, 3, 4, 5], W[i], [1, 6, 7, 4], [2, 3, 5, 6, 7])    # [a', w', b, v, o]
            X = _cp(X, [2, 3, 5, 6, 7], W[i].conj(), [3, 8, 7, 9], [2, 5, 6, 9, 8])  # [a', b, v, p', v']
            E = _cp(X, [2, 5, 6, 9, 8], a.conj(), [2, 9, 10], [5, 6, 10, 8])   # [b, v, b', v']
        envs[i + 1] = E
    out = [None] * L
    R = _seed(A)                                                             # R[b, v, k]
    for i in range(L - 1, -1, -1):
        # Y[a, w, o, k] = sum A[a, p, b] W[w, v, o, p] R[b, v, k]: the ket side
        Y = _carry(A[i], W[i], R)
        la, lw, o, k = Y.shape
        if i == 0:
            out[0] = Y.reshape(la * lw, o, k)
            break
        Z = _cp(envs[i], [0, 1, 2, 3], Y, [0, 1, 4, 5], [2, 3, 4, 5])         # [a', w', o, k]
        rho = _cp(Z, [2, 3, 4, 5], Y.conj(), [2, 3, 6, 7], [4, 5, 6, 7])      # [o, k, o', k']
        U, _, _ = array_split(rho.reshape(o * k, o * k), **opts)
        n = U.shape[1]
        U = ops.materialize(U).reshape(o, k, n)
        out[i] = ops.materialize(U.transpose(2, 0, 1))
        R = _cp(Y, [0, 1, 2, 3], U.conj(), [2, 3, 4], [0, 1, 4])             # [a, w, n]
    return out


# ------------------------------------------------------------------- driver ---
def mps_gate_with_mpo(sites, mpo, method="direct", max_bond=None, cutoff=1e-10,
                      cutoff_mode=None, transpose=False, normalize=False,
                      sweep_reverse=False, canonize=True, mpo_shape="lrud",
                      max_bond_oversample=None, cutoff_oversample=None, info=None,
                      equalize_norms=False, **split_opts):
    """``MatrixProductState.gate_with_mpo(mpo, method=...)`` (tn1d/core.py:
    2446-2509) for open-boundary (l, p, r) device sites: the MPO applied and
    the result compressed to ``max_bond`` / ``cutoff`` by one of

      'direct'       contract site by site, canonicalise, one truncating sweep
                     back (SVD of each product site's reduced factor)
      'dm'           density-matrix method: one (d chi')^2 reduced density
                     matrix per site, split by eigh
      'zipup'        zip-up in the reference's pseudo-canonical gauge
      'zipup-first'  zip-up to ``max_bond_oversample`` (default 2 max_bond; a
                     float multiplies max_bond) and ``cutoff_oversample``, then
                     one direct sweep (also 'zipup-oversample')

    ``cutoff_mode`` defaults to 'rsum1' for 'dm' and 'rsum2' otherwise.
    ``split_opts`` go to every truncating split and override its defaults
    as in the reference: 'zipup' splits with ``absorb='left'``, 'dm' with
    ``method='eigh', positive=1, absorb=None``, the direct sweeps with
    ``absorb='left', reduced='right'``.  The direct sweeps take only the
    options of ``split.tensor_compress_bond`` (max_bond, cutoff,
    cutoff_mode, absorb, renorm, reduced); any other key raises
    ``TypeError`` for 'direct' and 'zipup-first'.  ``mpo`` sites are in layout
    ``mpo_shape`` (quimb's end tensors accepted); by default the MPO's lower
    index meets the MPS, ``transpose`` contracts the upper one.

    Returns a new list of (l, p, r) device Arrays in the promoted dtype of
    MPS and MPO, right-canonical with the centre at site 0 (left-canonical,
    centre L - 1, with ``sweep_reverse``); ``normalize`` scales the centre to
    unit norm.  ``info["cur_orthog"]`` receives the centre.  The caller's
    sites and MPO are not modified."""
    _check_method(method)
    if equalize_norms:
        raise NotImplementedError("mps_gate_with_mpo: equalize_norms is not implemented")
    A, W, dt = _prepare(list(sites), list(mpo), mpo_shape, transpose)
    L = len(A)
    if cutoff_mode is None:
        cutoff_mode = _DEFAULT_CUTOFF_MODE[method]
    opts = dict(split_opts, max_bond=max_bond, cutoff=cutoff, cutoff_mode=cutoff_mode)
    if method in ("direct", "zipup-first", "zipup-oversample"):
        extra = sorted(set(split_opts) - _BOND_OPTS)
        if extra:
            raise TypeError(f"mps_gate_with_mpo: method {method!r} does not take the split "
                            f"option(s) {extra}")
    if method == "zipup-first" or method == "zipup-oversample":
        mbo = _oversample_bond(max_bond, max_bond_oversample)
        if cutoff_oversample is None:
            cutoff_oversample = cutoff / 10 if max_bond is None else cutoff
        zopts = dict(opts, max_bond=mbo, cutoff=cutoff_oversample)
        out = _zipup(A, W, canonize, not sweep_reverse, zopts)
        if sweep_reverse:
            out = _flip_mps(out)
        _direct_sweep(out, opts)
        if sweep_reverse:
            out = _flip_mps(out)
    elif method == "zipup":
        out = _zipup(A, W, canonize, sweep_reverse, opts)
    else:
        if sweep_reverse:
            A, W = _flip(A, W)
        if method == "direct":
            out = _direct(A, W, canonize, opts)
        else:
            if not canonize:
                import warnings
                warnings.warn("`canonize=False` is ignored for the `dm` method.")
            out = _dm(A, W, opts)
        if sweep_reverse:
            out = _flip_mps(out)
    c = L - 1 if sweep_reverse else 0
    if normalize:
        x = ops.materialize(out[c], force=True)
        out[c] = ops.scale_(x, 1.0, div_by=_norm(x))
    out = [ops.materialize(x).astype(dt, copy=False) for x in out]
    if info is not None:
        info["cur_orthog"] = (c, c)
    return out


def _oversample_bond(max_bond, max_bond_oversample):
    """compress.py:1011-1031, with a non-positive result rejected."""
    if max_bond_oversample is None:
        if max_bond is None:
            import warnings
            warnings.warn("Both `max_bond` and `max_bond_oversample` are None, typically "
                          "relying on `cutoff` and `cutoff_oversample` only is not "
                          "recommended for this method.")
            return None
        mbo = 2 * max_bond
    elif isinstance(max_bond_oversample, float):
        if max_bond is None:
            raise ValueError("`max_bond_oversample` cannot be a float (a multiplier) if "
                             "`max_bond` is None.")
        mbo = round(max_bond * max_bond_oversample)
    else:
        mbo = int(max_bond_oversample)
    if mbo < 1:
        raise ValueError(f"mps_gate_with_mpo: max_bond_oversample resolves to {mbo}, "
                         "it must be at least 1")
    return mbo
