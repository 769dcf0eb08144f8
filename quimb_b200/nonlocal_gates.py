"""Apply multi-site, long-range and controlled gates to an MPS on the device
as small MPOs compressed only over the sites they span.

Mirrors, at array level and for open-boundary (l, p, r) site lists,

  MatrixProductOperator.from_dense         tn1d/core.py:4241-4345
  MatrixProductState.gate_with_submpo      tn1d/core.py:2339-2442
  MatrixProductState.gate_nonlocal         tn1d/core.py:2514-2586
  Gate.build_mpo with controls             circuit/gates.py:1123-1152
    fill_empty_sites / add_MPO             tn1d/core.py:4450-4544
  _apply_controlled_gate_mps               circuit/gates.py:819-823

The gate is split into an MPO site by site (device SVD), the MPS is
canonicalised around the span si .. sf of the gate, and the MPS / MPO ladder
of those sites alone is compressed by the 'direct', 'dm' or 'zipup' sweeps of
:mod:`quimb_b200.mpo_compress`.  The ladder's two end bonds, to the rest of
the chain, stay open outer indices; a site inside the span that the gate
does not touch carries the MPO bond past it as an identity, which the sweeps
place as an index expansion of the MPS tensor rather than a contraction.
"""

import numbers

import numpy as np

from . import ops, tebd
from .array import Array
from .mpo_compress import (_BOND_OPTS, _DEFAULT_CUTOFF_MODE, _NOT_BUILT, _direct, _dm,
                           _flip, _flip_mps, _zipup)
from .linalg import norm as _norm
from .mps import mpo_lrud
from .observables import mps_canonicalize
from .split import tensor_split

METHODS = ("direct", "dm", "zipup")


def _check_method(method):
    if method in METHODS:
        return
    if method in ("zipup-first", "zipup-oversample"):
        raise NotImplementedError(
            f"mps_gate_with_submpo: method {method!r} is not implemented on a sub-range "
            "(the reference's own zipup-first fails on a sub-MPO, with KeyError: 'I0')")
    if method == "lazy":
        raise NotImplementedError("mps_gate_with_submpo: method 'lazy' is not implemented "
                                  "(the sites are always (l, p, r) arrays)")
    if any(method == m or method.startswith(m + "-") for m in _NOT_BUILT):
        raise NotImplementedError(f"mps_gate_with_submpo: method {method!r} is not "
                                  f"implemented (available: {', '.join(METHODS)})")
    raise ValueError(f"mps_gate_with_submpo: unknown method {method!r}")


def _sites_of(where, L=None, name="where"):
    where = (int(where),) if isinstance(where, numbers.Integral) else tuple(int(w) for w in where)
    if not where:
        raise ValueError(f"{name}: no sites")
    if len(set(where)) != len(where):
        raise ValueError(f"{name}: repeated site in {where}")
    if min(where) < 0 or (L is not None and max(where) >= L):
        raise ValueError(f"{name}: site out of range in {where} (L = {L})")
    return where


# ---------------------------------------------------------------- from_dense ---
def mpo_from_dense(G, dims=2, sites=None, L=None, **split_opts):
    """``MatrixProductOperator.from_dense`` (tn1d/core.py:4241-4345): the
    dense operator ``G``, reshaped to ``(*dims, *dims)`` (output indices
    first) in the order of ``sites``, split into an MPO one (upper, lower)
    pair at a time in sorted site order with :func:`split.tensor_split`
    (defaults as the reference: ``absorb='right'``, ``cutoff_mode='rsum2'``,
    cutoff 1e-10).

    ``dims``: an int (every site has that dimension, the number of sites is
    log_d(size) / 2) or one dimension per site of ``sites``.  ``L`` only
    bounds the sites.  Returns ``(mpo, sorted_sites)``: one (l, r, u, d)
    device Array per sorted site, end bonds of size 1."""
    tebd.set_default_compress_mode(split_opts)
    split_opts.setdefault("absorb", "right")
    G = ops.asarray(G)
    if isinstance(dims, numbers.Integral):
        ng = int(round(np.log(G.size) / np.log(int(dims)) / 2))
        dims = (int(dims),) * ng
    else:
        dims = tuple(int(d) for d in dims)
        ng = len(dims)
    if ng < 1 or int(np.prod(dims)) ** 2 != G.size:
        raise ValueError(f"mpo_from_dense: an operator of size {G.size} does not fit "
                         f"dims {dims}")
    sites = tuple(range(ng)) if sites is None else _sites_of(sites, L, "mpo_from_dense")
    if len(sites) != ng:
        raise ValueError(f"mpo_from_dense: {len(sites)} sites for {ng} dimensions")
    order = sorted(range(ng), key=lambda k: sites[k])
    T = G.reshape(*dims, *dims)
    inds = [("u", k) for k in range(ng)] + [("d", k) for k in range(ng)]
    out = []
    for n, k in enumerate(order[:-1]):
        rest = order[n + 1:]
        right = [("u", j) for j in rest] + [("d", j) for j in rest]
        left = [ix for ix in inds if ix not in right]
        parts = tensor_split(T, inds, left, right, **split_opts)
        lt, T = parts[0], parts[-1]
        inds = [("b", n)] + right
        if n == 0:                                        # (u, d, b)
            w = lt.reshape(1, *lt.shape).transpose(0, 3, 1, 2)
        else:                                             # (b', u, d, b)
            w = lt.transpose(0, 3, 1, 2)
        out.append(ops.materialize(w))
    if ng == 1:
        w = T.reshape(1, 1, *T.shape)
    else:                                                 # (b, u, d)
        w = T.reshape(*T.shape[:1], 1, *T.shape[1:])
    out.append(ops.materialize(w, force=True))
    return out, sorted(sites)


# ------------------------------------------------------------ gate_with_submpo ---
def _prepare(psi, submpo, present, mpo_shape, transpose):
    """The ladder of sites si .. sf: MPS views and MPO sites W[wl, wr, o, p]
    (o the output index) with, at a gap site, the int size of the bond
    passing it; one common dtype."""
    n = len(present)
    if len(submpo) != n:
        raise ValueError(f"mps_gate_with_submpo: the MPO has {len(submpo)} sites, "
                         f"where {n}")
    si, sf = present[0], present[-1]
    A = psi[si:sf + 1]
    Wp = []
    for k, s in enumerate(present):
        w = mpo_lrud(submpo[k], mpo_shape, k, n)
        w = w.transpose(0, 1, 3, 2) if transpose else w
        if w.shape[3] != A[s - si].shape[1]:
            raise ValueError(f"mps_gate_with_submpo: site {s} has physical dimension "
                             f"{A[s - si].shape[1]}, the MPO index meeting it {w.shape[3]}")
        if k and Wp[-1].shape[1] != w.shape[0]:
            raise ValueError(f"mps_gate_with_submpo: MPO bond mismatch between sites "
                             f"{present[k - 1]} and {s}")
        Wp.append(w)
    if Wp[0].shape[0] != 1 or Wp[-1].shape[1] != 1:
        raise ValueError("mps_gate_with_submpo: open-boundary MPO only")
    W, k = [], 0
    for s in range(si, sf + 1):
        if s == present[k]:
            W.append(Wp[k])
            k += 1
        else:
            W.append(int(Wp[k - 1].shape[1]))
    dt = np.result_type(*[x.dtype for x in A + Wp])
    A = [a.astype(dt, copy=False) for a in A]
    W = [w if isinstance(w, int) else w.astype(dt, copy=False) for w in W]
    return A, W, dt


def mps_gate_with_submpo(sites, submpo, where, method="direct", transpose=False, info=None,
                         max_bond=None, cutoff=1e-10, cutoff_mode=None, normalize=False,
                         sweep_reverse=False, canonize=True, mpo_shape="lrud",
                         equalize_norms=False, **split_opts):
    """``MatrixProductState.gate_with_submpo`` (tn1d/core.py:2339-2442) for
    open-boundary (l, p, r) device sites: the MPO ``submpo``, one site array
    (layout ``mpo_shape``) per site of ``sorted(where)``, applied and the
    result compressed over sites si = min(where) .. sf = max(where) only.

    The MPS is first canonicalised around (si, sf) by
    :func:`observables.mps_canonicalize`, starting from
    ``info["cur_orthog"]`` (so a centre already inside the range costs
    nothing).  ``method`` is 'direct' (default), 'dm' or 'zipup', with the
    options and defaults of :func:`mpo_compress.mps_gate_with_mpo`; 'zipup'
    truncates in the pseudo-canonical gauge of the sub-range network the
    reference builds.  By default the MPO's lower index meets the MPS,
    ``transpose`` contracts the upper one.

    Returns a new list: sites outside si .. sf are the caller's arrays unless
    the canonicalisation moved them; si .. sf are new arrays in the promoted
    dtype, right-canonical with the centre at si (left-canonical, centre sf,
    with ``sweep_reverse``), recorded in ``info["cur_orthog"]``.  The
    caller's list and arrays are not modified."""
    _check_method(method)
    if equalize_norms:
        raise NotImplementedError("mps_gate_with_submpo: equalize_norms is not implemented")
    psi = list(sites)
    L = len(psi)
    if L == 0:
        raise ValueError("mps_gate_with_submpo: empty MPS")
    present = sorted(_sites_of(where, L, "mps_gate_with_submpo"))
    if cutoff_mode is None:
        cutoff_mode = _DEFAULT_CUTOFF_MODE[method]
    opts = dict(split_opts, max_bond=max_bond, cutoff=cutoff, cutoff_mode=cutoff_mode)
    if method == "direct":
        extra = sorted(set(split_opts) - _BOND_OPTS)
        if extra:
            raise TypeError(f"mps_gate_with_submpo: method 'direct' does not take the split "
                            f"option(s) {extra}")
    si, sf = present[0], present[-1]
    if info is None:
        info = {}
    mps_canonicalize(psi, (si, sf), info)
    A, W, dt = _prepare(psi, submpo, present, mpo_shape, transpose)
    if method == "zipup":
        span = dict(open_ends=(si > 0, sf < L - 1), rung_between=True)
        out = _zipup(A, W, canonize, sweep_reverse, opts, span)
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
    c = sf if sweep_reverse else si
    if normalize:
        x = ops.materialize(out[c - si], force=True)
        out[c - si] = ops.scale_(x, 1.0, div_by=_norm(x))
    psi[si:sf + 1] = [ops.materialize(x).astype(dt, copy=False) for x in out]
    info["cur_orthog"] = (c, c)
    return psi


def mps_gate_nonlocal(sites, G, where, dims=None, method="direct", transpose=False,
                      info=None, **compress_opts):
    """``MatrixProductState.gate_nonlocal`` (tn1d/core.py:2514-2586): the
    dense gate ``G`` on sites ``where`` (any order, any distance; index order
    (out..., in...) in the order of ``where``) as :func:`mpo_from_dense`,
    then :func:`mps_gate_with_submpo`.  ``dims`` defaults to the sites'
    physical dimensions; ``transpose`` applies G^T."""
    L = len(sites)
    where = _sites_of(where, L, "mps_gate_nonlocal")
    if dims is None:
        dims = tuple(int(ops.asarray(sites[i]).shape[1]) for i in where)
    mpo, _ = mpo_from_dense(G, dims=dims, sites=where, L=L)
    return mps_gate_with_submpo(sites, mpo, where, method=method, transpose=transpose,
                                info=info, **compress_opts)


# ---------------------------------------------------------- controlled gates ---
def _block(x, y, first, last):
    """The direct sum of two MPO sites over their bonds (add_MPO): a row of
    blocks on the first site, a column on the last, block-diagonal between."""
    import torch
    xt, yt = x.resolve(), y.resolve()
    if first:
        return Array(torch.cat([xt, yt], dim=1))
    if last:
        return Array(torch.cat([xt, yt], dim=0))
    (l1, r1, u, d), (l2, r2, _, _) = xt.shape, yt.shape
    z = torch.zeros((l1 + l2, r1 + r2, u, d), dtype=xt.dtype, device=xt.device)
    z[:l1, :r1] = xt
    z[l1:, r1:] = yt
    return Array(z)


def _controlled_mpo(G, dims, qubits, controls, dtype, device):
    """``Gate.build_mpo`` with controls (circuit/gates.py:1123-1152): the MPO
    of (G - 1) on the targets, |1><1| on every control (a control between two
    targets carries their bond past it), plus the identity on all those
    sites; (l, r, u, d) arrays on ``sorted(qubits + controls)``."""
    import torch
    size = int(np.prod(dims))
    Gh = np.asarray(G.to_numpy() if hasattr(G, "to_numpy") else G).reshape(size, size)
    Gh = (Gh - np.eye(size)).astype(np.result_type(Gh.dtype, dtype))
    tmpo, tsites = mpo_from_dense(ops.asarray(Gh, device=device), dims=dims, sites=qubits)
    dt = tmpo[0].t.dtype
    allsites = sorted(qubits + controls)
    p1 = torch.zeros((2, 2), dtype=dt, device=device)
    p1[1, 1] = 1
    n = len(allsites)
    out = []
    k = 0
    for m, s in enumerate(allsites):
        if s in tsites:
            w = tmpo[k].resolve()
            k += 1
        else:
            # the bond between the targets either side, 1 outside them
            D = tmpo[k - 1].shape[1] if 0 < k < len(tsites) else 1
            w = torch.eye(D, dtype=dt, device=device)[:, :, None, None] * p1
        d = w.shape[2]
        ident = torch.eye(d, dtype=dt, device=device).reshape(1, 1, d, d)
        out.append(_block(Array(w), Array(ident), m == 0, m == n - 1) if n > 1
                   else Array(w + ident))
    return out, allsites


def mps_gate_controlled(sites, G, qubits, controls, **gate_opts):
    """A multi-controlled gate: ``G`` on the target sites ``qubits`` (index
    order (out..., in...)), applied where every site of ``controls`` is
    |1>, as the reference's CircuitMPS applies one (circuit/gates.py:819-823):
    the controlled MPO of ``Gate.build_mpo`` (bond dimension that of the
    (G - 1) MPO plus one) through :func:`mps_gate_with_submpo` on
    ``sorted(controls + qubits)``.  Control sites must be qubits;
    ``gate_opts`` go to :func:`mps_gate_with_submpo`."""
    L = len(sites)
    qubits = list(_sites_of(qubits, L, "mps_gate_controlled"))
    controls = list(_sites_of(controls, L, "mps_gate_controlled"))
    if set(qubits) & set(controls):
        raise ValueError("mps_gate_controlled: a site is both target and control")
    A = [ops.asarray(sites[i]) for i in qubits + controls]
    if any(a.shape[1] != 2 for a in A[len(qubits):]):
        raise ValueError("mps_gate_controlled: control sites must have dimension 2")
    dims = tuple(a.shape[1] for a in A[:len(qubits)])
    dtype = np.result_type(*[a.dtype for a in A])
    mpo, allsites = _controlled_mpo(G, dims, qubits, controls, dtype, A[0].device)
    return mps_gate_with_submpo(sites, mpo, allsites, **gate_opts)
