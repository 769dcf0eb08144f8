"""Pairwise contraction front-end over the C ABI.

``contract_pair`` is the single primitive that ``tensordot`` / ``einsum`` /
the tree executor lower to: it never transposes or copies an operand, the
permutation implied by the labels is folded into the CUDA kernel's tile
loads (see ``csrc/contract_dmma.cu``).
"""

import ctypes

import torch

from . import _lib

_WS = {}


def _workspace(nbytes, device):
    """Grow-only per-(device, stream) scratch buffer.  Allocated zeroed and
    handed to nothing but the contraction entry points, which keep its 1 KiB
    header (stream-K flag words) zero -- the QB_ENGINE_WS_ZEROED contract."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _WS.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.zeros(max(int(nbytes), 1 << 20), dtype=torch.uint8,
                          device=device)
        _WS[key] = buf
    return buf


def _scratch_dicts():
    """Every per-(device, stream) scratch cache of the package; keys end with
    the stream handle."""
    from . import lanczos, linalg, ops
    return (_WS, linalg._WS, ops._DOT_WS, lanczos._MD_WS)


def capture_graph(fn):
    """Capture ``fn()`` into a CUDA graph that owns its scratch; returns
    ``(graph, value of the captured call, scratch buffers)``.

    ``fn`` first runs eagerly on a new side stream and is then captured on
    that same stream, so every scratch buffer the captured launches use is
    allocated (and its zero fill has run) before capture begins.  Those
    buffers are then taken out of the per-stream caches: the caller keeps
    them alive with the graph, and no later eager call or capture -- torch
    recycles stream handles -- can reach them."""
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.Stream(device=dev)
    st.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(st):
        fn()                              # warm-up: scratch, kernel attributes
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        out = fn()
    scratch = []
    for d in _scratch_dicts():
        for key in [k for k in d if k[-1] == st.cuda_stream]:
            scratch.append(d.pop(key))
    return graph, out, scratch


_WIDE = {torch.float32: torch.float64, torch.complex64: torch.complex128}


def convert(t, dtype):
    """Contiguous copy of ``t`` in another precision through ``qb_convert``
    (strided inputs are first materialised by the permute kernel)."""
    _lib.require_cuda(t)
    if t.dtype == dtype:
        return t
    if not t.is_contiguous():
        src = torch.empty(t.shape, dtype=t.dtype, device=t.device)
        rc = _lib.load().qb_permute(_lib.desc(t), _lib.desc(src), 0, _lib.stream_ptr())
        _lib.check(rc, "qb_permute")
        t = src
    out = torch.empty(t.shape, dtype=dtype, device=t.device)
    rc = _lib.load().qb_convert(_lib.qb_dtype(t.dtype), _lib.qb_dtype(dtype), t.numel(),
                                t.data_ptr(), out.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "qb_convert")
    return out


def contract_pair(a, la, b, lb, lc, conj_a=False, conj_b=False, out=None,
                  engine=0, alpha=1.0, beta=0.0, _regrouped=False):
    """``out[lc] = sum op(a)[la] * op(b)[lb]`` with integer mode labels.

    Parameters
    ----------
    a, b : torch.Tensor (cuda)
        Arbitrarily strided views; never copied.
    la, lb, lc : sequences of int
        Mode labels of ``a``, ``b`` and the output (its axis order).
    out : torch.Tensor, optional
        Pre-allocated (possibly strided) output view.
    alpha, beta : float
        ``out = alpha * contraction + beta * out`` (beta != 0 needs ``out``).
    """
    _lib.require_cuda(a, "a")
    _lib.require_cuda(b, "b")
    if a.dtype != b.dtype:
        raise TypeError(f"dtype mismatch: {a.dtype} vs {b.dtype}")
    if len(la) != a.dim() or len(lb) != b.dim():
        raise ValueError("label count does not match operand rank")
    if a.dtype in _WIDE and not _native_single(a, la, b, lb, lc, out, engine):
        # single precision below the int8 engine's tile minimum (or with
        # batch modes): widen exactly, contract in fp64, round once
        wide = _WIDE[a.dtype]
        wout = None if out is None else convert(out, wide)
        res = contract_pair(convert(a, wide), la, convert(b, wide), lb, lc, conj_a,
                            conj_b, wout, engine, alpha, beta)
        narrow = convert(res, a.dtype)
        if out is not None:
            rc = _lib.load().qb_permute(_lib.desc(narrow), _lib.desc(out), 0,
                                        _lib.stream_ptr())
            _lib.check(rc, "qb_permute")
            return out
        return narrow
    lib = _lib.load()
    ext = {}
    for t, ls in ((a, la), (b, lb)):
        for l, s in zip(ls, t.shape):
            if ext.setdefault(l, s) != s:
                raise ValueError(
                    f"extent mismatch for label {l}: {ext[l]} vs {s}")
    if out is None:
        try:
            shape = [ext[l] for l in lc]
        except KeyError as e:
            raise ValueError(f"output label {e} appears in neither input")
        out = torch.empty(shape, dtype=a.dtype, device=a.device)
    else:
        _lib.require_cuda(out, "out")
    da, db, dc = _lib.desc(a), _lib.desc(b), _lib.desc(out)
    pla, plb, plc = _lib.labels(la), _lib.labels(lb), _lib.labels(lc)
    need = lib.qb_contract_pair_workspace(da, pla, db, plb, dc, plc, engine)
    if need == -100 and not _regrouped and "non-mergeable" in _lib.last_error():
        # more than 12 jointly non-mergeable modes in one group (high-rank
        # operands whose axes interleave: boundary / compression drivers on
        # tensors of rank > 12): regroup the operands once with the permute
        # kernel so that every group is a single contiguous mode
        return _contract_regrouped(a, la, b, lb, lc, conj_a, conj_b, out, engine, alpha, beta)
    if need < 0:
        _lib.check(int(need), "qb_contract_pair_workspace")
    ws_ptr, ws_n = None, 0
    if need > 0:
        ws = _workspace(need, a.device)
        ws_ptr, ws_n = ctypes.c_void_p(ws.data_ptr()), ws.numel()
    if alpha == 1.0 and beta == 0.0:
        rc = lib.qb_contract_pair(da, pla, db, plb, dc, plc, int(bool(conj_a)),
                                  int(bool(conj_b)), engine | _lib.QB_ENGINE_WS_ZEROED,
                                  ws_ptr, ws_n, _lib.stream_ptr())
    else:
        rc = lib.qb_contract_pair_ab(da, pla, db, plb, dc, plc,
                                     int(bool(conj_a)), int(bool(conj_b)),
                                     float(alpha), float(beta), ws_ptr, ws_n,
                                     _lib.stream_ptr())
    _lib.check(rc, "qb_contract_pair")
    return out


_NO_NATIVE_SINGLE = -101


def _native_single(a, la, b, lb, lc, out, engine):
    """True when the library takes this float32 / complex64 contraction on its
    native engine (int8 wgmma, 4 slices, float epilogue -- csrc/ozaki_tc.cu);
    decided by the library's own planner, so the rule lives in one place."""
    ext = {}
    for t, ls in ((a, la), (b, lb)):
        if len(ls) != t.dim():
            return False
        for l, s in zip(ls, t.shape):
            if ext.setdefault(l, s) != s:
                return False
    if any(l not in ext for l in lc):
        return False
    if out is None:
        shape = [ext[l] for l in lc]
        st, acc = [], 1
        for e in reversed(shape):
            st.append(acc)
            acc *= max(e, 1)
        dc = _lib.np_desc(shape, list(reversed(st)), _lib.qb_dtype(a.dtype))
    else:
        dc = _lib.desc(out)
    need = _lib.load().qb_contract_pair_workspace(_lib.desc(a), _lib.labels(la), _lib.desc(b),
                                                  _lib.labels(lb), dc, _lib.labels(lc), engine)
    return need != _NO_NATIVE_SINGLE and need >= 0


_CHUNK = 5


def permute_modes(t):
    """Number of modes the permute kernel sees when ``t`` (any strided view) is
    copied into a contiguous tensor of the same axis order: axes of extent > 1,
    ordered by destination stride, neighbours merged when they are jointly
    contiguous in source and destination (mirrors qb_permute's host logic,
    csrc/elementwise.cu; the kernel takes 17, or 18 when the fastest source
    mode differs from the fastest destination mode)."""
    dims = [(t.shape[i], t.stride(i)) for i in range(t.dim()) if t.shape[i] > 1]
    ds, acc = [], 1
    for e, _ in reversed(dims):
        ds.append(acc)
        acc *= e
    ds.reverse()
    ms = sorted(((e, ss, d) for (e, ss), d in zip(dims, ds)), key=lambda m: m[2])
    n, last = 0, None
    for e, ss, d in ms:
        if last is not None and ss == last[1] * last[0] and d == last[2] * last[0]:
            last = (last[0] * e, last[1], last[2])
            continue
        n += 1
        last = (e, ss, d)
    return n


PERMUTE_MAX_MODES = 17   # 16 generic modes + the fastest destination mode (+1 more when a distinct fastest source mode exists)


def permute_contiguous(t, order, conj=False):
    """Contiguous tensor whose axis k is axis ``order[k]`` of ``t``, for any
    rank: the permute kernel takes up to 15 jointly non-mergeable modes, so a
    general permutation of a high-rank tensor is done in passes that each move
    ``_CHUNK`` axes behind the rest (<= 2 * _CHUNK + 2 modes per pass)."""
    lib = _lib.load()

    def one_pass(src, perm, cj=False):
        view = src.permute(tuple(perm))
        dst = torch.empty(view.shape, dtype=src.dtype, device=src.device)
        if dst.numel():
            rc = lib.qb_permute(_lib.desc(view), _lib.desc(dst), int(cj), _lib.stream_ptr())
            _lib.check(rc, "qb_permute")
        return dst

    order = list(order)
    r = t.dim()
    if r <= 2 * _CHUNK:
        return one_pass(t, order, conj)
    # start from a copy laid out in the source's own stride order (few modes);
    # a lazy conjugation is applied in this first pass
    by_stride = sorted(range(r), key=lambda ax: (-abs(t.stride(ax)), ax))
    cur = one_pass(t, by_stride, conj)
    names = list(by_stride)                   # names[k] = original axis held by cur's axis k
    placed = 0
    while placed < r:
        chunk = order[max(0, r - placed - _CHUNK): r - placed]
        tail = order[r - placed:]
        rest = [ax for ax in names if ax not in chunk and ax not in tail]
        new = rest + chunk + tail
        if new != names:
            cur = one_pass(cur, [names.index(ax) for ax in new])
            names = new
        placed += len(chunk)
    return cur


def _contract_regrouped(a, la, b, lb, lc, conj_a, conj_b, out, engine, alpha, beta):
    la, lb, lc = list(la), list(lb), list(lc)
    if len(set(la)) != len(la) or len(set(lb)) != len(lb):
        raise ValueError("contract_pair: too many non-mergeable modes and a repeated "
                         "label inside one operand; take the diagonal first")
    sa, sb, sc = set(la), set(lb), set(lc)
    batch = [l for l in lc if l in sa and l in sb]
    free_a = [l for l in lc if l in sa and l not in sb]
    free_b = [l for l in lc if l in sb and l not in sa]
    k = [l for l in la if l in sb and l not in sc]
    sum_a = [l for l in la if l not in sb and l not in sc]
    sum_b = [l for l in lb if l not in sa and l not in sc]
    la2 = batch + free_a + k + sum_a
    lb2 = batch + k + sum_b + free_b
    lc2 = batch + free_a + free_b
    a2 = permute_contiguous(a, [la.index(l) for l in la2])
    b2 = permute_contiguous(b, [lb.index(l) for l in lb2])
    if out is None:
        res = contract_pair(a2, la2, b2, lb2, lc2, conj_a, conj_b, None, engine, alpha, beta,
                            _regrouped=True)
        return res.permute(tuple(lc2.index(l) for l in lc))   # a view in the requested order
    if beta != 0.0:
        cur = permute_contiguous(out, [lc.index(l) for l in lc2])
        res = contract_pair(a2, la2, b2, lb2, lc2, conj_a, conj_b, cur, engine, alpha, beta,
                            _regrouped=True)
    else:
        res = contract_pair(a2, la2, b2, lb2, lc2, conj_a, conj_b, None, engine, alpha, 0.0,
                            _regrouped=True)
    final = permute_contiguous(res, [lc2.index(l) for l in lc])
    rc = _lib.load().qb_permute(_lib.desc(final), _lib.desc(out), 0, _lib.stream_ptr())
    _lib.check(rc, "qb_permute")
    return out


def plan_pair(a_shape, a_strides, la, b_shape, b_strides, lb, c_shape,
              c_strides, lc, dtype_code=_lib.QB_F64):
    """Host-only: the GEMM view the C planner derives (no GPU needed)."""
    lib = _lib.load()
    da = _lib.np_desc(a_shape, a_strides, dtype_code)
    db = _lib.np_desc(b_shape, b_strides, dtype_code)
    dc = _lib.np_desc(c_shape, c_strides, dtype_code)
    out = (ctypes.c_int64 * 16)()
    rc = lib.qb_contract_pair_plan(da, _lib.labels(la), db, _lib.labels(lb),
                                   dc, _lib.labels(lc), out)
    _lib.check(rc, "qb_contract_pair_plan")
    keys = ("M", "N", "K", "batch", "n_m", "n_n", "n_k", "n_b", "cfg",
            "splitk", "vecA", "vecB", "vecC", "thrA", "thrB", "degenerate")
    return dict(zip(keys, list(out)))


ROUTE_KINDS = ("empty", "zero_fill", "widen", "int8", "stream", "dmma", "dmma_streamk")


def route_pair(a_shape, a_strides, la, b_shape, b_strides, lb, c_shape,
               c_strides, lc, dtype_code=_lib.QB_F64, engine=0, ptrs=None):
    """Host-only: the kernel route ``contract_pair`` takes for operands of
    these shapes and strides (the library's own dispatch decision, at the SM
    count of the current device or the H100 SXM's 132 without one).

    ``ptrs`` = (a, b, c) base addresses; the vector loads depend on 16-byte
    alignment, so pass the real ones when the route of a view matters.

    A streaming-engine route (kind ``"stream"``) also carries ``stream_k`` /
    ``stream_n``, the compiled (KMAX, NMAX) variant it launches; other routes
    have no variant and do not carry these keys."""
    lib = _lib.load()
    pa, pb, pc = ptrs if ptrs is not None else (0x10000000,) * 3
    da = _lib.np_desc(a_shape, a_strides, dtype_code, pa)
    db = _lib.np_desc(b_shape, b_strides, dtype_code, pb)
    dc = _lib.np_desc(c_shape, c_strides, dtype_code, pc)
    out = (ctypes.c_int64 * 16)()
    rc = lib.qb_contract_pair_route(da, _lib.labels(la), db, _lib.labels(lb),
                                    dc, _lib.labels(lc), int(engine), out)
    _lib.check(rc, "qb_contract_pair_route")
    keys = ("kind", "cfg", "splitk", "streamk", "sk_head", "bk", "layout", "sms",
            "launches")
    r = dict(zip(keys, list(out)))
    r["kind"] = ROUTE_KINDS[r["kind"]]
    if r["kind"] == "stream":
        r["stream_k"], r["stream_n"] = out[9], out[10]
    return r


FEEDS = {1: "affine", 0: "table", -1: None}


def feed_pair(a_shape, a_strides, la, b_shape, b_strides, lb, c_shape,
              c_strides, lc, dtype_code=_lib.QB_F64, ptrs=None):
    """Host-only: how ``contract_pair`` (engine auto) gathers each operand
    into the large real DMMA tile: ``"affine"`` (each thread's copies follow
    constant strides, no offset tables), ``"table"`` (per-tile offset tables)
    or None when the route does not run that tile.  ``ptrs`` as for
    ``route_pair``."""
    lib = _lib.load()
    pa, pb, pc = ptrs if ptrs is not None else (0x10000000,) * 3
    da = _lib.np_desc(a_shape, a_strides, dtype_code, pa)
    db = _lib.np_desc(b_shape, b_strides, dtype_code, pb)
    dc = _lib.np_desc(c_shape, c_strides, dtype_code, pc)
    out = (ctypes.c_int64 * 2)()
    rc = lib.qb_contract_pair_feed(da, _lib.labels(la), db, _lib.labels(lb),
                                   dc, _lib.labels(lc), out)
    _lib.check(rc, "qb_contract_pair_feed")
    return {"A": FEEDS[out[0]], "B": FEEDS[out[1]]}


SCHEDULES = {1: "pair", 0: "segments", -1: None}


def schedule_pair(a_shape, a_strides, la, b_shape, b_strides, lb, c_shape,
                  c_strides, lc, dtype_code=_lib.QB_F64, ptrs=None):
    """Host-only: how the stream-K grid of ``route_pair`` (engine auto) runs:
    ``"pair"`` (2-CTA clusters, one per tile, each CTA one k-half, the halves
    summed in distributed shared memory), ``"segments"`` (equal-cost k-block
    ranges, partial tiles summed through the workspace) or None when the
    route is not stream-K.  Without a device, half the grid is assumed to fit
    as clusters at once.  ``ptrs`` as for ``route_pair``."""
    lib = _lib.load()
    pa, pb, pc = ptrs if ptrs is not None else (0x10000000,) * 3
    da = _lib.np_desc(a_shape, a_strides, dtype_code, pa)
    db = _lib.np_desc(b_shape, b_strides, dtype_code, pb)
    dc = _lib.np_desc(c_shape, c_strides, dtype_code, pc)
    out = (ctypes.c_int64 * 1)()
    rc = lib.qb_contract_pair_schedule(da, _lib.labels(la), db, _lib.labels(lb),
                                       dc, _lib.labels(lc), out)
    _lib.check(rc, "qb_contract_pair_schedule")
    return SCHEDULES[out[0]]


def contract_batched(a_list, la, b_list, lb, lc, conj_a=False, conj_b=False):
    """Many independent contractions of identical signature in ONE launch
    (the small same-shape intermediates of MPS / PEPS / circuit sweeps).

    ``a_list[i]``, ``b_list[i]`` must share shape, strides and dtype across
    ``i``; returns the list of outputs (views of one allocation)."""
    if len(a_list) != len(b_list) or not a_list:
        raise ValueError("contract_batched: need equally many a and b operands")
    a0, b0 = a_list[0], b_list[0]
    for a, b in zip(a_list, b_list):
        _lib.require_cuda(a, "a")
        _lib.require_cuda(b, "b")
        if (a.shape != a0.shape or a.stride() != a0.stride() or a.dtype != a0.dtype
                or b.shape != b0.shape or b.stride() != b0.stride() or b.dtype != a0.dtype):
            raise ValueError("contract_batched: operands must share shape, "
                             "strides and dtype")
    lib = _lib.load()
    ext = {}
    for t, ls in ((a0, la), (b0, lb)):
        for l, s in zip(ls, t.shape):
            ext[l] = s
    shape = [ext[l] for l in lc]
    n = len(a_list)
    out = torch.empty([n] + shape, dtype=a0.dtype, device=a0.device)
    # representative descriptors carry the weakest pointer alignment
    def rep_ptr(ts):
        p = 0
        for t in ts:
            p |= t.data_ptr()
        low = p & 15
        return ts[0].data_ptr() if low == 0 else (ts[0].data_ptr() | low)
    da = _lib.desc(a0, rep_ptr(a_list))
    db = _lib.desc(b0, rep_ptr(b_list))
    dc = _lib.desc(out[0])
    ptrs = torch.tensor([[t.data_ptr() for t in a_list],
                         [t.data_ptr() for t in b_list],
                         [out[i].data_ptr() for i in range(n)]],
                        dtype=torch.int64).to(a0.device)
    rc = lib.qb_contract_batched(da, _lib.labels(la), db, _lib.labels(lb), dc,
                                 _lib.labels(lc), ptrs[0].data_ptr(),
                                 ptrs[1].data_ptr(), ptrs[2].data_ptr(), n,
                                 int(bool(conj_a)), int(bool(conj_b)),
                                 _lib.stream_ptr())
    _lib.check(rc, "qb_contract_batched")
    ptrs.record_stream(torch.cuda.current_stream())
    return [out[i] for i in range(n)]
