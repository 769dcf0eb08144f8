"""CPU tier: the label structures of ``tests/label_oracle.py`` on the host
planner (no device).

- The structure x route table: the cheapest grid shape of every structure for
  every route key it reaches, pinned at the H100 SXM's 132 SMs.  Every route
  key of ``route_oracle.required_keys()`` is reached by a structure that is
  not one of the canonical forms, except the pairs the code rules out.
- Plan invariants: M, N, K and batch are the products of the logical extents
  (K over contracted, one-sided and diagonal labels), and the host executor
  of the streaming engine -- the same row code the device runs -- reproduces
  the exact result through the planner's strides: repeated labels add their
  strides, one-sided labels sit in K with stride 0 in the other operand.
- The planner's error codes for invalid signatures.
"""

import numpy as np
import pytest

from quimb_b200 import _lib
from tests import label_oracle as lo
from tests import route_oracle as ro

def _key_str(key):
    return "-".join(str(k) for k in key)


def _table():
    return {name: [[list(k), list(v[:4])] for k, v in sorted(d.items(), key=str)]
            for name, d in lo.coverage().items()}


def test_structure_route_table():
    cov = lo.coverage()
    lines = []
    for name, d in cov.items():
        for key, (M, K, N, eng, r) in sorted(d.items(), key=str):
            G, Ml, Kl, Nl = lo.logical(lo.BY_NAME[name].make(M, K, N))
            lines.append(f"{name:22s} {_key_str(key):30s} G={G} M={Ml} K={Kl} N={Nl} "
                         f"engine={eng}")
    print("\n" + "\n".join(lines))
    sms = {r["sms"] for d in cov.values() for *_, r in d.values()}
    if sms != {132}:
        pytest.skip(f"this device has {sms} SMs; the pinned table is for 132")
    # every required route key is reached by a non-canonical structure
    reached = set().union(*(set(d) for d in cov.values()))
    missing = ro.required_keys() - reached
    assert not missing, sorted(missing, key=str)
    # pairs ruled out by the code are not reached
    for st in lo.STRUCTURES:
        for key in cov[st.name]:
            assert lo.unreachable(st, key) is None, (st.name, key, lo.unreachable(st, key))
    for st in lo.STRUCTURES:
        if st.batch:
            for dt in ("float64", "complex128"):
                assert (dt, "int8") not in cov[st.name]
                assert not any(k[0] == dt and k[1] == "streamk" for k in cov[st.name])
    # no structure moved off its pinned route (or lost one)
    assert _table() == lo.pinned_table()


def test_cfg0_real_feeds_with_multi_mode_k():
    """The large real tile's affine feed and its offset-table feed are both
    reached by a structure whose K group holds several modes."""
    feeds = set()
    for st in lo.STRUCTURES:
        for key, (M, K, N, eng, r) in lo.search(st.name, "float64").items():
            if key[1] in ("plain", "streamk") and key[2] == 0:
                case = st.make(M, K, N)
                if lo.plan_of(case)["n_k"] >= 2:
                    f = lo.feed_of(case, "float64")
                    feeds |= {f["A"], f["B"]}
    assert feeds == {"affine", "table"}, feeds


SHAPES = [(259, 135, 130), (64, 16, 16), (2, 0, 3)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name", [s.name for s in lo.STRUCTURES])
def test_plan_extents_are_the_logical_products(name, shape):
    st = lo.BY_NAME[name]
    M, K, N = shape
    case = st.make(M, K, N if st.has_n else 1)
    G, Ml, Kl, Nl = lo.logical(case)
    plan = lo.plan_of(case)
    if Kl == 0:
        assert plan["degenerate"] == 1   # zero fill
        return
    assert (plan["batch"], plan["M"], plan["K"], plan["N"]) == (G, Ml, Kl, Nl)


def _host_operand(op, values, dtype):
    """Host buffer laid out as `op` (NaN outside the view) and the view."""
    idx = lo.index_map(op)
    reach = np.unique(idx)
    buf = np.full(op.size, np.nan, dtype=dtype)
    buf[reach] = values(reach.size)
    item = buf.itemsize
    view = np.lib.stride_tricks.as_strided(buf[op.offset:], op.shape,
                                           [s * item for s in op.strides])
    return buf, view


def _desc(op, buf, dtype):
    return _lib.np_desc(op.shape, op.strides, ro.QB_DTYPE[dtype],
                        ptr=buf.ctypes.data + op.offset * buf.itemsize)


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
@pytest.mark.parametrize("name", [s.name for s in lo.STRUCTURES])
def test_strides_through_the_host_executor(name, dtype):
    """Integer operands through the streaming engine's host executor: the
    result is exact only when every planned stride is right."""
    st = lo.BY_NAME[name]
    lim = 16
    case = st.make(35, lim, lim if st.has_n else 1)
    rng = np.random.default_rng(len(name))
    vals = lambda n: ro.int_operand(rng, n, dtype)  # noqa: E731
    abuf, xa = _host_operand(case.A, vals, dtype)
    bbuf, xb = _host_operand(case.B, vals, dtype)
    C = lo.out_operand(case, transpose=True)
    cbuf, xc = _host_operand(C, lambda n: np.zeros(n, dtype), dtype)
    for conj_a, conj_b in ((False, False), (True, False), (False, True)):
        if not dtype.startswith("complex") and (conj_a or conj_b):
            continue
        rc = _lib.load().qb_debug_contract_stream_host(
            _desc(case.A, abuf, dtype), _lib.labels(case.la), _desc(case.B, bbuf, dtype),
            _lib.labels(case.lb), _desc(C, cbuf, dtype), _lib.labels(case.lc),
            int(conj_a), int(conj_b), 1.0, 0.0)
        assert rc == 0, _lib.last_error()
        want = lo.reference(case, xa, xb, conj_a, conj_b)
        np.testing.assert_array_equal(xc, want, err_msg=f"conj {conj_a, conj_b}")


def _plan_raw(sa, la, sb, lb, sc, lc):
    return lo.plan_pair(sa, ro.strides(sa), la, sb, ro.strides(sb), lb, sc, ro.strides(sc), lc)


def test_planner_error_codes():
    # a label repeated in the output
    with pytest.raises(ValueError, match=r"code -6\).*repeated in the output"):
        _plan_raw([3, 4], [0, 1], [4, 5], [1, 2], [3, 3], [0, 0])
    # an output label found in neither input
    with pytest.raises(ValueError, match=r"code -6\).*appears in neither input"):
        _plan_raw([3, 4], [0, 1], [4, 5], [1, 2], [3, 5, 2], [0, 2, 9])
    # extent mismatch between A and B, inside A (diagonal), and against C
    with pytest.raises(ValueError, match=r"code -4\).*extent mismatch"):
        _plan_raw([3, 4], [0, 1], [5, 6], [1, 2], [3, 6], [0, 2])
    with pytest.raises(ValueError, match=r"code -2\).*extent mismatch"):
        _plan_raw([3, 4, 5], [0, 1, 1], [5, 6], [1, 2], [3, 6], [0, 2])
    with pytest.raises(ValueError, match=r"code -6\).*extent mismatch"):
        _plan_raw([3, 4], [0, 1], [4, 6], [1, 2], [3, 7], [0, 2])


def test_more_than_twelve_modes_is_refused_by_the_planner():
    """13 non-mergeable modes in one group: the planner refuses the
    signature (contract_pair then regroups the operands)."""
    for repeat in (False, True):
        with pytest.raises(ValueError, match=r"code -100\).*non-mergeable"):
            lo.plan_of(lo.many_modes(repeat))
