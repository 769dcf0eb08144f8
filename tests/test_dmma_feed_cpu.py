"""The affine operand feed of the 128x128 fp64 DMMA tile (no GPU needed).

The planner proves, per operand, that every row of a tile and every k-block
sits at a constant stride from the tile's base; such an operand is gathered
from one per-thread address advanced by constant steps instead of the
per-tile offset tables.  ``feed_pair`` reports the choice; these tests pin it
for the shapes the MPS-norm benchmark and the DMRG matvec run, and pin the
table feed for layouts the proof must reject.  The affine kernels must not
spill more than the table kernels they replace.
"""

import re
import shutil
import subprocess

import pytest

import quimb_b200 as qb
from quimb_b200 import _lib

CHI, D, W = 1024, 2, 5
LB, L, P, R, RB = 0, 1, 2, 3, 4


def _strides(shape):
    st, acc = [], 1
    for s in reversed(shape):
        st.append(acc)
        acc *= s
    return list(reversed(st))


def _feed(sa, sta, la, sb, stb, lb, sc, lc):
    r = qb.route_pair(sa, sta, la, sb, stb, lb, sc, _strides(sc), lc)
    return qb.feed_pair(sa, sta, la, sb, stb, lb, sc, _strides(sc), lc), r


# an "lrp" site viewed as (l, p, r): what mps.norm_step contracts
SITE = ([CHI, D, CHI], [CHI * D, 1, D])


def test_mps_norm_ket_step_is_affine():
    # E[a', a] . A[a, p, b] -> T[a', p, b]: n = (p, b) is one run in the site
    f, r = _feed([CHI, CHI], [CHI, 1], [LB, L], *SITE, [L, P, R], [CHI, D, CHI], [LB, P, R])
    assert (r["kind"], r["cfg"]) == ("dmma", 0)
    assert f == {"A": "affine", "B": "affine"}


def test_mps_norm_bra_step_is_affine():
    # conj(A)[a', p, b'] . T[a', p, b] -> E'[b', b]: k = (p, a') is a run of
    # 16-byte pairs in the site and a run of elements in T
    f, r = _feed(*SITE, [LB, P, RB], [CHI, D, CHI], _strides([CHI, D, CHI]), [LB, P, R],
                 [CHI, CHI], [RB, R])
    assert (r["kind"], r["cfg"], r["layout"]) == ("dmma_streamk", 0, 2)
    assert f == {"A": "affine", "B": "affine"}


def test_dmrg_matvec_is_affine():
    # L[a, w, b] . x[b, p, q, c] -> (a, w, p, q, c)
    sa, sb, sc = [CHI, W, CHI], [CHI, D, D, CHI], [CHI, W, D, D, CHI]
    f, r = _feed(sa, _strides(sa), [0, 1, 2], sb, _strides(sb), [2, 3, 4, 5], sc,
                 [0, 1, 3, 4, 5])
    assert (r["kind"], r["cfg"]) == ("dmma", 0)
    assert f == {"A": "affine", "B": "affine"}


def test_row_group_with_a_gap_inside_a_tile_uses_tables():
    # A[m1, m2, k] with m2 (64 rows) padded to 66: a 128-row tile spans the gap
    K, N = 1024, 2048
    sa = [16, 64, K]
    f, r = _feed(sa, [66 * K, K, 1], [0, 1, 2], [K, N], [N, 1], [2, 3], [16, 64, N],
                 [0, 1, 3])
    assert (r["kind"], r["cfg"]) == ("dmma", 0)
    assert f == {"A": "table", "B": "affine"}


def test_k_group_with_a_short_fastest_mode_uses_tables():
    # k = (k0 of extent 3, k1) with a gap behind k0 in A: a 32-deep k-block
    # crosses k0's boundary at a different place in every block
    M, N, K1 = 1024, 2048, 352
    f, r = _feed([M, K1, 3], [K1 * 4, 4, 1], [0, 1, 2], [K1, 3, N], [3 * N, N, 1], [1, 2, 3],
                 [M, N], [0, 3])
    assert (r["kind"], r["cfg"]) == ("dmma", 0)
    assert f == {"A": "table", "B": "affine"}


def test_ragged_tiles_and_complex_use_tables():
    # M not a multiple of the tile: the last tile's rows need predicates
    n = 1000
    f, r = _feed([n, 4096], [4096, 1], [0, 1], [4096, 2048], [2048, 1], [1, 2], [n, 2048], [0, 2])
    assert r["cfg"] == 0 and f["A"] == "table" and f["B"] == "affine"
    s = [1024, 1024]
    f = qb.feed_pair(s, _strides(s), [0, 1], s, _strides(s), [1, 2], s, _strides(s), [0, 2],
                     _lib.QB_C128)
    assert f == {"A": None, "B": None}


def _resource_usage():
    _lib.load()
    out = subprocess.run([shutil.which("cuobjdump"), "-res-usage", _lib.LIB_PATH],
                         capture_output=True, text=True, check=True).stdout
    usage, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name:
            usage[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    return usage


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not found")
def test_affine_tiles_do_not_spill():
    pat = re.compile(r"_ZN2qb(26contract_f64_affine_kernel|34contract_f64_affine_streamk_kernel)"
                     r"ILi128ELi128ELi32ELi2ELi4ELi3E")
    aff = {n: u for n, u in _resource_usage().items() if pat.match(n)}
    # 4 layouts x 3 feeds (A, B, both affine) x 2 launch modes
    assert len(aff) == 24, sorted(aff)
    assert all(reg <= 255 for reg, _ in aff.values())
    # the classic launch keeps everything in registers; the stream-K one
    # stays below the 96 B its table kernel keeps on the stack
    limit = {"26contract_f64_affine_kernel": 0, "34contract_f64_affine_streamk_kernel": 32}
    over = {n: u for n, u in aff.items() if u[1] > limit[pat.match(n).group(1)]}
    assert not over, f"(registers, stack bytes) of spilling kernels: {over}"
