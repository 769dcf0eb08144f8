"""The stream-K pair schedule of the 128x128 fp64 DMMA tile (no GPU needed).

A stream-K grid with at most half as many tiles as CTAs runs as 2-CTA
clusters, one tile per cluster and one k-half per CTA, instead of the
equal-cost segment loop.  ``schedule_pair`` reports the choice; these tests
pin it for the MPS-norm benchmark's bra step, for a stream-K shape with too
many tiles, and for a shape that is not stream-K.  The pair kernels must not
spill.
"""

import re
import shutil
import subprocess

import pytest

import quimb_b200 as qb
from quimb_b200 import _lib

CHI, D = 1024, 2


def _strides(shape):
    st, acc = [], 1
    for s in reversed(shape):
        st.append(acc)
        acc *= s
    return list(reversed(st))


def _schedule(sa, sta, la, sb, stb, lb, sc, lc, dtype=_lib.QB_F64):
    args = (sa, sta, la, sb, stb, lb, sc, _strides(sc), lc, dtype)
    return qb.schedule_pair(*args), qb.route_pair(*args)


def _gemm(M, N, K, dtype=_lib.QB_F64):
    return _schedule([M, K], [K, 1], [0, 1], [K, N], [N, 1], [1, 2], [M, N], [0, 2], dtype)


def _need_132_sms(r):
    if r["sms"] != 132:
        pytest.skip(f"this device has {r['sms']} SMs; the pinned schedules are for 132")


def test_mps_norm_bra_step_runs_the_pair_schedule():
    # contiguous operands, as test_host_cpu pins the route
    s, r = _schedule([CHI, D, CHI], _strides([CHI, D, CHI]), [0, 1, 2],
                     [CHI, D, CHI], _strides([CHI, D, CHI]), [0, 1, 3], [CHI, CHI], [2, 3])
    _need_132_sms(r)
    assert (r["kind"], r["streamk"], r["sk_head"]) == ("dmma_streamk", 132, 4)
    assert s == "pair"
    # an "lrp" site viewed as (l, p, r), as the benchmark contracts it
    LB, P, R, RB = 0, 2, 3, 4
    s, r = _schedule([CHI, D, CHI], [CHI * D, 1, D], [LB, P, RB], [CHI, D, CHI],
                     _strides([CHI, D, CHI]), [LB, P, R], [CHI, CHI], [RB, R])
    assert (r["kind"], r["streamk"]) == ("dmma_streamk", 132)
    assert s == "pair"


def test_stream_k_with_more_tiles_than_clusters_runs_segments():
    s, r = _gemm(1280, 1280, 2048)   # 100 tiles
    _need_132_sms(r)
    assert r["kind"] == "dmma_streamk"
    assert s == "segments"


def test_pair_schedule_bounds():
    # 66 tiles fill the 66 clusters of a 132-CTA grid; 72 do not fit
    s, r = _gemm(768, 1408, 2048)
    _need_132_sms(r)
    assert (r["kind"], s) == ("dmma_streamk", "pair")
    assert _gemm(1000, 1100, 2080)[0] == "segments"
    assert _gemm(512, 512, 1024, _lib.QB_C128)[0] == "pair"


def test_classic_launch_has_no_schedule():
    # the benchmark's ket step: 128 tiles, classic grid
    s, r = _schedule([CHI, CHI], [CHI, 1], [0, 1], [CHI, D, CHI], [CHI * D, 1, D], [1, 2, 3],
                     [CHI, D, CHI], [0, 2, 3])
    assert r["kind"] == "dmma"
    assert s is None


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not found")
def test_pair_kernels_do_not_spill():
    _lib.load()
    out = subprocess.run([shutil.which("cuobjdump"), "-res-usage", _lib.LIB_PATH],
                         capture_output=True, text=True, check=True).stdout
    pat = re.compile(r"_ZN2qb(24contract_f64_pair_kernel|31contract_f64_affine_pair_kernel)"
                     r"ILi128ELi128ELi32ELi2ELi4ELi3E")
    usage, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name:
            if pat.match(name):
                usage[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    # table feed: 4 layouts + complex; affine feed: 4 layouts x {A, B, both}
    assert len(usage) == 17, sorted(usage)
    over = {n: u for n, u in usage.items() if u[0] > 255 or u[1] > 0}
    assert not over, f"(registers, stack bytes) of spilling kernels: {over}"
