"""The 128x128 DMMA contraction tiles must not spill to local memory.

Their main loop holds 64 fp64 accumulators and 24 fragment doubles per thread
in registers.  A stack frame means spill stores and reloads that go through L1
next to the fragment reads of shared memory, which is what the loop is short
of.  The check reads the resource usage ptxas recorded in the built library,
so it needs no GPU.
"""

import re
import shutil
import subprocess

import pytest

from quimb_b200 import _lib


def _resource_usage():
    _lib.load()
    out = subprocess.run([shutil.which("cuobjdump"), "-res-usage", _lib.LIB_PATH],
                         capture_output=True, text=True, check=True).stdout
    usage = {}
    name = None
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
def test_large_dmma_tiles_bk32_only_and_do_not_spill():
    # mangled contract_f64_kernel / contract_f64_streamk_kernel<128, 128, ...>
    pat = re.compile(r"_ZN2qb(19contract_f64_kernel|27contract_f64_streamk_kernel)"
                     r"ILi128ELi128E")
    large = {n: u for n, u in _resource_usage().items() if pat.match(n)}
    # 4 layouts + complex, BK 32, x 2 launch modes
    assert len(large) == 10, sorted(large)
    assert all(re.search(r"ILi128ELi128ELi32ELi2ELi4ELi3E", n) for n in large), sorted(large)
    assert all(reg <= 255 for reg, _ in large.values())
    # the stream-K kernels also carry the segment loop's state across the tile;
    # up to 96 B of it lives on the stack, reloaded around the epilogue and
    # twice per k-block (the 16-warp tile spilled 380-680 B, 1.7 KB reloaded)
    limit = {"19contract_f64_kernel": 0, "27contract_f64_streamk_kernel": 96}
    over = {n: u for n, u in large.items() if u[1] > limit[pat.match(n).group(1)]}
    assert not over, f"(registers, stack bytes) of spilling kernels: {over}"
