"""The k-pair layout of the 128x128 fp64 DMMA tile's A operand (no GPU needed).

An affine A operand whose 16-byte pairs lie along k and whose threads walk
rows (the MPS-norm bra step's site tensor read as [b', (a', p)]) is staged as
[k/2][row][2] so that each 32-byte sector a warp reads lands contiguously in
shared memory.  Its kernels are compiled under names of their own (one per B
layout and launch mode) and must not spill more than the affine kernels.
"""

import re
import shutil
import subprocess

import pytest

from quimb_b200 import _lib


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not found")
def test_kpair_kernels_do_not_spill():
    _lib.load()
    out = subprocess.run([shutil.which("cuobjdump"), "-res-usage", _lib.LIB_PATH],
                         capture_output=True, text=True, check=True).stdout
    pat = re.compile(r"_ZN2qb\d+(contract_f64_kpair(?:_streamk|_pair)?_kernel)"
                     r"ILi128ELi128ELi32ELi2ELi4ELi3ELi[01]EEEv")
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
    # 2 B layouts x {classic, stream-K, stream-K pair}
    assert len(usage) == 6, sorted(usage)
    # as for the affine kernels: no stack on the classic and pair launches,
    # at most 32 B on the stream-K segment loop
    limit = {"contract_f64_kpair_kernel": 0, "contract_f64_kpair_pair_kernel": 0,
             "contract_f64_kpair_streamk_kernel": 32}
    over = {n: u for n, u in usage.items()
            if u[0] > 255 or u[1] > limit[pat.match(n).group(1)]}
    assert not over, f"(registers, stack bytes) of spilling kernels: {over}"
