"""The forward kernels keep their wgmmas in flight: ptxas has not serialised them.

When ptxas cannot prove a kernel's wgmma pipeline safe (a device-side call anywhere in the kernel, such as the vprintf
a printf compiles to: C7510; a wgmma on a divergent path: C7520; too few registers: C7512) it makes EVERY wgmma wait
for the previous one to retire. The build still succeeds and the results do not change; only the tensor cores idle
for most of each MMA's latency. In SASS a serialised wgmma is an HGMMA carrying the `gsb0` wait flag (followed by a
WARPGROUP.DEPBAR); a pipelined commit group carries it on its last HGMMA only. The smallest commit group of these
kernels is 8 MMAs, so at most a quarter of a kernel's HGMMAs may carry the flag. Needs nvcc, not a GPU.
"""
import os
import re
import subprocess

import pytest

from condmdi_b200 import build as B

OBJECTS = ["gemm_chain.o", "gemm2.o", "attention.o"]


def _cuobjdump() -> str:
    path = os.path.join(os.path.dirname(os.path.realpath(B._nvcc())), "cuobjdump")
    if not os.path.exists(path):
        pytest.fail(f"cuobjdump not found next to nvcc ({path})")
    return path


def hgmma_counts(sass: str) -> dict:
    """{function: (HGMMA instructions, of those carrying gsb0)} for every function of a cuobjdump -sass listing."""
    counts, fn = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            fn = m.group(1)
        elif fn and re.search(r"\bHGMMA\b", line):
            n, g = counts.get(fn, (0, 0))
            counts[fn] = (n + 1, g + ("gsb0" in line))
    return counts


@pytest.fixture(scope="module")
def sass():
    B.build()
    tool = _cuobjdump()
    out = {}
    for obj in OBJECTS:
        r = subprocess.run([tool, "-sass", os.path.join(B.BUILD, obj)], capture_output=True, text=True)
        assert r.returncode == 0, f"cuobjdump -sass {obj}: {r.stderr}"
        out[obj] = r.stdout
    return out


@pytest.mark.parametrize("obj", OBJECTS)
def test_wgmma_not_serialised(sass, obj):
    counts = hgmma_counts(sass[obj])
    assert counts, f"{obj}: no function issues wgmma"
    serialised = {fn: c for fn, c in counts.items() if 4 * c[1] > c[0]}
    assert not serialised, f"{obj}: wgmma serialised by ptxas ((HGMMA, with gsb0) per function): {serialised}"
