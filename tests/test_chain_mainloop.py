"""The GEMM mainloops keep a second wgmma group in flight while they add up the previous one.

mma_kblock_promoted (common.cuh) cuts a k-block into sub-chunks held in a ring of two register fragments: it issues
sub-chunk s + 1, waits with wgmma.wait_group 1 and promotes sub-chunk s while s + 1 runs on the tensor cores. In SASS
that wait is a WARPGROUP.DEPBAR with a non-zero count; if ptxas cannot prove the ring safe it waits for everything
instead (count 0 only) or serialises every wgmma, and the build still succeeds. The chained kernel's stack frame (its
spill space) must not grow past what it was before the ring: 432 bytes at bf16x3, 256 at bf16.
Needs nvcc, not a GPU.
"""
import os
import re
import subprocess

import pytest

from condmdi_b200 import build as B

STACK_LIMIT = {"linear_chain_kernelILi3E": 432, "linear_chain_kernelILi1E": 256}


def _cuobjdump() -> str:
    path = os.path.join(os.path.dirname(os.path.realpath(B._nvcc())), "cuobjdump")
    if not os.path.exists(path):
        pytest.fail(f"cuobjdump not found next to nvcc ({path})")
    return path


def _run(*args) -> str:
    r = subprocess.run([_cuobjdump(), *args], capture_output=True, text=True)
    assert r.returncode == 0, f"cuobjdump {' '.join(args)}: {r.stderr}"
    return r.stdout


def _is_gemm(fn: str) -> bool:
    return "linear_chain_kernel" in fn or "linear2_kernel" in fn or "linear2_f16_sum32_kernel" in fn


def depbar_counts(sass: str) -> dict:
    """{function: set of the counts of its WARPGROUP.DEPBAR.LE gsb0 waits} for the GEMM kernels of a listing."""
    out, fn = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            fn = m.group(1) if _is_gemm(m.group(1)) else None
            if fn:
                out[fn] = set()
        elif fn:
            m = re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*(0x[0-9a-f]+)", line)
            if m:
                out[fn].add(int(m.group(1), 16))
    return out


@pytest.fixture(scope="module")
def objects():
    B.build()
    return {obj: os.path.join(B.BUILD, obj) for obj in ("gemm_chain.o", "gemm2.o")}


@pytest.mark.parametrize("obj", ["gemm_chain.o", "gemm2.o"])
def test_promotion_overlaps_the_next_group(objects, obj):
    counts = depbar_counts(_run("-sass", objects[obj]))
    assert counts, f"{obj}: no GEMM kernel found"
    if obj == "gemm_chain.o":
        assert sum("linear_chain_kernel" in fn for fn in counts) == 2, sorted(counts)
    missing = {fn: sorted(c) for fn, c in counts.items() if not any(n > 0 for n in c)}
    assert not missing, f"{obj}: kernels without a wgmma.wait_group 1 (DEPBAR counts per function): {missing}"


def test_chain_stack_frame_did_not_grow(objects):
    usage = _run("--dump-resource-usage", objects["gemm_chain.o"])
    seen = {}
    for fn, stack in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", usage):
        for key in STACK_LIMIT:
            if key in fn:
                seen[key] = int(stack)
    assert set(seen) == set(STACK_LIMIT), f"chain instances not found: {seen}"
    over = {k: (v, STACK_LIMIT[k]) for k, v in seen.items() if v > STACK_LIMIT[k]}
    assert not over, f"stack frame (bytes, limit) grew: {over}"
