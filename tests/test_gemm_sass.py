"""The compiled CTA-pair GEMM kernels keep GPU-scope memory barriers out of their main loop.

A consumer releases a ring slot to both CTAs of the pair after every k-block.  A `.release.cluster` remote mbarrier
arrive makes ptxas put `MEMBAR.ALL.GPU` in front of each of these arrives; the plain arrive does not.  The only
GPU-scope barriers a pair kernel may contain are the ones of its entry and exit `barrier.cluster` synchronisations."""
import os
import re
import shutil
import subprocess

import pytest


def _cuobjdump():
    from dust3r_b200 import build
    tool = os.path.join(os.path.dirname(build.NVCC), 'cuobjdump')
    if not os.path.exists(tool):
        tool = shutil.which('cuobjdump')
    if not tool:
        pytest.skip('cuobjdump not found')
    return tool


def _membar_gpu_per_kernel(sass):
    counts, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = m.group(1)
            counts[cur] = 0
        elif cur is not None and 'MEMBAR.ALL.GPU' in line:
            counts[cur] += 1
    return counts


@pytest.mark.timeout(900)
def test_pair_gemm_kernels_have_no_gpu_membar_in_main_loop():
    from dust3r_b200 import build, _lib
    build.build()
    sass = subprocess.run([_cuobjdump(), '-sass', _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    counts = _membar_gpu_per_kernel(sass)
    # gemm_kernel<BLOCK_N, EPI, PAIR = true>
    pair = {k: v for k, v in counts.items() if re.match(r'_ZN3d3r4gemm11gemm_kernelILi\d+ELi\d+ELb1E', k)}
    assert len(pair) >= 4, sorted(counts)
    # two cluster barriers (entry and exit), one MEMBAR.ALL.GPU each
    bad = {k: v for k, v in pair.items() if v > 2}
    assert not bad, bad
