"""The compiled TMA-store GEMM kernels write their output through the TMA unit only.

gemm_kernel<256, EPI_RESID | EPI_ACT | EPI_ROPE, PAIR, TMA_STORE = true> stage the epilogue in shared memory and hand
it to a TMA store (`UTMASTG`, bf16 outputs) or TMA reduce-add (`UTMAREDG`, the fp32 residual update).  No thread may
store to global memory itself, and the CTA-pair forms keep no more GPU-scope barriers than their two cluster barriers."""
import os
import re
import shutil
import subprocess

import pytest

EPI_RESID, EPI_ACT, EPI_ROPE = 1, 2, 3


def _cuobjdump():
    from dust3r_b200 import build
    tool = os.path.join(os.path.dirname(build.NVCC), 'cuobjdump')
    if not os.path.exists(tool):
        tool = shutil.which('cuobjdump')
    if not tool:
        pytest.skip('cuobjdump not found')
    return tool


def _kernels(sass):
    body, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = m.group(1)
            body[cur] = []
        elif cur is not None:
            body[cur].append(line)
    return body


@pytest.mark.timeout(900)
def test_tma_store_kernels_store_through_tma_only():
    from dust3r_b200 import build, _lib
    build.build()
    sass = subprocess.run([_cuobjdump(), '-sass', _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = _kernels(sass)
    seen = set()
    for name, lines in kernels.items():
        m = re.match(r'_ZN3d3r4gemm11gemm_kernelILi256ELi(\d)ELb([01])ELb1EEEv', name)
        if not m:
            continue
        epi, pair = int(m.group(1)), m.group(2) == '1'
        seen.add((epi, pair))
        ops = [re.search(r'\b(UTMASTG|UTMAREDG|STG\S*|MEMBAR\.ALL\.GPU)\b', ln) for ln in lines]
        ops = [o.group(1) for o in ops if o]
        want = 'UTMAREDG' if epi == EPI_RESID else 'UTMASTG'
        assert want in ops, (name, sorted(set(ops)))
        assert not [o for o in ops if o.startswith('STG')], (name, sorted(set(ops)))
        if pair:
            assert ops.count('MEMBAR.ALL.GPU') <= 2, name
    assert seen == {(e, p) for e in (EPI_RESID, EPI_ACT, EPI_ROPE) for p in (False, True)}, sorted(seen)
