"""The compiled conv_kernel instantiations (3x3 convolutions with the staged epilogue, BLOCK_N 256 / 128, 1-CTA and CTA
pair) write their output through the TMA unit only (`UTMASTG`, no `STG`), and the CTA-pair forms keep no more GPU-scope
barriers than their two cluster barriers."""
import re
import subprocess

import pytest

from test_gemm_tma_store_sass import _cuobjdump, _kernels


@pytest.mark.timeout(900)
def test_conv_kernels_store_through_tma_only():
    from dust3r_b200 import build, _lib
    build.build()
    sass = subprocess.run([_cuobjdump(), '-sass', _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    seen = set()
    for name, lines in _kernels(sass).items():
        m = re.match(r'_ZN3d3r4gemm11conv_kernelILi(\d+)ELb([01])EEEv', name)
        if not m:
            continue
        bn, pair = int(m.group(1)), m.group(2) == '1'
        seen.add((bn, pair))
        ops = [re.search(r'\b(UTMASTG|STG\S*|MEMBAR\.ALL\.GPU)\b', ln) for ln in lines]
        ops = [o.group(1) for o in ops if o]
        assert 'UTMASTG' in ops, (name, sorted(set(ops)))
        assert not [o for o in ops if o.startswith('STG')], (name, sorted(set(ops)))
        if pair:
            assert ops.count('MEMBAR.ALL.GPU') <= 2, name
    assert seen == {(bn, p) for bn in (128, 256) for p in (False, True)}, sorted(seen)
