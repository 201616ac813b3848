"""bench.py contract checks that run without a GPU: the reference arm (CPU oracle port) prints one JSON line with the
keys the driver reads."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.timeout(600)
def test_reference_arm_json_line():
    env = dict(os.environ, OMP_NUM_THREADS='1')     # torchrun exports this; the arm must still use every core
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--gpus', '1', '--steps', '1',
                        '--warmup', '0', '--skip-cloud-opt'], capture_output=True, text=True, env=env, cwd=ROOT, timeout=550)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line['impl'] == 'reference' and line['higher_is_better'] is True and line['n_gpus'] == 1
    for key in ('metric', 'value', 'unit', 'steps', 'warmup', 'ms_per_step', 'scaling', 'dtype', 'data', 'config', 'cpu_baseline', 'e2e'):
        assert key in line, key
    assert line['unit'] == 'image-pairs/s' and line['value'] > 0
    assert line['e2e']['h2d_bytes_per_step'] == 0 and line['e2e']['d2h_bytes_per_step'] == 0
    assert line['cpu_baseline']['kind'] == 'port' and line['cpu_baseline']['cores'] >= 1
    if (os.cpu_count() or 1) > 1:
        assert line['cpu_baseline']['cores'] > 1, 'reference arm must not stay on the single thread torchrun grants'


def test_host_threads_respects_cgroup_quota_and_cap():
    sys.path.insert(0, ROOT)
    import bench
    n = bench.host_threads()
    assert 1 <= n <= 64 and n <= len(os.sched_getaffinity(0))
    assert bench.host_threads(cap=2) <= 2


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK='1', WORLD_SIZE='2', LOCAL_RANK='1')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--gpus', '2', '--steps', '1',
                        '--warmup', '0'], capture_output=True, text=True, env=env, cwd=ROOT, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == ''


def test_build_roofline_on_a_recorded_breakdown():
    """The `roofline` object is assembled by a pure function: feed it a per-kernel breakdown in the format of the bench's
    `kernels` record (a fixed, made-up one: the function is checked, not a GPU)."""
    sys.path.insert(0, ROOT)
    import bench
    rec = dict(value=300.0, kernels={
        'gemm_wgmma_2cta_bn128': dict(launches=600, ms=60.0, tflops=700.0, gbs=None),
        'attention_wgmma': dict(launches=120, ms=20.0, tflops=400.0, gbs=None),
        'layernorm': dict(launches=200, ms=5.0, tflops=None, gbs=2500.0)})
    prof = {k: dict(count=v['launches'], ms=v['ms'], flops=(v['tflops'] or 0.0) * v['ms'] * 1e9, bytes=(v['gbs'] or 0.0) * v['ms'] * 1e6)
            for k, v in rec['kernels'].items()}
    pk = dict(hbm=3350.0, tf_burst=989.0, tf_sustained=900.0, source='test')
    for world in (1, 8):
        r = bench.build_roofline(prof, pk, rec['value'] * world, world)
        json.dumps(r)                                     # serialisable
        assert r['bound'] == 'tensor' and r['unit'] == 'TFLOP/s' and r['kernel'] == 'gemm_wgmma_2cta_bn128'
        assert abs(r['frac'] - r['achieved'] / r['peak']) < 1e-12 and 0.5 < r['frac'] < 1.0
        assert r['peak'] == pk['tf_sustained'] and 0 < r['frac_of_burst_peak'] < r['frac']
        assert r['launches'] == 600 and abs(r['share_of_step'] - 60.0 / 85.0) < 1e-12
        ws = r['whole_step']
        assert abs(ws['achieved'] - rec['value'] * world * bench.GFLOP_PER_PAIR / 1e3) < 1e-6
        assert abs(ws['frac'] - ws['achieved'] / (pk['tf_sustained'] * world)) < 1e-12
    odd = bench.build_roofline({'some_kernel': dict(count=1, ms=1.0, flops=1e12, bytes=0.0)}, pk, 1.0, 1)
    assert odd['achieved'] == 1000.0
