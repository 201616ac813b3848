"""Builds libdust3r_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

Usage:  python -m dust3r_b200.build [--force]
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libdust3r_b200.so')
OBJ_DIR = os.path.join(CSRC, 'build')

NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
CFLAGS = ['-O3', '-std=c++17', '-lineinfo', '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr',
          '-Xptxas', '-v', '-Xcudafe', '--diag_suppress=177']


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _deps():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    hdrs.append(os.path.join(HERE, '..', 'include', 'dust3r_b200.h'))
    return hdrs


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, 'rb') as f:
            h.update(f.read())
    h.update(' '.join(CFLAGS + ARCH).encode())
    return h.hexdigest()


def _compile(src, log):
    obj = os.path.join(OBJ_DIR, os.path.basename(src) + '.o')
    stamp = obj + '.sha'
    dig = _digest([src] + _deps())
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj
    cmd = [NVCC] + ARCH + CFLAGS + ['-c', src, '-o', obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log.append((src, r.stdout + r.stderr))
    if r.returncode != 0:
        raise RuntimeError(f'nvcc failed on {src}:\n{r.stdout}\n{r.stderr}')
    with open(stamp, 'w') as f:
        f.write(dig)
    return obj


def build(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, f))
    log = []
    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(lambda s: _compile(s, log), sources()))
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(OUT) or os.path.getmtime(OUT) < newest:
        cmd = [NVCC] + ARCH + ['-shared', '-o', OUT] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f'link failed:\n{r.stdout}\n{r.stderr}')
    if verbose:
        for src, out in log:
            print('==', os.path.basename(src))
            print(out)
    return OUT


if __name__ == '__main__':
    path = build(force='--force' in sys.argv, verbose=True)
    print('built', path)
