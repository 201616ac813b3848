"""g++ builds of the host harnesses in tests/native, which compile the kernels' per-thread bodies (dust3r_b200/csrc/*_core.h)
for the CPU.  Every harness is held to one flag set; -ffp-contract=off keeps g++ from fusing a multiply and an add that the
kernels round separately."""
import os
import shutil
import subprocess
import tempfile

import pytest

NATIVE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'native')
FLAGS = ['-std=c++17', '-Wall', '-Wextra', '-Werror', '-ffp-contract=off']

_built = {}
_tmp = None


def build(name, *extra, shared=True):
    """Path of tests/native/<name>.cpp built with FLAGS and `extra`: a shared library (-O2) to load with ctypes, or with
    shared=False an executable.  Built once per session; the test is skipped when there is no g++."""
    global _tmp
    key = (name, extra, shared)
    if key not in _built:
        gxx = shutil.which('g++')
        if gxx is None:
            pytest.skip('no g++')
        if _tmp is None:
            _tmp = tempfile.TemporaryDirectory(prefix='native_harness_')
        out = os.path.join(_tmp.name, f'{name}_{len(_built)}' + ('.so' if shared else ''))
        kind = ['-O2', '-shared', '-fPIC'] if shared else []
        subprocess.run([gxx, *FLAGS, *kind, *extra, '-o', out, os.path.join(NATIVE, f'{name}.cpp')], check=True)
        _built[key] = out
    return _built[key]
