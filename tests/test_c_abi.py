"""The C-ABI library loads and exports every symbol include/dust3r_b200.h declares (no compute)."""
import ctypes
import os
import re

from conftest import ROOT


def _declared():
    src = open(os.path.join(ROOT, 'include', 'dust3r_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(d3r_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    from dust3r_b200 import build, _lib
    build.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 8
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/dust3r_b200.h but not exported'


def test_abi_version_5_and_struct_size():
    from dust3r_b200 import _lib
    lib = _lib.get_lib()
    assert lib.d3r_abi_version() == 5
    assert lib.d3r_align_chunk_pixels() == 2048   # maximum; the host picks chunk_px <= this per problem
    # python mirror of d3r_align_desc must match the C layout: probe through workspace sizing
    assert lib.d3r_align_workspace_floats(8, 28) > 0
    assert ctypes.sizeof(_lib.AlignDesc) == lib.d3r_sizeof_align_desc()


def test_no_oracle_or_reference_import_in_product():
    """The product package must never reach into oracle/ or the reference (parity claims depend on it)."""
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, 'dust3r_b200')):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.cpp', '.h')):
                s = open(os.path.join(dirpath, f)).read()
                if re.search(r'^\s*(from|import)\s+oracle\b', s, flags=re.M) or '/root/reference' in s:
                    bad.append(os.path.join(dirpath, f))
    assert not bad, bad
