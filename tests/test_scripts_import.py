"""Every measurement script under scripts/ imports on the CPU without launching anything and keeps its work in main(): a
script that imports a name someone deleted fails here, not on the next GPU run (no compute)."""
import glob
import importlib.util
import os
import sys

import pytest

from conftest import ROOT

SCRIPTS = os.path.join(ROOT, 'scripts')
NAMES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(SCRIPTS, '*.py')) if not p.endswith('common.py'))


@pytest.fixture
def no_library(monkeypatch):
    """The scripts' own path setup (scripts/ first, as `python scripts/x.py` has it), undone afterwards, and a C library
    that raises on first use: importing a script must not reach it."""
    from dust3r_b200 import _lib

    def get_lib():
        raise AssertionError('a script called into the C library at import')
    monkeypatch.setattr(_lib, 'get_lib', get_lib)
    monkeypatch.syspath_prepend(SCRIPTS)
    yield
    sys.modules.pop('common', None)


@pytest.mark.parametrize('name', NAMES)
def test_script_imports_without_running(name, no_library):
    spec = importlib.util.spec_from_file_location(f'_script_{name}', os.path.join(SCRIPTS, f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert callable(getattr(mod, 'main', None)), f'scripts/{name}.py has no main()'
