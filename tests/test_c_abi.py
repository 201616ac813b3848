"""The C-ABI library loads and exports every symbol include/dust3r_b200.h declares, the binding's prototypes and structure
mirrors match the header and the library (no compute)."""
import ctypes
import os
import re

from conftest import ROOT


def _declared():
    src = open(os.path.join(ROOT, 'include', 'dust3r_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(d3r_[a-z0-9_]+)\s*\(', src)))


# width of every C type the header uses, as _ctypes_width spells it
_C_WIDTHS = {'int32_t': 'i4', 'int': 'i4', 'int64_t': 'i8', 'long long': 'i8', 'uint32_t': 'u4', 'float': 'f4', 'double': 'f8'}


def _c_width(decl):
    """'const float*' / 'int32_t' / 'void' -> 'ptr' / 'i4' / None."""
    decl = decl.replace('const ', '').strip()
    if '*' in decl:
        return 'ptr'
    return None if decl == 'void' else _C_WIDTHS[decl]


def _ctypes_width(t):
    if t is None:
        return None
    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return 'ptr'
    return ('f' if t._type_ in 'fd' else 'u' if t._type_.isupper() else 'i') + str(ctypes.sizeof(t))


def _header_prototypes():
    """{name: (return width, [argument widths])} of every d3r_* function include/dust3r_b200.h declares."""
    src = open(os.path.join(ROOT, 'include', 'dust3r_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    protos = {}
    for ret, name, args in re.findall(r'([A-Za-z_][\w \t*]*?)\b(d3r_\w+)\s*\(([^)]*)\)\s*;', src):
        args = [a.strip() for a in args.split(',')]
        protos[name] = (_c_width(ret), [] if args == ['void'] else [_c_width(a.rsplit(None, 1)[0]) for a in args])
    return protos


def test_library_exports_every_declared_symbol():
    from dust3r_b200 import build, _lib
    build.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 8
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/dust3r_b200.h but not exported'


def test_abi_version_6_and_struct_size():
    from dust3r_b200 import _lib
    lib = _lib.get_lib()
    assert lib.d3r_abi_version() == 6
    assert lib.d3r_align_chunk_pixels() == 2048   # maximum; the host picks chunk_px <= this per problem
    # python mirror of d3r_align_desc must match the C layout: probe through workspace sizing
    assert lib.d3r_align_workspace_floats(8, 28) > 0
    assert ctypes.sizeof(_lib.AlignDesc) == lib.d3r_sizeof_align_desc()
    # the other mirrored structures: the forward's model descriptor and the engine's numpy tables
    from dust3r_b200 import _lib_fwd
    from dust3r_b200.cloud_opt.engine import ITEM, PACK_ENTRY
    assert ctypes.sizeof(_lib_fwd.Model) == lib.d3r_sizeof_model()
    assert ITEM.itemsize == lib.d3r_sizeof_align_item()
    assert PACK_ENTRY.itemsize == lib.d3r_sizeof_pack_entry()


def test_prototype_table_matches_the_header():
    """_lib.PROTOTYPES and include/dust3r_b200.h name the same functions with the same return and argument widths: a
    c_int32 where the header says int64_t would truncate the argument without an error."""
    from dust3r_b200 import _lib
    header = _header_prototypes()
    assert sorted(header) == _declared()
    table = {name: (_ctypes_width(res), [_ctypes_width(a) for a in args]) for name, (res, args) in _lib.PROTOTYPES.items()}
    missing, extra = sorted(set(header) - set(table)), sorted(set(table) - set(header))
    assert not missing, f'declared in include/dust3r_b200.h but not in _lib.PROTOTYPES: {missing}'
    assert not extra, f'in _lib.PROTOTYPES but not declared in include/dust3r_b200.h: {extra}'
    wrong = [f'{name}: header {header[name]}, table {table[name]}' for name in header if table[name] != header[name]]
    assert not wrong, 'prototypes differ from include/dust3r_b200.h:\n' + '\n'.join(wrong)


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
