"""CPU-side tests of the ctypes binding derived from include/pixelssl_b200.h: the parser sees every declaration and
types it as written, the two hand-written struct mirrors match the header, and no Python source names an entry point
the header does not declare."""
import ctypes
import glob
import os
import re

import pytest

from pixelssl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, I, I64, F, D = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_double


def test_parser_covers_every_declaration():
    calls = re.findall(r'\b(pxl_\w+)\s*\(', _lib.header_code())
    assert calls and len(calls) == len(set(calls)), 'an entry point is declared twice'
    assert set(calls) == set(_lib.SIGNATURES)


def test_derived_signatures():
    sig = _lib.SIGNATURES
    assert sig['pxl_abi_version'] == (I, [])
    assert sig['pxl_launch_count'] == (I64, [])
    assert sig['pxl_reset_launch_count'] == (None, [])
    assert sig['pxl_mse_consistency'] == (I, [P, P, I64, F, P, P, P, P])
    # struct pointers and host int arrays are plain pointers too
    assert sig['pxl_conv_h16_launch'] == (I, [P] * 10)
    assert sig['pxl_bn_bwd_dx'] == (I, [P, P, P, P, P, P, P, D, I, P, P, I64, I, P, P, P, P, P, P, P, I, P, P])
    # void* const*, unsigned char*
    assert sig['pxl_peer_allreduce_bn'][1][:8] == [P, I, P, I, I, I64, D, I]
    assert sig['pxl_peer_open'] == (I, [P, P])


@pytest.mark.parametrize('decl', ['int pxl_bad(long n, void* stream);', 'unsigned pxl_bad(void* stream);',
                                  'int pxl_bad(size_t n);'])
def test_parser_rejects_other_scalar_types(tmp_path, decl):
    path = tmp_path / 'h.h'
    path.write_text('/* pxl_commented(int x); */\n#define PXL_X 1\nint pxl_ok(void);\n' + decl + '\n')
    with pytest.raises(ValueError, match='pxl_bad'):
        _lib.parse_signatures(str(path))
    path.write_text('int pxl_ok(void);\nvoid* pxl_ptr(const float* const* a, int64_t n);\n')
    assert _lib.parse_signatures(str(path)) == {'pxl_ok': (I, []), 'pxl_ptr': (P, [P, I64])}


def _header_structs():
    """name -> [(field, is_pointer, scalar type or None)] of the header's typedef structs."""
    out = {}
    for body, name in re.findall(r'typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;', _lib.header_code(), flags=re.S):
        fields = []
        for decl in filter(None, (d.strip() for d in body.split(';'))):
            m = re.match(r'((?:const\s+)?\w+)\s*(\**)\s*(.*)$', decl, flags=re.S)
            base, stars, names = m.groups()
            for f in names.split(','):
                ptr = bool(stars or f.strip().startswith('*'))
                fields.append((f.strip().lstrip('*').strip(), ptr, None if ptr else _lib.ctype_of(base + ' x', name)))
        out[name] = fields
    return out


def test_struct_mirrors_match_the_header():
    structs = _header_structs()
    assert set(structs) == {'pxl_conv_geom', 'pxl_conv_tc_ext'}
    for name, cls in (('pxl_conv_geom', _lib.ConvGeom), ('pxl_conv_tc_ext', _lib.ConvTcExt)):
        mine = []
        for f, t in cls._fields_:
            ptr = t is ctypes.c_void_p or issubclass(t, ctypes._Pointer)
            mine.append((f, ptr, None if ptr else t))
        assert mine == structs[name], name


def test_python_sources_name_only_declared_entry_points():
    declared = set(_lib.SIGNATURES) | set(_header_structs())
    files = glob.glob(os.path.join(ROOT, 'pixelssl_b200', '**', '*.py'), recursive=True) + \
        glob.glob(os.path.join(ROOT, 'tools', '**', '*.py'), recursive=True)
    assert len(files) > 20
    bad = []
    for path in files:
        for name, star in re.findall(r'\b(pxl_\w+)(\*?)', open(path).read()):
            # `pxl_eval_*` in prose: a prefix of declared names
            ok = any(d.startswith(name) for d in declared) if star else name in declared
            if not ok:
                bad.append('%s: %s' % (os.path.relpath(path, ROOT), name + star))
    assert not bad, 'not declared in include/pixelssl_b200.h: ' + ', '.join(bad)


def test_undeclared_names_are_not_bound():
    import __graft_entry__ as ge
    ge.build()
    ctypes.CDLL(_lib.LIB_PATH).pxl_h16_sat_counter       # exported for the library's own use, not declared
    with pytest.raises(AttributeError, match='pxl_h16_sat_counter is not declared'):
        _lib.call('pxl_h16_sat_counter')
    with pytest.raises(AttributeError, match='not declared'):
        _lib.load().pxl_no_such_entry_point()
