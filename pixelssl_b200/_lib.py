"""ctypes binding of libpixelssl_b200.so (the C ABI declared in include/pixelssl_b200.h).

The signatures are read from the header itself, so the binding cannot drift from it: every pointer parameter is
passed as c_void_p and the four scalar types the header uses map to their ctypes types.  There is NO fallback: if the
shared library is missing, a symbol is absent or a name is not declared in the header, loading / calling raises."""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libpixelssl_b200.so')
HEADER_PATH = os.path.join(os.path.dirname(_HERE), 'include', 'pixelssl_b200.h')

c_void_p, c_int, c_int64, c_float, c_double = (ctypes.c_void_p, ctypes.c_int, ctypes.c_int64,
                                               ctypes.c_float, ctypes.c_double)
_SCALARS = {'int': c_int, 'int64_t': c_int64, 'float': c_float, 'double': c_double}


class ConvGeom(ctypes.Structure):
    """mirror of pxl_conv_geom"""
    _fields_ = [('N', c_int), ('H', c_int), ('W', c_int), ('Cin', c_int),
                ('OH', c_int), ('OW', c_int), ('Cout', c_int), ('ldo', c_int),
                ('mul', c_int), ('div', c_int), ('ntaps', c_int), ('precision', c_int)]


class ConvTcExt(ctypes.Structure):
    """mirror of pxl_conv_tc_ext"""
    _fields_ = [('w_ntaps', c_int), ('widx_host', ctypes.POINTER(c_int)), ('out_mul', c_int),
                ('out_offy', c_int), ('out_offx', c_int), ('out_H', c_int), ('out_W', c_int),
                ('bn_stats', c_void_p), ('out_scale', c_float), ('out_scale_dev', c_void_p), ('out_accumulate', c_int)]


def header_code(path=HEADER_PATH):
    """The header without its comments and preprocessor lines."""
    text = re.sub(r'/\*.*?\*/', ' ', open(path).read(), flags=re.S)
    return re.sub(r'^\s*#.*$', ' ', text, flags=re.M)


def ctype_of(decl, name, returned=False):
    """ctypes type of a parameter declaration (type and name) or, returned=True, of a return type."""
    if '*' in decl:
        return c_void_p
    words = [w for w in decl.split() if w != 'const']
    if returned and words == ['void']:
        return None
    t = ' '.join(words if returned else words[:-1])
    if t not in _SCALARS:
        raise ValueError('%s: unsupported type in %r (pointers, %s only)' % (name, decl.strip(), ', '.join(_SCALARS)))
    return _SCALARS[t]


def parse_signatures(path=HEADER_PATH):
    """name -> (restype, argtypes) of every pxl_* function declared in the header."""
    sigs = {}
    for ret, name, params in re.findall(r'([^;{}()]*?)\b(pxl_\w+)\s*\(([^()]*)\)\s*;', header_code(path)):
        params = params.strip()
        args = [] if params in ('', 'void') else [ctype_of(p, name) for p in params.split(',')]
        sigs[name] = (ctype_of(ret, name, returned=True), args)
    return sigs


SIGNATURES = parse_signatures()

PXL_ERR_BAD_ARG = -1
PXL_ERR_UNSUPPORTED = -2

_lib = None


class PxlError(RuntimeError):
    def __init__(self, fn, code):
        self.fn, self.code = fn, code
        what = {PXL_ERR_BAD_ARG: 'bad argument', PXL_ERR_UNSUPPORTED: 'unsupported configuration'}.get(
            code, 'cudaError_t %d' % code)
        super().__init__('%s failed: %s' % (fn, what))


class _Declared:
    """The typed entry points of the library; any other name raises."""

    def __getattr__(self, name):
        raise AttributeError('%s is not declared in %s' % (name, HEADER_PATH))


def load():
    """Load (once) and type the library.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'pixelssl_b200: %s not found. Build it with `python -c "import __graft_entry__ as g; '
            'g.build()"` (nvcc, sm_90a). There is no CPU/PyTorch fallback.' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    bound = _Declared()
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing: loud by design
        fn.restype = res
        fn.argtypes = args
        setattr(bound, name, fn)
    _lib = bound
    return bound


_bound = {}


def call(name, *args):
    """Call an int-returning entry point and raise PxlError on a non-zero return."""
    fn = _bound.get(name)
    if fn is None:
        fn = _bound[name] = getattr(load(), name)
    rc = fn(*args)
    if rc != 0:
        raise PxlError(name, rc)
    return rc
