"""ctypes binding of libelfi_b200.so (the C ABI declared in include/elfi_b200.h).

There is no CPU fallback: if the shared library is missing or a call fails, an exception is
raised.  Build it with ``python -c "import __graft_entry__ as g; g.build()"`` (nvcc, sm_90a).
"""
import ctypes
import os
import re

LIB_PATH = os.environ.get(
    'ELFI_B200_LIB',
    os.path.join(os.path.dirname(os.path.abspath(__file__)), 'lib', 'libelfi_b200.so'))

HEADER_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                           'include', 'elfi_b200.h')


class ElfiB200Error(RuntimeError):
    """A call into libelfi_b200.so failed."""


_CTYPES = {'int': ctypes.c_int, 'int32_t': ctypes.c_int, 'int64_t': ctypes.c_int64,
           'uint64_t': ctypes.c_uint64, 'double': ctypes.c_double}


def _ctype(decl, is_return=False):
    """ctypes type of a declaration such as `const double* S` or, with is_return, `int64_t`."""
    if '*' in decl:
        char_ptr = is_return and decl.split('*')[0].split() == ['const', 'char']
        return ctypes.c_char_p if char_ptr else ctypes.c_void_p
    words = [w for w in decl.split() if w != 'const']
    if len(words) != 2 - is_return or words[0] not in _CTYPES:
        raise ElfiB200Error('{}: no ctypes mapping for `{}`'.format(HEADER_PATH, decl.strip()))
    return _CTYPES[words[0]]


def _literal(name, value):
    m = re.fullmatch(r'\(?\s*(-?[0-9]+(\.[0-9]*)?([eE][-+]?[0-9]+)?)[uU]?[lL]{0,2}\s*\)?', value)
    if m is None:
        raise ElfiB200Error('{}: ELFI_B200_{} is not a plain literal: {!r}'.format(
            HEADER_PATH, name, value))
    return float(m.group(1)) if m.group(2) or m.group(3) else int(m.group(1))


def _parse_header():
    """(signatures, restypes, constants) of the C ABI as include/elfi_b200.h declares it."""
    if not os.path.exists(HEADER_PATH):
        raise ElfiB200Error('C ABI header not found at {}'.format(HEADER_PATH))
    with open(HEADER_PATH) as f:
        text = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', f.read(), flags=re.S)
    signatures, restypes, constants = {}, {}, {}
    prototypes = r'^[ \t]*([\w \t*]+?)\s*\b(elfi_b200_\w+)\s*\(([^)]*)\)\s*;'
    for ret, name, params in re.findall(prototypes, text, re.M):
        params = [] if params.strip() == 'void' else params.split(',')
        signatures[name] = [_ctype(p) for p in params]
        restypes[name] = _ctype(ret, is_return=True)
    for name, paren, value in re.findall(r'^[ \t]*#[ \t]*define[ \t]+ELFI_B200_(\w+)(\(?)(.*)$',
                                         text, re.M):
        if not paren and name != 'H':        # function-like macros and the include guard
            constants[name] = _literal(name, value.strip())
    return signatures, restypes, constants


# name -> argtypes and name -> restype of every entry point; CONSTANTS: the header's object-like
# ELFI_B200_<NAME> macros by <NAME> (the limits ops.py checks before a call)
SIGNATURES, _RESTYPES, CONSTANTS = _parse_header()
# entry points whose int result is a value, not a status
_NO_STATUS = {'elfi_b200_version', 'elfi_b200_last_error', 'elfi_b200_ctx_sm_count',
              'elfi_b200_gp_padded_size'}

_lib = None


def load():
    """Load the shared library (once) and declare all signatures."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ElfiB200Error(
            "libelfi_b200.so not found at {}. The CUDA extension must be built "
            "(__graft_entry__.build()); elfi_b200 has no CPU fallback.".format(LIB_PATH))
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.argtypes = argtypes
        fn.restype = _RESTYPES[name]
    _lib = lib
    return lib


def last_error():
    msg = load().elfi_b200_last_error()
    return msg.decode('utf-8', 'replace') if msg else ''


def call(name, *args):
    """Call a status-returning entry point; raise ElfiB200Error on a non-zero code."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if name in _NO_STATUS:
        return rc
    if rc != 0:
        raise ElfiB200Error('{} failed ({}): {}'.format(name, rc, last_error()))
    return rc
