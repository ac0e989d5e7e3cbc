"""CPU-side checks of the drop-in boundary: the shared library loads and exports exactly
the entry points include/elfi_b200.h declares (no compute calls: no GPU here)."""
import ctypes
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    text = open(os.path.join(ROOT, 'include', 'elfi_b200.h')).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(elfi_b200_\w+)\s*\(', text)))


def test_header_declares_functions():
    names = header_functions()
    assert 'elfi_b200_ctx_create' in names
    assert 'elfi_b200_dist_euclid_thr_f64' in names
    assert len(names) >= 6


def test_library_exports_every_header_symbol():
    from elfi_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in header_functions() if not hasattr(lib, n)]
    assert not missing, 'declared in include/elfi_b200.h but not exported: {}'.format(missing)


def test_binding_covers_header():
    """Every prototype parses into known ctypes, one per declared parameter; each type class maps
    as the header declares it."""
    from elfi_b200 import _lib
    assert sorted(_lib.SIGNATURES) == header_functions()
    text = re.sub(r'/\*.*?\*/', '', open(_lib.HEADER_PATH).read(), flags=re.S)
    known = {ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int64, ctypes.c_uint64,
             ctypes.c_double}
    for name, argtypes in _lib.SIGNATURES.items():
        params = re.search(name + r'\s*\(([^)]*)\)', text).group(1).strip()
        assert len(argtypes) == (0 if params == 'void' else params.count(',') + 1), name
        assert set(argtypes) | {_lib._RESTYPES[name]} <= known, name
    assert _lib._RESTYPES['elfi_b200_last_error'] is ctypes.c_char_p
    assert _lib._RESTYPES['elfi_b200_gp_padded_size'] is ctypes.c_int64
    assert _lib.SIGNATURES['elfi_b200_gp_padded_size'] == [ctypes.c_int64]
    assert _lib._RESTYPES['elfi_b200_dist_euclid_thr_f64'] is ctypes.c_int
    # (ctx, P, ldP, n_params, B, n_obs, double stock_init, uint64_t seed, uint64_t offset, Y, ...)
    ricker = _lib.SIGNATURES['elfi_b200_sim_ricker_f64']
    assert ricker[:9] == [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int64] * 4 + [
        ctypes.c_double, ctypes.c_uint64, ctypes.c_uint64]
    # (ctx, int32_t metric, double pexp, const double* S, int64_t ldS, ...)
    assert _lib.SIGNATURES['elfi_b200_dist_metric_thr_f64'][:5] == [
        ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_void_p, ctypes.c_int64]
    lib = _lib.load()
    assert lib.elfi_b200_version() == _lib.CONSTANTS['VERSION'] == 101


def test_constants_cover_header_macros():
    """Every object-like ELFI_B200_ macro but the include guard is in CONSTANTS, int or float as
    its literal is written."""
    from elfi_b200 import _lib
    text = re.sub(r'/\*.*?\*/', '', open(_lib.HEADER_PATH).read(), flags=re.S)
    names = re.findall(r'^\s*#\s*define\s+ELFI_B200_(\w+)(?!\w|\()', text, re.M)
    assert sorted(_lib.CONSTANTS) == sorted(n for n in names if n != 'H')
    assert _lib.CONSTANTS['ERR_ARG'] == -1 and _lib.CONSTANTS['TOAD_CELLS_MAX'] == 2 ** 31
    assert isinstance(_lib.CONSTANTS['POISSON_LAM_MAX'], float)
    assert all(type(v) is int for k, v in _lib.CONSTANTS.items() if k != 'POISSON_LAM_MAX')


def test_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from elfi_b200 import _lib, ops
    import numpy as np
    with pytest.raises(_lib.ElfiB200Error):
        ops.dist_euclid(np.zeros((4, 2)), np.zeros(2))


def test_product_never_imports_oracle():
    """The product path must not route through the CPU oracle (or the reference)."""
    pkg = os.path.join(ROOT, 'elfi_b200')
    bad = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                src = open(os.path.join(dirpath, f)).read()
                if re.search(r'^\s*(import|from)\s+(elfi_oracle|oracle|ref_shim|streams)\b', src, re.M):
                    bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_native_code_reads_no_environment():
    """Every kernel choice follows from the inputs and the device: no source of the library reads
    an environment variable, so a variable set in a user's shell cannot change what runs."""
    csrc = os.path.join(ROOT, 'elfi_b200', 'csrc')
    bad = sorted(f for f in os.listdir(csrc)
                 if re.search(r'getenv\s*\(', open(os.path.join(csrc, f)).read()))
    assert not bad, bad


def test_every_header_function_has_a_product_caller():
    """Every function the header declares is named by product code (the package, integration/ or
    bench.py), so the library exports no entry point that only tests reach."""
    sources = glob.glob(os.path.join(ROOT, 'elfi_b200', '**', '*.py'), recursive=True)
    sources += glob.glob(os.path.join(ROOT, 'integration', '*.py')) + [os.path.join(ROOT, 'bench.py')]
    text = '\n'.join(open(f).read() for f in sources)
    unused = [n for n in header_functions() if not re.search(r'\b' + n + r'\b', text)]
    assert not unused, 'declared in include/elfi_b200.h but named by no product code: {}'.format(unused)
