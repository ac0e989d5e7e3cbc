"""Import the UNMODIFIED reference (elfi-dev/elfi) from the source checkout named by the
environment variable ELFI_REFERENCE_ROOT (the directory that contains its `elfi` package).

TEST / BASELINE INFRASTRUCTURE ONLY.  Used by tests/golden/gen_golden*.py to produce the
committed golden fixtures, by the reference-driven plugin tests and by ``bench.py --impl
reference`` (the CPU arm); never imported by the product (`elfi_b200/`).  Without the variable
those tests skip and the CPU arm is not run.

The reference needs packages that are absent here (matplotlib, GPy, arviz, numdifftools,
ipyparallel, dask, toolz) and uses NumPy-1 aliases; none of them touch the sampler hot
path, so they are stubbed (SURVEY.md §8c recipe).
"""
import sys
import types
from unittest.mock import MagicMock

import numpy as np

import os

REFERENCE_ROOT = os.path.abspath(os.environ.get('ELFI_REFERENCE_ROOT') or os.devnull)


def reference_available():
    return 'ELFI_REFERENCE_ROOT' in os.environ and \
        os.path.isdir(os.path.join(REFERENCE_ROOT, 'elfi'))


def import_reference():
    """Return the reference `elfi` module (import it on first call)."""
    if 'elfi' in sys.modules and getattr(sys.modules['elfi'], '__file__', '').startswith(
            REFERENCE_ROOT):
        return sys.modules['elfi']
    for name in ['matplotlib', 'matplotlib.pyplot', 'matplotlib.colors', 'matplotlib.axes',
                 'GPy', 'GPy.kern', 'GPy.models', 'GPy.priors', 'arviz', 'numdifftools',
                 'ipyparallel', 'dask', 'dask.distributed']:
        sys.modules.setdefault(name, MagicMock())
    if 'toolz' not in sys.modules:
        toolz = types.ModuleType('toolz')
        functoolz = types.ModuleType('toolz.functoolz')

        def compose(*funcs):
            def composed(*a, **k):
                out = funcs[-1](*a, **k)
                for f in reversed(funcs[:-1]):
                    out = f(out)
                return out
            return composed
        functoolz.compose = compose
        toolz.functoolz = functoolz
        toolz.compose = compose
        sys.modules['toolz'] = toolz
        sys.modules['toolz.functoolz'] = functoolz
    if not hasattr(np, 'Inf'):
        np.Inf = np.inf
    if not hasattr(np, 'float_'):
        np.float_ = np.float64
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import elfi
    return elfi
