"""CPU test double of the birth-death-mutation entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (installed first, by the `cpu_double` fixture) with restatements of
elfi_b200_sim_bdm_f64 and elfi_b200_bdm_summaries_f64 on host pointers: the simulator is
tests/bdm_replay.py (the kernel's Philox streams, so the same rows as the device), the summaries
are the reference's NumPy T1 and T2 (elfi_b200.examples.bdm on host arrays), NaN for a row with a
negative count.
"""
import numpy as np

import abi_double as d
import bdm_replay
from elfi_b200 import _lib, ops


def summaries(x, n):
    from elfi_b200.examples import bdm
    with np.errstate(all='ignore'):
        S = np.column_stack([bdm.T1(x), bdm.T2(x, n)])
    S[(x < 0).any(axis=1)] = np.nan
    return S


def sim_bdm_f64(ctx, P, ldP, B, N, n_t2, max_events, seed, offset, X, ldX, S, ldS, n_events,
                stream):
    d._require(ldP >= 3 and 1 <= N <= ops.BDM_N_MAX and 0 <= B <= ops.BDM_BATCH_MAX and
               1 <= max_events <= ops.BDM_MAX_EVENTS_LIMIT, 'sim_bdm: bad shape')
    if not B:
        return
    x, n = bdm_replay.simulate(d._mat(P, B, 3, ldP), N, seed, offset, max_events)
    Xv = d._mat(X, B, N, ldX, dtype=np.int16)
    if Xv is not None:
        Xv[:] = x
    Sv = d._mat(S, B, ops.BDM_NSUMM, ldS)
    if Sv is not None:
        Sv[:] = summaries(x, n_t2)
    d._vec(n_events, B, np.int64)[:] = n


def bdm_summaries_f64(ctx, X, ld_row, ld_col, B, N, n, S, ldS, stream):
    d._require(1 <= N <= ops.BDM_N_MAX and ldS >= ops.BDM_NSUMM, 'bdm_summaries: bad shape')
    if not B:
        return
    span = (B - 1) * ld_row + (N - 1) * ld_col + 1
    x = np.array(np.lib.stride_tricks.as_strided(d._vec(X, span, np.int16), (B, N),
                                                 (2 * ld_row, 2 * ld_col)))
    d._mat(S, B, ops.BDM_NSUMM, ldS)[:] = summaries(x, n)


_TABLE = {'elfi_b200_' + f.__name__: f for f in (sim_bdm_f64, bdm_summaries_f64)}


def install(monkeypatch):
    """Route the BDM entry points here, everything else to the installed _lib.call."""
    base = _lib.call

    def call(name, *args):
        fn = _TABLE.get(name)
        if fn is None:
            return base(name, *args)
        if len(args) != len(_lib.SIGNATURES[name]):
            raise TypeError('{} takes {} arguments, got {}'.format(
                name, len(_lib.SIGNATURES[name]), len(args)))
        d.CALLS.append(name)
        fn(*args)
        return 0
    monkeypatch.setattr(_lib, 'call', call)
