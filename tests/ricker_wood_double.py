"""CPU test double of elfi_b200_ricker_wood_f64 -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with a restatement of
Wood's 13 Ricker statistics on host pointers: the NumPy definition of
elfi_b200.examples.ricker.wood_statistics on the rows of Y and the design P the call passes, with
the kernel's argument checks.
"""
import abi_double as d
from elfi_b200 import ops


def ricker_wood_f64(ctx, Y, ldY, B, n, P, out, ld_out, stream):
    from elfi_b200.examples import ricker
    d._require(B >= 0 and ops.RICKER_WOOD_NOBS_MIN <= n <= ops.RICKER_WOOD_NOBS_MAX and ldY >= n
               and ld_out >= ops.RICKER_WOOD_WIDTH, 'ricker_wood: bad shape')
    if not B:
        return
    d._require(d._addr(Y) and d._addr(P) and d._addr(out), 'ricker_wood: NULL argument')
    d._mat(out, B, ops.RICKER_WOOD_WIDTH, ld_out)[:] = ricker.wood_statistics(
        d._mat(Y, B, n, ldY).copy(), d._mat(P, 3, n - 1).copy())


TABLE = {'elfi_b200_' + f.__name__: f for f in (ricker_wood_f64,)}
