"""Wood's 13 Ricker statistics restated one row at a time, and the accuracy checks of
elfi_b200_ricker_wood_f64's contract (include/elfi_b200.h), shared by the host and the GPU tests.

The restatement is independent of elfi_b200.examples.ricker: loops with correctly rounded sums
(math.fsum), np.linalg.pinv for the cubic design and np.linalg.lstsq(rcond=None), the
minimum-norm least-squares solution, for the autoregression.
"""
import math

import numpy as np

U = 2.0 ** -53
WIDTH = 13


def design(obs):
    o = np.sort(np.diff(np.asarray(obs, dtype=np.float64).reshape(-1)))
    return np.linalg.pinv(np.column_stack([o, o ** 2, o ** 3]))


def rank_kind(row):
    """The branch of the rank rule: 'none', 'one' or 'full' distinct nonzero values of row[:-1]."""
    values = {float(v) for v in row[:-1] if v != 0}
    return 'none' if not values else 'one' if len(values) == 1 else 'full'


def ar_columns(row):
    x = np.asarray(row[:-1], dtype=np.float64)
    return np.column_stack([x ** 0.3, x ** 0.6]), np.asarray(row[1:], dtype=np.float64) ** 0.3


def restate(row, P):
    """The 13 statistics of one row."""
    row = [float(v) for v in row]
    n = len(row)
    if not all(math.isfinite(v) for v in row):
        return np.full(WIDTH, np.nan)
    m = math.fsum(row) / n
    out = [m, float(sum(1 for v in row if v == 0))]
    for k in range(6):
        out.append(math.fsum((row[t] - m) * (row[t + k] - m) for t in range(n - k)) / n)
    e = sorted(row[t + 1] - row[t] for t in range(n - 1))
    for j in range(3):
        out.append(math.fsum(float(P[j, t]) * e[t] for t in range(n - 1)))
    A, w = ar_columns(row)
    out.extend(np.linalg.lstsq(A, w, rcond=None)[0])
    return np.array(out)


def restate_rows(Y, P):
    return np.array([restate(r, P) for r in Y]).reshape(-1, WIDTH)


def check(got, ref, Y, P, exact_sums):
    """got against ref row by row, to the contract: columns 0..7 bit for bit (exact_sums) or within
    a relative 1e-12 of their scale; the cubic coefficients within 2 (n-1) 2^-53 sum_t |P_jt e_t|;
    the autoregression on the rank rule's branch: 0 exactly, proportional rows within 1e-13, full
    rank within 1e3 2^-53 cond([u v])^2 relative.  Non-finite rows are NaN in both."""
    Y = np.asarray(Y, dtype=np.float64)
    B, n = Y.shape
    assert got.shape == ref.shape == (B, WIDTH)
    bad = ~np.isfinite(Y).all(axis=1)
    assert np.isnan(got[bad]).all() and np.isnan(ref[bad]).all()
    g, r, y = got[~bad], ref[~bad], Y[~bad]
    if exact_sums:
        np.testing.assert_array_equal(g[:, :8], r[:, :8])
    else:
        np.testing.assert_array_equal(g[:, 1], r[:, 1])
        m = r[:, 0]
        scale = np.abs(m)
        assert np.all(np.abs(g[:, 0] - m) <= 1e-12 * scale), np.max(np.abs(g[:, 0] - m) / scale)
        yc = y - m[:, None]
        for k in range(6):
            s = np.sum(np.abs(yc[:, :n - k] * yc[:, k:]), axis=1) / n + m * m
            err = np.abs(g[:, 2 + k] - r[:, 2 + k])
            assert np.all(err <= 1e-12 * s), (k, np.max(err / s))
    e = np.sort(np.diff(y, axis=1), axis=1)
    for j in range(3):
        bound = 2 * (n - 1) * U * np.sum(np.abs(P[j][None, :] * e), axis=1)
        err = np.abs(g[:, 8 + j] - r[:, 8 + j])
        assert np.all(err <= bound), (j, np.max(err - bound))
    for i in range(len(y)):
        kind = rank_kind(y[i])
        a, b = g[i, 11:], r[i, 11:]
        if kind == 'none':
            assert np.all(a == 0) and np.all(b == 0), (i, a, b)
        elif kind == 'one':
            np.testing.assert_allclose(a, b, rtol=1e-13, atol=0, err_msg=str(i))
        else:
            A, _ = ar_columns(y[i])
            tol = 1e3 * U * np.linalg.cond(A) ** 2
            assert np.linalg.norm(a - b) <= tol * np.linalg.norm(b), (i, a, b, tol)
