"""CPU test doubles of the two entry points that run a Testbench's BSL repetitions in lock-step
(elfi_b200_synlik_obs_f64, elfi_b200_bsl_mh_step_keyed_f64) -- TEST INFRASTRUCTURE ONLY.

Both are stated as the existing doubles applied group by group or chain by chain:
* `synlik_obs_f64` is tests/bsl_double.py's synlik_f64 on group g alone with y = Y + g ld_y;
* `bsl_mh_step_keyed_f64` runs tests/bsl_chains_double.py's mh_step for each chain slot c with
  the seed keys[c], on lanes[c] + 1 chains of which the one at index lanes[c] is slot c (the
  unkeyed step draws chain l's numbers on lane l).
`TABLE` routes both here on top of tests/abi_double.py (through `abi_double.install`);
tests/bsl_double.py and tests/bsl_chains_double.py route the unkeyed entry points.
"""
import numpy as np

import abi_double as d
import bsl_chains_double
import bsl_double


def synlik_obs_f64(ctx, S, ld_row, ld_group, G, n, dim, Y, ld_y, W, estimator, penalties_host, K,
                   loglik, stream):
    d._require(ld_y == 0 or ld_y >= dim, 'synlik: the observation stride must be 0 or at least d')
    d._require(G >= 0, 'synlik: bad shape')
    if not G:
        return bsl_double.synlik_f64(ctx, S, ld_row, ld_group, 0, n, dim, Y, W, estimator,
                                     penalties_host, K, loglik, stream)
    s, y, out = d._addr(S), d._addr(Y), d._addr(loglik)
    for g in range(G):
        bsl_double.synlik_f64(ctx, s + 8 * g * ld_group, ld_row, 0, 1, n, dim, y + 8 * g * ld_y, W,
                              estimator, penalties_host, K, out + 8 * g * max(K, 1), stream)


def bsl_mh_step_keyed_f64(ctx, C, p, t, n_samples, burn_in, b, keys, lanes, spec_host, chol_host,
                          bounds_host, loglik, prop, prop_lp, chains, logpost, n_acc, rows,
                          ld_rows, stream):
    d._require(d._addr(keys) and d._addr(lanes), 'bsl_mh_step_keyed: NULL keys or lanes')
    d._require(1 <= C <= 1 << 22 and 1 <= p <= 16, 'bsl_mh_step: bad shape')
    d._require(0 <= t < n_samples < 2 ** 32 and burn_in >= 0, 'bsl_mh_step: bad iteration')
    d._require(b >= 1 and C * b < 2 ** 31 and ld_rows >= C * b, 'bsl_mh_step: bad rows')
    table7 = d._mat(spec_host, p, 7).copy()
    L = d._mat(chol_host, p, p).copy()
    bounds = d._mat(bounds_host, p, 2)
    bounds = None if bounds is None else bounds.copy()
    key = d._vec(keys, C, np.uint64)
    lane = d._vec(lanes, C, np.uint32)
    ch = d._mat(chains, C * n_samples, p).reshape(C, n_samples, p)
    lpost = d._mat(logpost, C, n_samples)
    acc = d._vec(n_acc, C, dtype=np.int64)
    ll = d._vec(loglik, C)
    pr = d._mat(prop, C, p)
    plp = d._vec(prop_lp, C)
    out = d._mat(rows, p, C * b, ld_rows)
    for c in range(C):
        at = int(lane[c])

        def placed(x):
            a = np.zeros((at + 1,) + x.shape[1:], dtype=x.dtype)
            a[at] = x[c]
            return a
        arrays = [placed(x) for x in (ll, pr, plp, ch, lpost, acc)]
        r, _, _ = bsl_chains_double.mh_step(t, table7, L, bounds, int(key[c]), burn_in, *arrays)
        for x, a in zip((pr, plp, ch, lpost, acc), arrays[1:]):
            x[c] = a[at]
        if r is not None:
            out[:, c * b:(c + 1) * b] = r[at][:, None]


TABLE = {'elfi_b200_synlik_obs_f64': synlik_obs_f64,
         'elfi_b200_bsl_mh_step_keyed_f64': bsl_mh_step_keyed_f64}
