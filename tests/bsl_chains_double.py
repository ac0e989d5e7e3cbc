"""NumPy restatements of the lock-step BSL chains -- TEST INFRASTRUCTURE ONLY.

* `mh_step` restates elfi_b200_bsl_mh_step_f64 (include/elfi_b200.h) with oracle/streams.py's
  Philox4x32-10, u01 and Box-Muller, in the kernel's order of operations; `TABLE` routes the entry
  point here on top of tests/abi_double.py, so throughput mode's host logic runs without a GPU.
* `parity_chains` restates parity mode as C reference-style Metropolis-Hastings loops (each with
  its own RandomState) that share one batch stream per iteration: batch k is simulated by the
  model at the sampler's batch seed (sub seed k of the sampler's seed) with batch_size rows of
  every chain, and one likelihood evaluates the C rounds.
"""
import numpy as np

import abi_double as d
import bsl_double
import conditional_prior_replay as cpr
import streams
from elfi_b200 import model as em
from elfi_b200.bsl import BSL
from elfi_b200.samplers import ModelPrior

SALT_BSL = 0x4253434C
BOTH, UPPER, LOWER, NONE = 0, 1, 2, 3


def bound_kinds(bounds, p):
    if bounds is None:
        return np.full(p, NONE)
    inf = np.isinf(np.asarray(bounds, dtype=float))
    return inf[:, 0] * 1 + inf[:, 1] * 2


def logit(kinds, bounds, x):
    out = x.copy()
    with np.errstate(all='ignore'):
        for a, k in enumerate(kinds):
            if k == NONE:
                continue
            lo, hi = bounds[a]
            out[:, a] = (np.log((x[:, a] - lo) / (hi - x[:, a])) if k == BOTH else
                         np.log(1.0 / (hi - x[:, a])) if k == UPPER else np.log(x[:, a] - lo))
    return out


def logit_back(kinds, bounds, y):
    out = y.copy()
    with np.errstate(all='ignore'):
        for a, k in enumerate(kinds):
            if k == NONE:
                continue
            lo, hi = bounds[a]
            ey = np.exp(y[:, a])
            out[:, a] = (lo / (1.0 + ey) + hi / (1.0 + (1.0 / ey)) if k == BOTH else
                         hi - (1.0 / ey) if k == UPPER else lo + ey)
    return out


def jacobian(kinds, bounds, x):
    s = np.zeros(x.shape[0])
    with np.errstate(all='ignore'):
        for a, k in enumerate(kinds):
            if k == BOTH:
                lo, hi = bounds[a]
                ey = np.exp(x[:, a])
                s = s + (np.log(hi - lo) - np.log((1.0 / ey) + 2.0 + ey))
            elif k != NONE:
                s = s + x[:, a]
    return s


def mh_step(t, table7, L, bounds, seed, burn_in, loglik, prop, prop_lp, chains, logpost, n_acc):
    """The step in place on host arrays (shapes of ops.bsl_mh_step).  Returns (rows (C, p): the
    next batch's parameter of each chain or None at the last iteration, accept (C,), margin (C,):
    |log u - r| of the decisions made, inf elsewhere)."""
    C, n_samples, p = chains.shape
    kinds = bound_kinds(bounds, p)
    c = np.arange(C, dtype=np.uint64)
    lp_new = loglik + prop_lp
    margin = np.full(C, np.inf)
    if t == 0:
        accept = np.ones(C, dtype=bool)
        state = prop.copy()
    else:
        prev = chains[:, t - 1]
        with np.errstate(all='ignore'):
            res = (jacobian(kinds, bounds, prop) - jacobian(kinds, bounds, prev)) \
                + (lp_new - logpost[:, t - 1])
            clipped = np.where(np.isnan(res), -700.0, np.clip(res, -700.0, 700.0))
            prob = np.minimum(1.0, np.exp(clipped))
        w = streams.philox4x32_10(t, c, 0, SALT_BSL, seed)
        u = streams.u01(w[0], w[1])
        inside = np.isfinite(prop_lp)
        accept = inside & (u < prob)
        margin[inside] = np.abs(np.log(u[inside]) - clipped[inside])
        state = np.where(accept[:, None], prop, prev)
        lp_new = np.where(accept, lp_new, logpost[:, t - 1])
    chains[:, t] = state
    logpost[:, t] = lp_new
    if t >= burn_in:
        n_acc += accept
    if t + 1 >= n_samples:
        return None, accept, margin
    y = logit(kinds, bounds, state)
    for k in range(0, p, 2):
        z0, z1, _ = streams.normal2(streams.philox4x32_10(t + 1, c, 1 + k // 2, SALT_BSL, seed))
        for a in range(k, p):
            y[:, a] = y[:, a] + L[a, k] * z0
            if a > k:
                y[:, a] = y[:, a] + L[a, k + 1] * z1
    y = logit_back(kinds, bounds, y)
    lp = cpr.joint_logpdf(table7, y)
    prop[:] = y
    prop_lp[:] = lp
    rows = np.where(np.isfinite(lp)[:, None], y, state)
    return rows, accept, margin


def bsl_mh_step_f64(ctx, C, p, t, n_samples, burn_in, b, seed, spec_host, chol_host, bounds_host,
                    loglik, prop, prop_lp, chains, logpost, n_acc, rows, ld_rows, stream):
    d._require(1 <= C <= 1 << 22 and 1 <= p <= 16, 'bsl_mh_step: bad shape')
    d._require(0 <= t < n_samples < 2 ** 32 and burn_in >= 0, 'bsl_mh_step: bad iteration')
    d._require(b >= 1 and C * b < 2 ** 31 and ld_rows >= C * b, 'bsl_mh_step: bad rows')
    table7 = d._mat(spec_host, p, 7).copy()
    L = d._mat(chol_host, p, p).copy()
    bounds = d._mat(bounds_host, p, 2)
    bounds = None if bounds is None else bounds.copy()
    ch = d._mat(chains, C * n_samples, p).reshape(C, n_samples, p)
    lpost = d._mat(logpost, C, n_samples)
    acc = d._vec(n_acc, C, dtype=np.int64)
    r, _, _ = mh_step(t, table7, L, bounds, seed, burn_in, d._vec(loglik, C).copy(),
                      d._mat(prop, C, p), d._vec(prop_lp, C), ch, lpost, acc)
    if r is not None:
        out = d._mat(rows, p, C * b, ld_rows)
        out[:] = np.repeat(r, b, axis=0).T


TABLE = {'elfi_b200_bsl_mh_step_f64': bsl_mh_step_f64}


# ------------------------------------------------------------------------------ parity mode
def parity_chains(model, feature, n_sim_round, batch_size, seed, n_samples, sigma, params0,
                  burn_in=0, bounds=None, likelihood=bsl_double.synlik):
    """C reference-style chains sharing one batch stream.  Returns (chains (C, n_samples, p),
    logposterior (C, n_samples), accepted (C,) after burn-in, batches simulated)."""
    names = model.parameter_names
    prior = ModelPrior(model)
    params0 = np.asarray(params0, dtype=float)
    C, p = params0.shape
    bounds = None if bounds is None else np.asarray(bounds, dtype=float)
    states = [np.random.RandomState(seed)] + [
        np.random.RandomState(em.get_sub_seed(seed, c)) for c in range(1, C)]
    obs = np.column_stack([np.asarray(model[feature].observed)]).reshape(-1)
    params = np.zeros((C, n_samples, p))
    logprior = np.zeros((C, n_samples))
    logpost = np.zeros((C, n_samples))
    accepted = np.zeros(C, dtype=np.int64)
    batch = [0]

    def simulate(theta):
        rows = np.repeat(theta, batch_size, axis=0)
        blocks = []
        for _ in range(n_sim_round // batch_size):
            ctx = em.ComputationContext(C * batch_size, seed=seed)
            out = em.execute_batch(model, [feature], ctx, batch[0],
                                   with_values={q: rows[:, i] for i, q in enumerate(names)})
            batch[0] += 1
            blocks.append(np.asarray(out[feature], dtype=float).reshape(C, batch_size, -1))
        return likelihood(np.concatenate(blocks, axis=1), obs)

    def propose(c, mean):
        rs = states[c]
        if bounds is None:
            return rs.multivariate_normal(mean, sigma)
        return BSL._para_logit_back_transform(rs.multivariate_normal(
            BSL._para_logit_transform(mean, bounds), sigma), bounds)

    params[:, 0] = params0
    logprior[:, 0] = np.reshape(prior.logpdf(params0), -1)
    ll = simulate(params0)
    logpost[:, 0] = ll + logprior[:, 0]
    if burn_in == 0:
        accepted += 1
    for n in range(1, n_samples):
        props = np.vstack([propose(c, params[c, n - 1]) for c in range(C)])
        lp = np.reshape(prior.logpdf(props), -1)
        live = np.isfinite(lp)
        params[:, n] = np.where(live[:, None], props, params[:, n - 1])
        logprior[:, n] = np.where(live, lp, logprior[:, n - 1])
        logpost[:, n] = logpost[:, n - 1]
        if not live.any():
            continue
        ll = simulate(params[:, n])
        for c in np.flatnonzero(live):
            logpost[c, n] = ll[c] + logprior[c, n]
            res = logpost[c, n] - logpost[c, n - 1]
            if bounds is not None:
                res = (BSL._jacobian_logit_transform(params[c, n], bounds)
                       - BSL._jacobian_logit_transform(params[c, n - 1], bounds)) + res
            prob = np.minimum(1.0, np.exp(min(700, max(-700, res))))
            if states[c].uniform() < prob:
                accepted[c] += n >= burn_in
            else:
                params[c, n] = params[c, n - 1]
                logprior[c, n] = logprior[c, n - 1]
                logpost[c, n] = logpost[c, n - 1]
    return params, logpost, accepted, batch[0]
