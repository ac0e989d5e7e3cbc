"""Golden fixture of elfi.Testbench from the UNMODIFIED reference (elfi-dev/elfi, the checkout
named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_testbench.py

testbench.npz holds three cases on ma2.get_model(seed_obs=4), repetitions=3, seed=156:
* 'sim'    -- neither observations nor reference parameters given;
* 'obs'    -- observations given (one MA2 series);
* 'param'  -- reference parameters given (t1 = 0.6, t2 = 0.2).
Each case runs four methods: Rejection in the default quantile mode (batch_size=500,
n_samples=500), Rejection with n_sim, Rejection with a threshold and SMC with thresholds
[2.0, 1.0].  Keys: {case}_observations, {case}_ref_{t}, {case}_m{k}_seeds and per repetition r
{case}_m{k}_r{r}_{t} (samples), _d (discrepancies) and _nsim, plus {case}_m{k}_smd_{t}, the
sample-mean differences ('obs' has no reference parameters, hence none).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import ma2  # noqa: E402

CASE = dict(seed_obs=4, repetitions=3, seed=156)
OBS_SEED = 11
REF_PARAM = {'t1': np.array([0.6]), 't2': np.array([0.2])}
METHODS = [
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=500)),
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=100, n_sim=2000)),
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=50, threshold=0.5)),
    ('SMC', dict(discrepancy_name='d', batch_size=500), dict(n_samples=100,
                                                            thresholds=[2.0, 1.0])),
]


def given_observation():
    m = ma2.get_model(seed_obs=CASE['seed_obs'])
    return m.generate(batch_size=1, outputs=['MA2'], seed=OBS_SEED)['MA2']


def run_case(name, out, **given):
    m = ma2.get_model(seed_obs=CASE['seed_obs'])
    tb = elfi.Testbench(model=m, repetitions=CASE['repetitions'], seed=CASE['seed'],
                        progress_bar=False, **given)
    for k, (cls, mk, sk) in enumerate(METHODS):
        method = elfi.TestbenchMethod(method=getattr(elfi, cls), name='m{}'.format(k))
        method.set_method_kwargs(**mk)
        method.set_sample_kwargs(bar=False, **sk)
        tb.add_method(method)
    tb.run()
    out[name + '_observations'] = np.asarray(tb.observations)
    if tb.reference_parameter is not None:
        for t in ('t1', 't2'):
            out['{}_ref_{}'.format(name, t)] = np.asarray(tb.reference_parameter[t])
    for k, res in enumerate(tb.testbench_results):
        out['{}_m{}_seeds'.format(name, k)] = np.asarray(tb.method_seed_list[k])
        for r, s in enumerate(res['results']):
            for t in ('t1', 't2'):
                out['{}_m{}_r{}_{}'.format(name, k, r, t)] = np.asarray(s.samples[t])
            out['{}_m{}_r{}_d'.format(name, k, r)] = np.asarray(s.discrepancies)
            out['{}_m{}_r{}_nsim'.format(name, k, r)] = np.asarray(s.n_sim)
    if tb.reference_parameter is not None:
        smd = tb.parameterwise_sample_mean_differences()
        for k in range(len(METHODS)):
            for t in ('t1', 't2'):
                out['{}_m{}_smd_{}'.format(name, k, t)] = np.asarray(smd['m{}'.format(k)][t])


def main():
    out = {}
    run_case('sim', out)
    run_case('obs', out, observations=given_observation())
    run_case('param', out, reference_parameter={k: v.copy() for k, v in REF_PARAM.items()})
    np.savez(os.path.join(HERE, 'testbench.npz'), **out)
    print('wrote testbench', len(out), 'arrays')


if __name__ == '__main__':
    main()
