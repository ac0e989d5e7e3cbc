"""Golden fixture of elfi.Testbench with elfi.BSL from the UNMODIFIED reference (elfi-dev/elfi, the
checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_testbench_bsl.py

testbench_bsl.npz: ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4), repetitions=3,
seed=156, neither observations nor reference parameters given, one method: BSL with feature MA2,
n_sim_round=200, the default likelihood, 50 iterations from params0 = [.6, .2] with the proposal
covariance [[.02, .01], [.01, .02]].  Proposals that leave MA2's triangular prior simulate nothing,
so the repetitions end with different n_sim.  Keys: observations, ref_{t}, seeds, and per
repetition r: r{r}_samples_all (n_iter, 2), r{r}_logposterior, r{r}_acc_rate and r{r}_nsim.
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

LOGPOSTERIORS = []


class RecordingBSL(elfi.BSL):
    """elfi.BSL that keeps a copy of state['logposterior'] when a run ends; the sampler's
    arithmetic is the reference's own."""

    def extract_result(self):
        LOGPOSTERIORS.append(np.array(self.state['logposterior']))
        return super().extract_result()


CASE = dict(n_obs=50, true_params=[.6, .2], seed_obs=4, repetitions=3, seed=156)
METHOD = dict(n_sim_round=200, feature_names=['MA2'])
SAMPLE = dict(n_samples=50, sigma_proposals=[[.02, .01], [.01, .02]], params0=[.6, .2])


def main():
    m = ma2.get_model(n_obs=CASE['n_obs'], true_params=CASE['true_params'],
                      seed_obs=CASE['seed_obs'])
    tb = elfi.Testbench(model=m, repetitions=CASE['repetitions'], seed=CASE['seed'],
                        progress_bar=False)
    method = elfi.TestbenchMethod(method=RecordingBSL, name='BSL')
    method.set_method_kwargs(**METHOD)
    method.set_sample_kwargs(n_samples=SAMPLE['n_samples'],
                             sigma_proposals=np.array(SAMPLE['sigma_proposals']),
                             params0=np.array(SAMPLE['params0']))
    tb.add_method(method)
    tb.run()
    out = dict(observations=np.asarray(tb.observations), seeds=np.asarray(tb.method_seed_list[0]))
    for t in ('t1', 't2'):
        out['ref_' + t] = np.asarray(tb.reference_parameter[t])
    for r, s in enumerate(tb.testbench_results[0]['results']):
        out['r{}_samples_all'.format(r)] = np.column_stack([s.samples_all[p] for p in ('t1', 't2')])
        out['r{}_logposterior'.format(r)] = LOGPOSTERIORS[r]
        out['r{}_acc_rate'.format(r)] = np.float64(s.acc_rate)
        out['r{}_nsim'.format(r)] = np.int64(s.n_sim)
    np.savez(os.path.join(HERE, 'testbench_bsl.npz'), **out)
    print('wrote testbench_bsl', {k: np.shape(v) for k, v in out.items()},
          [int(out['r{}_nsim'.format(r)]) for r in range(CASE['repetitions'])])


if __name__ == '__main__':
    main()
