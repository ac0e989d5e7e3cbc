"""The six-parameter model of the DeviceModelPrior tests (one prior of every supported kind) and
the per-kind cases -- shared by tests/test_priors_host.py and tests/test_device_priors_gpu.py."""
import numpy as np
import scipy.stats as ss

# (kind, scipy positional parameters): every kind, defaulted loc / scale, the upper tail of
# truncnorm, gamma shapes below, at and above 1, beta's U shape, flat and skewed forms
KIND_CASES = [('uniform', (-1.0, 2.0)), ('uniform', ()), ('norm', (50.0, 7.0)), ('norm', ()),
              ('truncnorm', (0.0, 5.0)), ('truncnorm', (9.0, 12.0)), ('truncnorm', (-12.0, -9.0)),
              ('truncnorm', (-1.0, 2.0, 1.0, 2.0)), ('expon', (np.e, 2.0)), ('expon', ()),
              ('gamma', (0.3,)), ('gamma', (1.0,)), ('gamma', (2.5,)), ('gamma', (2.0, 0.0, 0.5)),
              ('beta', (0.5, 0.5)), ('beta', (1.0, 1.0)), ('beta', (2.0, 5.0)),
              ('beta', (2.0, 3.0, -1.0, 4.0))]

SIX_PRIORS = [('norm', (0.0, 1.0)), ('uniform', (-1.0, 2.0)), ('truncnorm', (0.0, 3.0)),
              ('expon', (0.0, 1.0)), ('gamma', (2.0, 0.0, 0.5)), ('beta', (2.0, 3.0))]
SIX_NAMES = ['t{}'.format(i) for i in range(6)]
SIX_TRUE = np.array([0.3, 0.2, 1.0, 0.8, 1.2, 0.4])
NOISE = 0.1


def case_id(case):
    return '{}{}'.format(case[0], ','.join('{:g}'.format(v) for v in case[1]))


def frozen(kind, params):
    return getattr(ss, kind)(*params)


def sim6(*theta, batch_size=1, random_state=None):
    """y = theta + 0.1 eps: on the device (eps from a torch generator seeded from the batch's
    random state) when any parameter is a device array, else on the host from the RandomState."""
    import torch
    from elfi_b200 import device as dev
    from elfi_b200.examples.gauss import _key
    if any(dev.is_device_array(t) for t in theta):
        cols = [t.reshape(-1) if dev.is_device_array(t) else
                dev.to_device(np.broadcast_to(np.asarray(t, dtype=np.float64).reshape(-1),
                                              (batch_size,)).copy()) for t in theta]
        th = torch.stack(cols, 1)
        g = torch.Generator(device=th.device)
        g.manual_seed(_key(random_state))
        eps = torch.randn(tuple(th.shape), generator=g, device=th.device, dtype=torch.float64)
        return th + dev.to_device(eps) * NOISE
    random_state = random_state or np.random
    th = np.column_stack([np.broadcast_to(np.asarray(t, dtype=np.float64).reshape(-1), (batch_size,))
                          for t in theta])
    return th + NOISE * random_state.randn(*th.shape)


def _column(i):
    def col(y):
        return y[:, i]
    return col


def six_model(seed_obs=11):
    """theta ~ (norm(0, 1), uniform(-1, 2), truncnorm(0, 3), expon(0, 1), gamma(2, 0, 0.5),
    beta(2, 3)); y = theta + 0.1 eps; Euclidean distance over six identity summaries."""
    from elfi_b200 import model as em
    m = em.new_model()
    priors = [em.Prior(kind, *params, model=m, name=n) for n, (kind, params) in zip(SIX_NAMES, SIX_PRIORS)]
    y_obs = SIX_TRUE[None, :] + NOISE * np.random.RandomState(seed_obs).randn(1, 6)
    em.Simulator(sim6, *priors, observed=y_obs, name='sim')
    summaries = [em.Summary(_column(i), m['sim'], name='s{}'.format(i)) for i in range(6)]
    em.Distance('euclidean', *summaries, name='d')
    return m
