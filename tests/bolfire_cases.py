"""Models shared by the BOLFIRE tests: the LFIRE paper's toy Gaussian with power summaries (the
reference's tests/functional/test_bolfire.py) -- TEST INFRASTRUCTURE ONLY."""
import numpy as np

import elfi_b200 as elfi


def gauss(mu, sigma=3, n_obs=1, batch_size=1, seed=None, *args, **kwargs):
    if isinstance(seed, int):
        np.random.seed(seed)
    mu = np.asanyarray(mu).reshape((-1, 1))
    sigma = np.asanyarray(sigma).reshape((-1, 1))
    return np.random.normal(mu, sigma, size=(batch_size, n_obs))


def power(x, y):
    return x ** y


def simple_gaussian_model(true_param=2.6, seed=4, n_summaries=10):
    m = elfi.ElfiModel()
    mu = elfi.Prior('uniform', -5, 10, model=m, name='mu')
    y = elfi.Simulator(gauss, *[mu], observed=gauss(true_param, seed=seed), name='y')
    for i in range(n_summaries):
        elfi.Summary(power, y, i, model=m, name='power_{}'.format(i))
    return m
