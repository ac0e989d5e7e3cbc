"""Models of the ROMC tests, built with either package's API (elfi_b200 or the reference's elfi):
TEST INFRASTRUCTURE ONLY.

`one_d_model` is the one-parameter example of the reference's ROMC functional test, restated: a
uniform prior on [-2.5, 2.5] and one observation y ~ N(m(theta), 1) with m(theta) = -theta - c for
theta <= -0.5, theta^4 for |theta| <= 0.5 and theta - c above, c = 0.5 - 0.5^4; observed y = 0 and
a Euclidean distance.  Its posterior has E[theta] = 0 and E[theta^2] close to 1.1."""
import numpy as np
import scipy.stats as ss

C = 0.5 - 0.5 ** 4


class UniformPrior:
    """Uniform on [-2.5, 2.5]; draws of shape (size..., 1)."""

    def rvs(self, size=None, random_state=None):
        if size is not None:
            size = tuple(np.atleast_1d(size)) + (1,)
        return ss.uniform(loc=-2.5, scale=5).rvs(size=size, random_state=random_state)

    def pdf(self, theta):
        return ss.uniform(loc=-2.5, scale=5).pdf(theta)

    def logpdf(self, theta):
        return ss.uniform(loc=-2.5, scale=5).logpdf(theta)


def likelihood_mean(theta):
    theta = np.asarray(theta, dtype=float)
    return np.where(theta <= -0.5, -theta - C, np.where(theta <= 0.5, theta ** 4, theta - C))


def simulator(theta, dim, batch_size=1, random_state=None):
    """One N(m(theta), 1) draw per entry of theta repeated dim times along the last axis."""
    m = likelihood_mean(np.repeat(theta, dim, -1))
    rs = random_state if random_state is not None else np.random
    return m + rs.standard_normal(m.shape)


def one_d_model(api):
    """The model and its discrepancy node name, built with `api` (a module with new_model, Prior,
    Simulator and Distance)."""
    m = api.new_model('romc_1d')
    prior = api.Prior(UniformPrior(), name='theta')
    sim = api.Simulator(simulator, prior, 1, observed=np.zeros((1, 1)), name='simulator')
    api.Distance('euclidean', sim, name='dist')
    return m, 'dist'
