"""BOLFIRE with the device classifier: the reference's rounds on the host ARCH model, the
reference's functional test on its toy Gaussian, and a fully device-side ARCH run."""
import numpy as np
import pytest
import torch

from bolfire_cases import simple_gaussian_model
from elfi_b200 import device as dev
from elfi_b200 import ops
from elfi_b200.bolfire import BOLFIRE
from elfi_b200.examples import arch
from elfi_b200.results import BOLFIRESample

pytestmark = pytest.mark.gpu

BOUNDS = {'t1': (-1, 1), 't2': (0, 1)}


def test_rounds_match_reference(golden, monkeypatch):
    g = golden('bolfire_rounds')
    reads = []
    to_host = dev.to_host

    def counting(x):
        if isinstance(x, torch.Tensor) and x.is_cuda and x.numel() == ops.logreg_block_size(17) + 1:
            reads.append(1)
        return to_host(x)
    monkeypatch.setattr(dev, 'to_host', counting)
    m = arch.get_model(n_obs=100, seed_obs=int(g['seed_obs']))
    n = int(g['n_initial_evidence'])
    bolfire = BOLFIRE(m, int(g['n_training_data']), seed_marginal=int(g['seed_marginal']),
                      bounds=BOUNDS, n_initial_evidence=n, seed=int(g['seed']))
    post = bolfire.fit(n, bar=False)
    np.testing.assert_array_equal(bolfire.marginal.cpu().numpy(), g['marginal'])
    np.testing.assert_array_equal(bolfire.target_model.X, g['theta'])
    v, ref = bolfire.target_model.Y[:, 0], g['value_tight']
    assert np.all(np.abs(v - ref) <= 1e-7 * (1 + np.abs(ref)))
    assert len(reads) == n                          # one result read per round
    assert len(post.classifier_attributes) == n


def test_functional_toy_gaussian():
    """The reference's tests/functional/test_bolfire.py at its own size."""
    m = simple_gaussian_model(2.6, 4)
    bolfire_method = BOLFIRE(model=m, n_training_data=500, n_initial_evidence=10,
                             update_interval=1, bounds={'mu': (-5, 5)}, seed=1)
    post = bolfire_method.fit(100, bar=False)
    assert bolfire_method.n_evidence == 100
    map_estimates = post.compute_map_estimates()
    assert np.abs(map_estimates['mu'] - 2.6) <= 0.5
    sample = bolfire_method.sample(400)
    assert isinstance(sample, BOLFIRESample)
    assert np.abs(sample.sample_means['mu'] - 2.6) <= 1.5


def test_device_arch():
    m, _ = arch.get_device_model(n_obs=100, true_params=[0.3, 0.7], seed_obs=5)
    bolfire = BOLFIRE(m, 500, bounds=BOUNDS, n_initial_evidence=10, seed=3, seed_marginal=4)
    post = bolfire.fit(40, bar=False)
    assert bolfire.n_evidence == 40
    est = post.compute_map_estimates()
    assert abs(est['t1'] - 0.3) <= 0.5 and abs(est['t2'] - 0.7) <= 0.5, est
    sample = bolfire.sample(200, n_chains=2)
    assert sample.chains.shape == (2, 200, 2)
    s = sample.samples_array
    assert np.all((s[:, 0] >= -1) & (s[:, 0] <= 1) & (s[:, 1] >= 0) & (s[:, 1] <= 1))
    attrs = post.classifier_attributes
    assert len(attrs) == 40 and np.shape(attrs[0]['parameters']['coef_']) == (1, 17)
    sm = post.surrogate_model_attributes
    assert len(sm['parameters']) == 4 and len(sm['X']) == 40
