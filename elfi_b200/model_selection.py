"""ABC model choice from the samples of several models (elfi/methods/model_selection.py)."""
import numpy as np


def compare_models(sample_objs, model_priors=None):
    """Posterior probabilities of the models that produced `sample_objs` (elfi.compare_models).

    The discrepancies of all samples are pooled and the n_min smallest kept, n_min being the
    smallest sample size.  Each model's share of them is divided by the number of simulations it
    ran, multiplied by its prior probability (1 / n_models when `model_priors` is None) and the
    shares are normalised.  The discrepancies must be comparable for this to mean anything: the
    same distance on the same summaries of the same observed data.

    Parameters
    ----------
    sample_objs : list of Sample
        Results of prerun inference (e.g. Rejection.sample), each with `discrepancies`,
        `n_samples` and `n_sim`.
    model_priors : array_like, optional
        Prior probability of each model.

    Returns
    -------
    np.array of the posterior probabilities, one per model.

    The arithmetic is the reference's on host arrays (device-backed discrepancies are read to the
    host: n_samples doubles per model), so equal inputs give equal bits.
    """
    n_models = len(sample_objs)
    sizes = [s.n_samples for s in sample_objs]
    n_min = min(sizes)
    try:
        pooled = np.concatenate([s.discrepancies for s in sample_objs])
    except ValueError:
        raise ValueError('All Sample objects must include valid discrepancies.')
    best = np.argsort(pooled)[:n_min]

    p = np.empty(n_models)
    start = 0
    for i, s in enumerate(sample_objs):
        end = start + sizes[i]
        p[i] = np.logical_and(best >= start, best < end).sum()
        p[i] /= s.n_sim
        if model_priors is not None:
            p[i] *= model_priors[i]
        start = end
    return p / p.sum()
