"""Regression adjustment of a posterior sample (elfi/methods/post_processing.py): the local-linear
adjustment of Beaumont et al. (2002), the usual last step after rejection ABC.

Each parameter is regressed, with an intercept, on the differences x = S - observed of the named
summaries, over the rows where x and the parameter are finite, and the adjusted draws are
theta - x @ coef.  `adjust_posterior`, `LinearAdjustment`, `RegressionAdjustment` and
`_get_adjustment` keep the reference's names, arguments, attributes and errors.

`LinearAdjustment` runs on the device (ops.linear_adjust): the row masks, the centred moments of
[x | theta] and the adjusted columns are CUDA kernels, and the adjusted sample's outputs stay on the
device until they are read.  The least-squares solve is done on the host, once per group of rows,
from the count, means and (q + p)^2 moments read back (at most 0.5 MB): one eigen-decomposition of
the q x q block, keeping eigenvalues above tol^2 lambda_max, which is scikit-learn's singular-value
cut (tol = 1e-6) carried over to the normal equations, and giving its minimum-norm solution.  It is
the same kind of small set-up step as bsl.estimate_whitening_matrix.

A subclass of `RegressionAdjustment` with its own `_regression_model` (anything with
`fit(X, y)`), `_adjust` and `_input_variables` runs on the host with NumPy, as in the reference.
"""
import warnings

import numpy as np

from . import ops, results

__all__ = ('LinearAdjustment', 'adjust_posterior')

_NONFINITE_WARNING = 'Non-finite inputs and outputs will be omitted.'


def _column(sample, name):
    """The output `name` of a sample: the device array when the outputs live on the device."""
    if isinstance(sample.outputs, results.DeviceOutputs):
        return sample.outputs.device[name]
    return sample.outputs[name]


def _observed(model, summary_names):
    """The observed value of each summary, one scalar each."""
    obs = []
    for s in summary_names:
        v = np.asarray(results._host(model[s].observed), dtype=np.float64).reshape(-1)
        if v.size != 1:
            raise ValueError('summary {!r} must have one observed value per row, its observed '
                             'value has {}'.format(s, v.size))
        obs.append(v[0])
    return np.array(obs)


class LinearRegression:
    """A least-squares fit with an intercept, with the attributes of scikit-learn's
    LinearRegression on dense input: coef_, intercept_, rank_ and singular_, with singular values
    at or below tol * sigma_max counted as zero.  `fit` runs on the device (ops.linear_adjust).
    copy_X and n_jobs are accepted and have no effect."""

    def __init__(self, fit_intercept=True, copy_X=True, tol=1e-6, n_jobs=None, positive=False):
        if not fit_intercept:
            raise NotImplementedError('LinearRegression(fit_intercept=False) is not supported: '
                                      'the adjustment always fits an intercept')
        if positive:
            raise NotImplementedError('LinearRegression(positive=True) is not supported: the '
                                      'adjustment solves unconstrained least squares')
        self.fit_intercept, self.copy_X, self.n_jobs, self.positive = True, copy_X, n_jobs, False
        self.tol = float(tol)

    def _set(self, fit):
        self.coef_ = fit['coef']
        self.intercept_ = fit['intercept']
        self.rank_ = fit['rank']
        self.singular_ = fit['singular']
        self.n_rows_ = fit['n_rows']
        return self

    def fit(self, X, y):
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64)
        if X.ndim != 2 or y.ndim != 1 or len(y) != len(X):
            raise ValueError('fit takes X (n, q) and y (n,), got shapes {} and {}'.format(
                X.shape, y.shape))
        _, fits = ops.linear_adjust(X, y[:, None], np.zeros(X.shape[1]), tol=self.tol)
        return self._set(fits[0])

    def predict(self, X):
        return np.asarray(X, dtype=np.float64) @ self.coef_ + self.intercept_


class RegressionAdjustment:
    """Base class of regression adjustments: one regression per scalar parameter, with the
    summaries as regressors.  Keyword arguments go to the regression model.

    A subclass sets `_regression_model` (a class whose instances have `fit(X, y)`), `_name`,
    `_adjust(i, theta_i, regression_model)` and `_input_variables(model, sample, summary_names)`.

    Attributes, readable after `fit` (ValueError before): `parameter_names`, `sample` and `X`, the
    regressors.  `regression_models` holds the fitted models."""

    _regression_model = None
    _name = 'RegressionAdjustment'

    def __init__(self, **kwargs):
        self._model_kwargs = kwargs
        self._fitted = False
        self.regression_models = []
        self._X = None
        self._sample = None
        self._parameter_names = None
        self._finite = []
        self._model = None
        self._summary_names = None

    def _check_fitted(self):
        if not self._fitted:
            raise ValueError('The regression model must be fitted first. Use the fit() method.')

    @property
    def parameter_names(self):
        self._check_fitted()
        return self._parameter_names

    @property
    def sample(self):
        self._check_fitted()
        return self._sample

    @property
    def X(self):
        self._check_fitted()
        if self._X is None:
            self._X = self._input_variables(self._model, self._sample, self._summary_names)
        return self._X

    def _remember(self, sample, model, summary_names, parameter_names):
        self._sample, self._model = sample, model
        self._summary_names = list(summary_names)
        self._parameter_names = parameter_names or sample.parameter_names

    def fit(self, sample, model, summary_names, parameter_names=None):
        """Fit one regression per parameter to the sample; rows with a non-finite regressor or
        parameter value are left out of that parameter's fit (one UserWarning if any is)."""
        self._remember(sample, model, summary_names, parameter_names)
        self._X = self._input_variables(model, sample, summary_names)
        rows = np.isfinite(self._X).all(axis=1)
        self._finite = [rows & np.isfinite(np.asarray(sample.outputs[name]))
                        for name in self._parameter_names]
        if not all(mask.all() for mask in self._finite):
            warnings.warn(_NONFINITE_WARNING)
        for i, name in enumerate(self._parameter_names):
            mask = self._finite[i]
            theta = np.asarray(sample.outputs[name])[mask]
            self.regression_models.append(self._fit1(self._X[mask, :], theta))
        self._fitted = True

    def _fit1(self, X, y):
        return self._regression_model(**self._model_kwargs).fit(X, y)

    def adjust(self):
        """A Sample holding the adjusted parameters, each over the rows its fit used."""
        outputs = {}
        for i, name in enumerate(self.parameter_names):
            theta = np.asarray(self.sample.outputs[name])[self._finite[i]]
            outputs[name] = self._adjust(i, theta, self.regression_models[i])
        return results.Sample(method_name=self._name, outputs=outputs,
                              parameter_names=self._parameter_names)

    def _adjust(self, i, theta_i, regression_model):
        """The adjusted values of parameter i from its finite values theta_i and its fit."""
        raise NotImplementedError

    def _input_variables(self, model, sample, summary_names):
        """The (N, q) host matrix of regressors."""
        raise NotImplementedError


class LinearAdjustment(RegressionAdjustment):
    """Regression adjustment with a local linear model, run on the device.  Keyword arguments are
    LinearRegression's: `tol` is honoured, `copy_X` and `n_jobs` have no effect, and
    `fit_intercept=False` or `positive=True` raise NotImplementedError."""

    _regression_model = LinearRegression
    _name = 'LinearAdjustment'

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        if type(self)._regression_model is LinearRegression:
            LinearRegression(**kwargs)       # reject unsupported options now, not at fit
        self._adjusted = None

    def _on_device(self):
        cls = type(self)
        return (cls._regression_model is LinearRegression and
                cls._adjust is LinearAdjustment._adjust and
                cls._input_variables is LinearAdjustment._input_variables)

    def fit(self, sample, model, summary_names, parameter_names=None):
        if not self._on_device():
            return super().fit(sample, model, summary_names, parameter_names)
        S = [_column(sample, s) for s in summary_names]
        observed = _observed(model, summary_names)
        names = list(parameter_names or sample.parameter_names)
        theta = [_column(sample, name) for name in names]
        template = LinearRegression(**self._model_kwargs)
        adjusted, fits = ops.linear_adjust(S, theta, observed, tol=template.tol)
        if any(f['n_rows'] < _rows(S) for f in fits):
            warnings.warn(_NONFINITE_WARNING)
        self._remember(sample, model, summary_names, parameter_names)
        self._X = None
        self.regression_models = [LinearRegression(**self._model_kwargs)._set(f) for f in fits]
        self._adjusted = dict(zip(names, adjusted))
        self._fitted = True

    def adjust(self):
        if self._adjusted is None:
            return super().adjust()
        self._check_fitted()
        return results.Sample(method_name=self._name,
                              outputs=results.DeviceOutputs(self._adjusted),
                              parameter_names=self._parameter_names)

    def _adjust(self, i, theta_i, regression_model):
        return theta_i - self.X[self._finite[i], :] @ regression_model.coef_

    def _input_variables(self, model, sample, summary_names):
        """The differences to the observed summaries."""
        S = np.stack([np.asarray(sample.outputs[s], dtype=np.float64) for s in summary_names],
                     axis=1)
        return S - _observed(model, summary_names)


def _rows(columns):
    return int(columns[0].shape[0]) if hasattr(columns[0], 'shape') else len(columns[0])


def adjust_posterior(sample, model, summary_names, parameter_names=None, adjustment='linear'):
    """Adjust a posterior sample by local regression on the summaries.

    The summaries must be in the sample's outputs: pass them as `output_names` to the sampler.

    Parameters
    ----------
    sample : results.Sample
      a sample of an ABC method
    model : ElfiModel
      the inference model, which holds the observed summaries
    summary_names : list[str]
      names of the summary nodes
    parameter_names : list[str], optional
      the parameters to adjust (default: all of the sample's)
    adjustment : RegressionAdjustment or str
      an adjustment object, or 'linear'

    Returns
    -------
    results.Sample with the adjusted parameters (no weights)."""
    adjustment = _get_adjustment(adjustment)
    adjustment.fit(model=model, sample=sample, parameter_names=parameter_names,
                   summary_names=summary_names)
    return adjustment.adjust()


def _get_adjustment(adjustment):
    if isinstance(adjustment, RegressionAdjustment):
        return adjustment
    cls = {'linear': LinearAdjustment}.get(adjustment) if isinstance(adjustment, str) else None
    if cls is None:
        raise ValueError('Could not find adjustment method: {}'.format(adjustment))
    return cls()
