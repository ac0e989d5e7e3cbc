"""Ratio-estimation classifiers of BOLFIRE (elfi/methods/classifier.py).

`LogisticRegression` is the reference's default classifier (StandardScaler, then liblinear's
L1-penalised logistic regression) fitted on the device by ops.logreg_fit.  It solves the same
objective to its optimum rather than to liblinear's tolerance 1e-4 (DESIGN.md section 7), so its
coefficients are those of liblinear at a tight tolerance.  A user subclass of `Classifier` runs on
the host with NumPy (X, y).  scikit-learn is not used.
"""
import abc
import logging
import warnings

import numpy as np

from . import device as dev
from . import ops

logger = logging.getLogger(__name__)

__all__ = ['Classifier', 'LogisticRegression', 'GPClassifier', 'ConvergenceWarning']


class ConvergenceWarning(UserWarning):
    """The classifier's solver stopped before its optimality test held."""


class Classifier(abc.ABC):
    """An abstract base class for a ratio estimation classifier: fit(X, y) on NumPy features and
    binary labels, predict_log_likelihood_ratio(X) and an `attributes` dictionary."""

    @abc.abstractmethod
    def __init__(self):
        raise NotImplementedError

    @abc.abstractmethod
    def fit(self, X, y):
        raise NotImplementedError

    @abc.abstractmethod
    def predict_log_likelihood_ratio(self, X):
        raise NotImplementedError

    def predict_likelihood_ratio(self, X):
        return np.exp(self.predict_log_likelihood_ratio(X))

    @property
    @abc.abstractmethod
    def attributes(self):
        raise NotImplementedError


class LogisticRegression(Classifier):
    """A logistic regression classifier for ratio estimation, fitted on the device.

    config: the reference's scikit-learn keyword dictionary.  Supported keys: 'penalty' ('l1' or
    'l2'), 'solver' ('liblinear'), 'C' (> 0) and 'max_iter' (Newton steps); anything else raises
    NotImplementedError.  class_min (int or float) is the floor of the class probability."""

    SUPPORTED = ('penalty', 'solver', 'C', 'max_iter')

    def __init__(self, config=None, class_min=0):
        self.config = self._resolve_config(config)
        self.class_min = self._resolve_class_min(class_min)
        self.penalty = self.config['penalty']
        self.C = float(self.config.get('C', 1.0))
        self.max_iter = int(self.config.get('max_iter', 100))
        if not (self.C > 0 and np.isfinite(self.C)):
            raise ValueError('C must be positive and finite, got {}'.format(self.C))
        self._fit = None

    def _default_config(self):
        return {'penalty': 'l1', 'solver': 'liblinear'}

    def _resolve_config(self, config):
        if not isinstance(config, dict):
            return self._default_config()
        config = dict(config)
        for key in config:
            if key not in self.SUPPORTED:
                raise NotImplementedError(
                    'LogisticRegression: config key {!r} is not supported (supported: {})'.format(
                        key, ', '.join(self.SUPPORTED)))
        config.setdefault('penalty', 'l2')     # scikit-learn's default when the key is absent
        config.setdefault('solver', 'liblinear')
        if config['penalty'] not in ops.LOGREG_PENALTIES:
            raise NotImplementedError("LogisticRegression: penalty={!r} is not supported (use 'l1' "
                                      "or 'l2')".format(config['penalty']))
        if config['solver'] != 'liblinear':
            raise NotImplementedError("LogisticRegression: solver={!r} is not supported (use "
                                      "'liblinear')".format(config['solver']))
        return config

    def _resolve_class_min(self, class_min):
        if isinstance(class_min, (int, float)):
            return class_min
        raise TypeError('class_min has to be either non-negative int or float')

    def fit(self, X, y):
        """Fit on (n, d) features and n labels of two classes; the larger label is the positive
        class (the numerator of the ratio).  X may be a device tensor."""
        y = np.asarray(dev.to_host(y)).reshape(-1)
        classes = np.unique(y)
        if len(classes) != 2:
            raise ValueError('This solver needs samples of exactly 2 classes in the data, but the '
                             'data contains {} classes'.format(len(classes)))
        labels = np.where(y == classes[1], 1.0, -1.0)
        self.fit_device(X, labels)
        self._fit.check()
        self._warn_if_not_converged()

    def fit_device(self, X, labels, out=None):
        """Start the device fit of X with labels +1 / -1 (host or device) without reading it."""
        self._fit = ops.logreg_fit(X, labels, penalty=self.penalty, C=self.C,
                                   max_iter=self.max_iter, out=out)
        return self._fit

    def _warn_if_not_converged(self):
        if not self._fit.converged:
            warnings.warn('LogisticRegression: the Newton iterations did not converge within '
                          'max_iter={}; the last iterate is used'.format(self.max_iter),
                          ConvergenceWarning)

    def predict_device(self, X, out=None):
        if self._fit is None:
            raise ValueError('LogisticRegression: call fit before predicting')
        return ops.logreg_predict(self._fit, X, class_min=self.class_min, out=out)

    def predict_log_likelihood_ratio(self, X):
        """log(p / (1 - p)) per row, p = max(P(positive class), class_min), as NumPy."""
        if not dev.is_device_array(X):
            X = np.atleast_2d(np.asarray(X, dtype=np.float64))
            if not np.all(np.isfinite(X)):
                raise ValueError('Input X contains NaN or infinity.')
        out = dev.to_host(self.predict_device(X))
        if np.any(np.isnan(out)):
            raise ValueError('Input X contains NaN or infinity.')
        return out

    @property
    def coef_(self):
        return self._fit.coef_[None, :].copy()

    @property
    def intercept_(self):
        return np.array([self._fit.intercept_])

    @property
    def n_iter_(self):
        return np.array([self._fit.n_iter], dtype=np.int32)

    @property
    def attributes(self):
        return {'parameters': {'coef_': self.coef_.tolist(),
                               'intercept_': self.intercept_.tolist(),
                               'n_iter': self.n_iter_.tolist()}}


class GPClassifier(Classifier):
    """The reference's Gaussian process classifier needs GPy, which is not available."""

    def __init__(self, kernel=None, mean_function=None, class_min=0):
        raise NotImplementedError('GPClassifier (GPy\'s GPClassification) is not provided; use '
                                  'LogisticRegression or a Classifier subclass')

    def fit(self, X, y):
        raise NotImplementedError

    def predict_log_likelihood_ratio(self, X):
        raise NotImplementedError

    @property
    def attributes(self):
        raise NotImplementedError
