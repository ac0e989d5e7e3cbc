"""Device priors and SMC proposals for any model whose priors are stock scipy.stats distributions.

``DeviceModelPrior(model)`` checks that every parameter of the model is an independent Prior of a
supported kind (uniform, norm, truncnorm, expon, gamma, beta; also ELFI's shorthands 'normal',
'exponential', 'unif' and the scipy distribution objects) with constant scalar parameters, and
then offers the throughput mode's two device paths for it:

* ``.model``: a copy of the model whose priors draw on the device (ops.prior_rvs, keyed by the
  batch's random state like the bundled examples' device priors); their pdf / logpdf are scipy's,
  so the host ModelPrior of the copy is unchanged;
* the ``device_proposal`` protocol of SMC / AdaptiveDistanceSMC / AdaptiveThresholdSMC:
  ``rvs`` = the mixture proposal redrawn until the joint prior log density is finite
  (ops.gm_rvs support 3, the rule of GMDistribution.rvs), ``logpdf`` = ops.prior_logpdf.

    dp = elfi_b200.DeviceModelPrior(m)
    elfi_b200.SMC(dp.model['d'], device_proposal=dp, batch_size=..., seed=...)

Conditional priors.  ``DeviceModelPrior(model, conditional=True)`` also accepts a prior whose loc
and / or scale is another Prior of the model, ELFI's hierarchical style, as in
``Prior('uniform', m['t1'], 10, name='t2')`` (t2 ~ U(t1, t1 + 10)).  The parent's column is recorded
in ``sources`` ((p, 2): [loc_src, scale_src], -1 for a constant): the device draws take the
parent's draws as per-row loc / scale (ops.prior_rvs), and the proposals and densities read them
from the same row (ops.gm_rvs support 4, ops.prior_logpdf with sources).  A model without such a
parameter makes exactly the calls of one with constant priors (support 3, a (p, 5) table).  The
default, ``conditional=False``, keeps the constant-parameter contract: a prior with a node parent
is refused, so a model is never silently given a different device prior family than it was
checked for.

Rejected with a ValueError naming the node: a node parent (without ``conditional=True``; with it, a
node parent in a shape position -- truncnorm's a, b, gamma's a, beta's a, b -- or a parent that is
not a Prior, such as an Operation or a Simulator), vector priors (``size=``) and other
distributions.

    dp = elfi_b200.DeviceModelPrior(m, conditional=True)     # e.g. examples.mg1
"""
from functools import partial

import numpy as np
import scipy.stats as ss

from . import device as dev
from . import model as em
from . import ops
from .throughput import batch_key

SUPPORTED = ops.PRIOR_KINDS


def _kind_of(distribution):
    """(kind name or None, description) of a Prior's distribution attribute."""
    if isinstance(distribution, str):
        name = distribution.lower()
        name = em._SCIPY_SHORTHAND.get(name, name)
        return (name if name in SUPPORTED else None), "'{}'".format(distribution)
    if isinstance(distribution, DevicePriorDistribution):
        return distribution.kind, distribution.kind
    for name in SUPPORTED:
        if distribution is getattr(ss, name):
            return name, 'scipy.stats.' + name
    if isinstance(distribution, ss.rv_continuous) or isinstance(distribution, ss.rv_discrete):
        return None, 'scipy.stats.' + str(getattr(distribution, 'name', distribution))
    return None, 'custom distribution {}'.format(getattr(distribution, '__name__', distribution))


def prior_spec(kind, params):
    """[kind index, p0, p1, p2, p3] of scipy's positional parameters, loc 0 and scale 1 by
    default (as in scipy)."""
    shapes = ops.PRIOR_SHAPES[kind]
    params = [float(v) for v in params]
    ns = len(shapes)
    if len(params) < ns or len(params) > ns + 2:
        raise ValueError('{} takes {} positional parameters ({}), got {}'.format(
            kind, 'from {} to {}'.format(ns, ns + 2) if ns else 'at most 2',
            ', '.join(shapes + ('loc', 'scale')), len(params)))
    full = params + [0.0, 1.0][len(params) - ns:]
    spec = [float(SUPPORTED.index(kind))] + full
    return spec + [0.0] * (ops.PRIOR_SPEC_WORDS - len(spec))


class DevicePriorDistribution:
    """A stock prior that draws on the device: ``rvs`` returns a device tensor from
    ops.prior_rvs keyed by the batch's random state; ``pdf`` / ``logpdf`` are scipy's."""

    def __init__(self, kind):
        self.kind = kind
        self.scipy = getattr(ss, kind)
        self.__name__ = 'device_' + kind

    def rvs(self, *params, size=1, random_state=None):
        """Draws with scalar parameters; a loc or scale that is a vector (the draws of a parent
        prior, one per row) goes to ops.prior_rvs per row."""
        n = int(np.prod(size))
        ns = len(ops.PRIOR_SHAPES[self.kind])
        consts, rows = [], {}
        for i, v in enumerate(params):
            if i >= ns and (dev.is_device_array(v) or np.ndim(v) > 0):
                rows['loc' if i == ns else 'scale'] = v
                v = 0.0 if i == ns else 1.0
            consts.append(v)
        return ops.prior_rvs(prior_spec(self.kind, consts), n, batch_key(random_state), **rows)

    def pdf(self, x, *params):
        return self.scipy.pdf(x, *params)

    def logpdf(self, x, *params):
        return self.scipy.logpdf(x, *params)


def _node_spec(model, name, conditional):
    rec = model.record(name)
    if not issubclass(rec.cls, em.RandomVariable):
        raise ValueError("parameter '{}' is not a Prior ({})".format(name, rec.cls.__name__))
    if rec.attrs.get('size') is not None:
        raise ValueError("prior '{}' is a vector prior (size={}); only scalar priors run on the "
                         "device".format(name, rec.attrs['size']))
    kind, what = _kind_of(rec.attrs['distribution'])
    if kind is None:
        raise ValueError("prior '{}': {} is not supported on the device (supported: {})".format(
            name, what, ', '.join(SUPPORTED)))
    ns = len(ops.PRIOR_SHAPES[kind])
    values, parents = [], [None, None]
    for i, parent in enumerate(rec.inputs):
        prec = model.record(parent)
        if not issubclass(prec.cls, em.Constant):
            if not conditional:
                raise ValueError("prior '{}': parameter {} depends on node '{}'; only priors with "
                                 "constant parameters run on the device (a loc or scale that is "
                                 "another Prior needs DeviceModelPrior(model, conditional=True))"
                                 .format(name, i, parent))
            if i < ns:
                raise ValueError("prior '{}': its shape parameter {} ({}) depends on node '{}'; "
                                 "only loc and scale may come from another prior".format(
                                     name, i, ops.PRIOR_SHAPES[kind][i], parent))
            if not issubclass(prec.cls, em.Prior) or i > ns + 1:
                raise ValueError("prior '{}': parameter {} depends on node '{}' ({}); loc and "
                                 "scale may come from another Prior only".format(
                                     name, i, parent, prec.cls.__name__))
            parents[i - ns] = parent
            values.append(0.0 if i == ns else 1.0)     # placeholders
            continue
        v = prec.constant
        if np.ndim(v) != 0 or not np.isreal(v):
            raise ValueError("prior '{}': parameter {} is not a real scalar ({!r})".format(
                name, i, v))
        values.append(float(np.real(v)))
    try:
        spec = prior_spec(kind, values)
    except ValueError as e:
        raise ValueError("prior '{}': {}".format(name, e)) from None
    why = ops._prior_spec_error(np.asarray(spec))
    if why:
        raise ValueError("prior '{}': {}".format(name, why))
    return kind, spec, parents


def _device_copy(model, kinds):
    """The model with each named Prior drawing on the device (same name, parents, observed)."""
    twin = model.copy()
    for name, kind in kinds.items():
        rec = twin.record(name)
        dist = DevicePriorDistribution(kind)
        new = rec.twin()
        new.attrs = dict(rec.attrs, distribution=dist)
        new.op = partial(em._draw, distribution=dist, size=None)
        twin._records[name] = new
    return twin


class DeviceModelPrior:
    """Joint prior of a model with stock scipy.stats priors, on the device (see the module
    docstring).  ``parameter_names`` are the model's (sorted) parameter names; ``specs`` is the
    (p, 5) table handed to the kernels and ``sources`` (p, 2) the columns a conditional loc /
    scale comes from (-1: the constant in ``specs``).  ``conditional=True`` accepts a loc or scale
    that is another Prior; by default only constant parameters are accepted."""

    def __init__(self, model, conditional=False):
        names = list(model.parameter_names)
        if not names:
            raise ValueError('the model has no parameters')
        if len(names) > ops.MAX_PRIOR_PARAMS:
            raise ValueError('{} parameters; the device priors take at most {}'.format(
                len(names), ops.MAX_PRIOR_PARAMS))
        kinds, specs, sources = {}, [], []
        for name in names:
            kind, spec, parents = _node_spec(model, name, conditional)
            kinds[name] = kind
            specs.append(spec)
            sources.append([-1 if p is None else names.index(p) for p in parents])
        self.parameter_names = names
        self.kinds = [kinds[n] for n in names]
        self.specs = np.asarray(specs, dtype=np.float64)
        self.sources = np.asarray(sources, dtype=np.int64).reshape(len(names), 2)
        self._cond = bool((self.sources >= 0).any())
        self.model = _device_copy(model, kinds)

    def rvs(self, means, cov, weights, size, key, cdf=None):
        """Mixture proposals (GMDistribution.rvs) redrawn until the joint prior density is
        positive; a (size, p) device tensor."""
        if self._cond:
            return ops.gm_rvs(means, cov, weights, size, seed=key, support=4, prior=self.specs,
                              sources=self.sources, cdf=cdf)
        return ops.gm_rvs(means, cov, weights, size, seed=key, support=3, prior=self.specs, cdf=cdf)

    def logpdf(self, params):
        """Joint prior log density of the rows of params (B, p); a device tensor (B,)."""
        return ops.prior_logpdf(params, self.specs, self.sources if self._cond else None)
