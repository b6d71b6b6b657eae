"""Scalar likelihoods.  Gaussian (mirrors gpflow/likelihoods/scalar_continuous.py:41-148): a constant variance / scale
Parameter, or heteroskedastic -- `variance=Function` / `scale=Function` (any callable Module mapping X [N, D] to a device
tensor [N, 1], e.g. the mean functions) clipped from below as in the reference.  Bernoulli (probit link), Poisson (exp
link) and StudentT (constant scale) mirror scalar_discrete.py:29-117 and scalar_continuous.py:177-213; what the
reference computes by Gauss-Hermite quadrature (likelihoods/base.py:279-456, 20 points) runs on the device
(csrc/lik.cu), as do the closed forms.  MultiClass with the RobustMax inverse link (multiclass.py:55-243) couples the
latents of a row: its 20-point quadrature of the probability that the labelled latent is the largest runs on the device
too.  HeteroskedasticTFPConditional with a Normal distribution (multilatent.py:95-133) drives the location and the scale
of one output by two latents; its 20 x 20 Gauss-Hermite grid factorises to 20 nodes per row on the device."""
from __future__ import annotations

import math
from typing import Any, Optional

import numpy as np

from . import config, ops
from .base import Exp, Module, Parameter, Shifted, Sigmoid, Softplus, positive


class Likelihood(Module):
    pass


class ScalarLikelihood(Likelihood):
    pass


class Gaussian(ScalarLikelihood):
    def __init__(self, variance: Any = None, *, scale: Any = None, variance_lower_bound: Optional[float] = None):
        self.variance_lower_bound = (config.default_likelihood_positive_minimum()
                                     if variance_lower_bound is None else variance_lower_bound)
        self.scale_lower_bound = math.sqrt(self.variance_lower_bound)
        if scale is None:
            if variance is None:
                variance = 1.0
            # prepare_parameter_or_function (likelihoods/utils.py): a Function is kept, a constant becomes a Parameter
            self.variance: Any = variance if callable(variance) else Parameter(
                variance, transform=positive(lower=self.variance_lower_bound))
            self.scale: Any = None
        else:
            assert variance is None, "Cannot set both `variance` and `scale`."
            self.variance = None
            self.scale = scale if callable(scale) else Parameter(scale, transform=positive(lower=self.scale_lower_bound))

    @property
    def heteroskedastic(self) -> bool:
        return callable(self.variance) or callable(self.scale)

    def _variance_value(self) -> float:  # scalar_continuous.py:92-102, constant case
        if self.heteroskedastic:
            raise NotImplementedError("this operator takes a constant noise variance; heteroskedastic Gaussian "
                                      "likelihoods go through variance_at(X) (GPR, predict_y, predict_log_density)")
        if self.variance is not None:
            return float(self.variance.numpy())
        return float(self.scale.numpy()) ** 2

    def _lik_desc(self, variance: Optional[float] = None):  # the device descriptor (csrc/lik.cu) of a constant variance
        from . import _lib

        variance = self._variance_value() if variance is None else variance
        return _lib.LikDesc(_lib.LIK_GAUSSIAN, DEFAULT_NUM_GAUSS_HERMITE_POINTS, 0.0, 0.0, 0.0, variance)

    def variance_at(self, X):  # scalar_continuous.py:92-111 -> device [N, 1]
        X = ops.to_device(X)
        if not self.heteroskedastic:
            return ops.full((X.shape[0], 1), self._variance_value(), like=X)
        fn, lower, square = (self.variance, self.variance_lower_bound, 0) if self.variance is not None else (
            self.scale, self.scale_lower_bound, 1)
        v = ops.copy(ops.to_device(fn(X)))
        if v.dim() != 2 or v.shape[0] != X.shape[0] or v.shape[1] != 1:
            raise ValueError(f"the noise Function must return [N, 1], got {tuple(v.shape)}")
        from . import _lib
        _lib.check(_lib.load().gpk_clamp_min(ops._p(v), v.shape[0], 1, 1, float(lower), square, ops.dtype_code(v),
                                             ops._stream()), "gpk_clamp_min")
        return v

    def variational_expectations(self, X, Fmu, Fvar, Y):
        """Sum over the batch of scalar_continuous.py:139-148, returned as a device fp64 scalar [1].
        (The reference returns the per-row vector; every hot-path caller immediately reduce_sums it,
        svgp.py:181, so the reduction is fused.)"""
        return ops.lik_varexp_sum(self._lik_desc(), ops.to_device(Fmu), ops.to_device(Fvar), ops.to_device(Y))

    def predict_mean_and_var(self, X, Fmu, Fvar):  # scalar_continuous.py:127-130
        out = ops.copy(Fvar)
        ops.axpby(1.0, self.variance_at(X), 1.0, out)   # [N, 1] broadcasts over the output columns
        return Fmu, out

    def predict_log_density(self, X, Fmu, Fvar, Y):  # scalar_continuous.py:133-136 -> device vector [N]
        Fmu, Fvar, Y = ops.to_device(Fmu), ops.to_device(Fvar), ops.to_device(Y)
        if self.heteroskedastic:  # the variance folded into Fvar, the descriptor's noise 0
            tot = ops.copy(Fvar)
            ops.axpby(1.0, self.variance_at(X), 1.0, tot)
            return ops.lik_predict_log_density(self._lik_desc(0.0), Fmu, tot, Y)
        return ops.lik_predict_log_density(self._lik_desc(), Fmu, Fvar, Y)


def inv_probit(x):
    """utils.py::inv_probit: the standard normal CDF squeezed into [1e-3, 1 - 1e-3] (the link Bernoulli computes with)."""
    from scipy.special import erf

    jitter = 1e-3
    return 0.5 * (1.0 + erf(np.asarray(x) / np.sqrt(2.0))) * (1 - 2 * jitter) + jitter


DEFAULT_NUM_GAUSS_HERMITE_POINTS = 20


def _no_custom_quadrature(quadrature) -> None:
    if quadrature is not None:
        raise NotImplementedError("the device likelihoods use the reference's default quadrature "
                                  f"(NDiagGHQuadrature with {DEFAULT_NUM_GAUSS_HERMITE_POINTS} points)")


class _DeviceScalarLikelihood(ScalarLikelihood):
    """A scalar likelihood evaluated by the device operators of csrc/lik.cu through its descriptor `_lik_desc()`.
    variational_expectations returns the device fp64 sum [1] (as Gaussian's does), predict_log_density [N] and
    predict_mean_and_var two [N, P] device tensors."""

    def _lik_desc(self):
        raise NotImplementedError

    def variational_expectations(self, X, Fmu, Fvar, Y):
        return ops.lik_varexp_sum(self._lik_desc(), ops.to_device(Fmu), ops.to_device(Fvar), ops.to_device(Y))

    def predict_mean_and_var(self, X, Fmu, Fvar):
        return ops.lik_predict_mean_and_var(self._lik_desc(), ops.to_device(Fmu), ops.to_device(Fvar))

    def predict_log_density(self, X, Fmu, Fvar, Y):
        return ops.lik_predict_log_density(self._lik_desc(), ops.to_device(Fmu), ops.to_device(Fvar),
                                           ops.to_device(Y))


class Bernoulli(_DeviceScalarLikelihood):
    """scalar_discrete.py:81-117 with the probit link: variational expectations by quadrature, predict_mean_and_var and
    predict_log_density in the closed probit forms."""

    def __init__(self, invlink: Any = inv_probit, *, quadrature: Any = None):
        if invlink is not inv_probit:
            raise NotImplementedError("Bernoulli covers the probit link (likelihoods.inv_probit)")
        _no_custom_quadrature(quadrature)
        self.invlink = invlink

    def _lik_desc(self):
        from . import _lib

        return _lib.LikDesc(_lib.LIK_BERNOULLI, DEFAULT_NUM_GAUSS_HERMITE_POINTS, 0.0, 0.0, 0.0, 0.0)


def _is_exp(f) -> bool:
    if f is np.exp or f is math.exp:
        return True
    try:
        import torch

        return f is torch.exp
    except ImportError:  # pragma: no cover
        return False


class Poisson(_DeviceScalarLikelihood):
    """scalar_discrete.py:29-78 with the exp link: variational expectations in closed form, predict_mean_and_var and
    predict_log_density by quadrature."""

    def __init__(self, invlink: Any = np.exp, binsize: float = 1.0, *, quadrature: Any = None):
        if not _is_exp(invlink):
            raise NotImplementedError("Poisson covers the exp link (numpy.exp, math.exp or torch.exp)")
        _no_custom_quadrature(quadrature)
        self.invlink = invlink
        self.binsize = np.array(binsize, dtype=config.default_float())

    def _lik_desc(self):
        from . import _lib

        return _lib.LikDesc(_lib.LIK_POISSON, DEFAULT_NUM_GAUSS_HERMITE_POINTS, 0.0, 0.0, float(self.binsize), 0.0)


class StudentT(_DeviceScalarLikelihood):
    """scalar_continuous.py:177-213 with a constant scale Parameter: quadrature throughout."""

    def __init__(self, scale: Any = 1.0, df: float = 3.0, scale_lower_bound: Optional[float] = None, *,
                 quadrature: Any = None):
        if callable(scale):
            raise NotImplementedError("StudentT covers a constant scale; a scale Function is not supported")
        _no_custom_quadrature(quadrature)
        self.df = df
        self.scale_lower_bound = (config.default_likelihood_positive_minimum()
                                  if scale_lower_bound is None else scale_lower_bound)
        self.scale = Parameter(scale, transform=positive(lower=self.scale_lower_bound))

    def _lik_desc(self):
        from . import _lib

        return _lib.LikDesc(_lib.LIK_STUDENT_T, DEFAULT_NUM_GAUSS_HERMITE_POINTS, float(self.scale.numpy()),
                            float(self.df), 0.0, 0.0)


class BetaPrior:
    """The record of a Beta(concentration1, concentration0) prior.  The package evaluates no prior densities: a trainable
    Parameter with a prior is refused by the device gradients (the reference would add the prior's log density)."""

    def __init__(self, concentration1: float, concentration0: float):
        self.concentration1, self.concentration0 = float(concentration1), float(concentration0)

    def __repr__(self) -> str:
        return f"Beta({self.concentration1}, {self.concentration0})"


class RobustMax(Module):
    """multiclass.py:55-155: the inverse link y_i = 1 - epsilon for i = argmax(f), epsilon / (k - 1) otherwise.  epsilon,
    the fraction of label errors, is a Parameter in (0, 1) (Sigmoid transform, Beta(0.2, 5) prior) that is not trainable
    by default."""

    def __init__(self, num_classes: int, epsilon: float = 1e-3):
        self.epsilon: Any = Parameter(epsilon, transform=Sigmoid(), prior=BetaPrior(0.2, 5.0), trainable=False)
        self.num_classes = num_classes
        self._squash = 1e-6

    @property
    def eps_k1(self) -> float:
        """epsilon / (num_classes - 1), following epsilon when it is reassigned."""
        return float(self.epsilon) / (self.num_classes - 1.0)


class MultiClass(Likelihood):
    """multiclass.py:158-243 with the RobustMax inverse link: num_classes latent GPs and labels Y [N, 1] (cast to integers
    by truncation; a label outside [0, num_classes) leaves no class out of the product, as the reference's all-zero
    one-hot does).  variational_expectations returns the device fp64 sum [1], predict_mean_and_var the class
    probabilities and their variances [N, num_classes], predict_log_density [N]."""

    def __init__(self, num_classes: int, invlink: Optional[RobustMax] = None):
        self.num_classes = num_classes
        self.num_gauss_hermite_points = DEFAULT_NUM_GAUSS_HERMITE_POINTS
        if invlink is None:
            invlink = RobustMax(num_classes)
        if not isinstance(invlink, RobustMax):
            raise NotImplementedError("MultiClass covers the RobustMax inverse link")
        if invlink.num_classes != num_classes:
            raise ValueError(f"the RobustMax link has {invlink.num_classes} classes, the likelihood {num_classes}")
        self.invlink = invlink

    def _lik_desc(self):
        from . import _lib

        return _lib.LikDesc(_lib.LIK_MULTICLASS, self.num_gauss_hermite_points, 0.0, 0.0, 0.0, 0.0,
                            float(self.invlink.epsilon), int(self.num_classes))

    @staticmethod
    def _labels(Y):
        Y = ops.to_device(Y)
        if Y.dim() != 2 or Y.shape[1] != 1:
            raise ValueError(f"MultiClass takes the labels as Y [N, 1], got {tuple(Y.shape)}")
        return Y

    def variational_expectations(self, X, Fmu, Fvar, Y):
        return ops.lik_varexp_sum(self._lik_desc(), ops.to_device(Fmu), ops.to_device(Fvar), self._labels(Y))

    def predict_mean_and_var(self, X, Fmu, Fvar):
        return ops.lik_predict_mean_and_var(self._lik_desc(), ops.to_device(Fmu), ops.to_device(Fvar))

    def predict_log_density(self, X, Fmu, Fvar, Y):
        return ops.lik_predict_log_density(self._lik_desc(), ops.to_device(Fmu), ops.to_device(Fvar),
                                           self._labels(Y))


class Normal:
    """The record of tfp.distributions.Normal, the distribution class HeteroskedasticTFPConditional takes: y ~ N(loc,
    scale^2).  The package evaluates it on the device; this class only names it."""

    def __init__(self, loc: Any, scale: Any):
        self.loc, self.scale = loc, scale


class HeteroskedasticTFPConditional(Likelihood):
    """multilatent.py:95-133 with distribution_class=Normal: two latent GPs per row, F = [f, g], and Y [N, 1] ~ N(f,
    scale_transform(g)^2).  scale_transform is Exp or Softplus (gpflow_b200.base), optionally Shifted by a lower bound --
    everything positive(...) returns; None gives positive(base="exp") as in the reference (numpy / math / torch exp are
    taken as Exp).  variational_expectations returns the device fp64 sum [1], predict_mean_and_var two [N, 1] tensors
    (E[y] = mu_f, Var[y] = E[s(g)^2] + v_f) and predict_log_density [N] (the 400-point logspace quadrature)."""

    latent_dim = 2
    observation_dim = 1

    def __init__(self, distribution_class: Any = Normal, scale_transform: Any = None, *, quadrature: Any = None):
        from . import _lib

        if distribution_class is not Normal:
            name = getattr(distribution_class, "__name__", type(distribution_class).__name__)
            raise NotImplementedError(f"HeteroskedasticTFPConditional covers distribution_class=Normal, not {name}")
        _no_custom_quadrature(quadrature)
        if scale_transform is None:
            scale_transform = positive(base="exp")
        base, lower = (scale_transform.base, scale_transform.lower) if isinstance(scale_transform, Shifted) else (
            scale_transform, 0.0)
        if _is_exp(base) or isinstance(base, Exp):
            code = _lib.LIK_SCALE_EXP
        elif isinstance(base, Softplus):
            code = _lib.LIK_SCALE_SOFTPLUS
        else:
            name = getattr(base, "__name__", type(base).__name__)
            raise NotImplementedError(f"HeteroskedasticTFPConditional covers the Exp and Softplus scale transforms "
                                      f"(optionally Shifted), not {name}")
        if not (math.isfinite(lower) and lower >= 0.0):
            raise ValueError(f"the scale transform's lower bound must be finite and >= 0, got {lower}")
        self.distribution_class = distribution_class
        self.scale_transform = scale_transform
        self.num_gauss_hermite_points = DEFAULT_NUM_GAUSS_HERMITE_POINTS
        self._scale_code, self._scale_lower = code, float(lower)

    def _lik_desc(self):
        from . import _lib

        return _lib.LikDesc(_lib.LIK_HETEROSKEDASTIC, self.num_gauss_hermite_points, 0.0, 0.0, 0.0, 0.0, 0.0, 0,
                            self._scale_code, self._scale_lower)

    @staticmethod
    def _check(F, Y=None):
        F = ops.to_device(F)
        if F.dim() != 2 or F.shape[1] != 2:
            raise ValueError(f"HeteroskedasticTFPConditional takes two latents per row, F [N, 2]; got "
                             f"{tuple(F.shape)}")
        if Y is not None:
            Y = ops.to_device(Y)
            if Y.dim() != 2 or Y.shape[1] != 1 or Y.shape[0] != F.shape[0]:
                raise ValueError(f"HeteroskedasticTFPConditional takes the targets as Y [N, 1], got {tuple(Y.shape)}")
        return F, Y

    def variational_expectations(self, X, Fmu, Fvar, Y):
        Fmu, Y = self._check(Fmu, Y)
        return ops.lik_varexp_sum(self._lik_desc(), Fmu, self._check(Fvar)[0], Y)

    def predict_mean_and_var(self, X, Fmu, Fvar):
        return ops.lik_predict_mean_and_var(self._lik_desc(), self._check(Fmu)[0], self._check(Fvar)[0])

    def predict_log_density(self, X, Fmu, Fvar, Y):
        Fmu, Y = self._check(Fmu, Y)
        return ops.lik_predict_log_density(self._lik_desc(), Fmu, self._check(Fvar)[0], Y)
