"""Model base classes (mirrors gpflow/models/model.py:29-343, training_mixins.py:43-147, util.py:31-107)."""
from __future__ import annotations

import abc
from typing import Any, Callable, Dict, Optional, Sequence, Tuple

import numpy as np

from .. import _lib, ops
from ..base import Module
from ..kernels import Kernel, compile_kernel
from ..likelihoods import Likelihood
from ..mean_functions import MeanFunction, Zero


def data_input_to_tensor(data):  # models/util.py:91-107
    return tuple(ops.to_device(d) for d in data)


def centred_targets(mean_function: Optional[MeanFunction], X, Y):
    """Y - m(X): Y itself (no copy) for a Zero or absent mean function, else a new tensor."""
    if mean_function is None or isinstance(mean_function, Zero):
        return Y
    return ops.axpby(-1.0, mean_function(X), 1.0, ops.copy(Y))


def checked_mean_values(likelihood: Likelihood, mean_function: MeanFunction, X, Y, P: int):
    """Checks the targets Y [B, .] against the likelihood for P latent GPs and returns m(X) [B, P] (None for a Zero
    mean): the device entries take Y raw and m(X) apart, which shifts fmean."""
    from ..likelihoods import HeteroskedasticTFPConditional, MultiClass

    lik = likelihood
    if isinstance(lik, MultiClass):
        if Y.shape[1] != 1:
            raise ValueError(f"MultiClass takes the labels as Y [B, 1]; Y has {Y.shape[1]} columns")
        if P != lik.num_classes:
            raise ValueError(f"MultiClass needs one latent GP per class: the model has {P} latent GPs and the "
                             f"likelihood {lik.num_classes} classes")
    elif isinstance(lik, HeteroskedasticTFPConditional):
        if Y.shape[1] != 1:
            raise ValueError(f"HeteroskedasticTFPConditional takes the targets as Y [B, 1]; Y has {Y.shape[1]} "
                             "columns")
        if P != lik.latent_dim:
            raise ValueError(f"HeteroskedasticTFPConditional needs P = 2 outputs (location and scale): the model "
                             f"has {P}")
    elif Y.shape[1] != P:
        raise ValueError(f"Y has {Y.shape[1]} columns but the model has {P} latent GPs")
    if isinstance(mean_function, Zero):
        return None
    mX = ops.to_device(mean_function(X))
    if mX.shape[1] != P:  # one mean column shared by the latents
        mX = mX.expand(X.shape[0], P).contiguous()
    return mX


def likelihood_scalars(likelihood: Likelihood, index: int) -> dict:
    """{the likelihood's Parameter: index}, the slot of its gradient in a fused call's output vector (the Gaussian
    variance, the StudentT scale or the RobustMax epsilon); empty when it has none."""
    from ..base import Parameter
    from ..likelihoods import Gaussian, MultiClass, StudentT

    lik = likelihood
    par = lik.variance if isinstance(lik, Gaussian) else (lik.scale if isinstance(lik, StudentT) else (
        lik.invlink.epsilon if isinstance(lik, MultiClass) else None))
    return {par: index} if isinstance(par, Parameter) else {}


class BayesianModel(Module, metaclass=abc.ABCMeta):
    def log_prior_density(self) -> float:  # model.py:47-60 (priors are outside the hot path)
        if any(p.prior is not None for p in self.parameters):
            raise NotImplementedError("parameter priors are outside the hot path")
        return 0.0

    def log_posterior_density(self, *args: Any, **kwargs: Any):
        return self.maximum_log_likelihood_objective(*args, **kwargs)

    def _training_loss(self, *args: Any, **kwargs: Any):  # model.py:71-76
        obj = self.maximum_log_likelihood_objective(*args, **kwargs)
        out = ops.copy(obj)
        return ops.axpby(-1.0, obj, 0.0, out)

    @abc.abstractmethod
    def maximum_log_likelihood_objective(self, *args: Any, **kwargs: Any):
        raise NotImplementedError


class GPModel(BayesianModel):
    def __init__(self, kernel: Kernel, likelihood: Likelihood, mean_function: Optional[MeanFunction] = None,
                 num_latent_gps: Optional[int] = None) -> None:
        assert num_latent_gps is not None, "GPModel requires specification of num_latent_gps"
        self.num_latent_gps = num_latent_gps
        self.mean_function = mean_function if mean_function is not None else Zero(output_dim=num_latent_gps)
        self.kernel = kernel
        self.likelihood = likelihood

    @staticmethod
    def calc_num_latent_gps_from_data(data, kernel: Kernel, likelihood: Likelihood) -> int:  # model.py:146-160
        _, Y = data
        return Y.shape[-1]

    @abc.abstractmethod
    def predict_f(self, Xnew, full_cov: bool = False, full_output_cov: bool = False):
        raise NotImplementedError

    def predict_f_samples(self, Xnew, num_samples: Optional[int] = None, full_cov: bool = True,
                          full_output_cov: bool = False, *, eps=None, generator=None):
        """model.py:232-288: samples of the posterior latent function(s) at Xnew, [N, P] or [S, N, P].  `eps` injects the
        standard-normal draws (shapes of conditionals.sample_mvn)."""
        from ..conditionals import sample_mvn

        if full_cov and full_output_cov:
            raise NotImplementedError("The combination of both `full_cov` and `full_output_cov` is not supported.")
        Xnew = ops.to_device(Xnew)
        mean, cov = self.predict_f(Xnew, full_cov=full_cov, full_output_cov=full_output_cov)
        if full_cov:                                                       # model.py:273-279
            samples = sample_mvn(ops.transpose(mean), cov, True, num_samples, eps=eps, generator=generator)  # [(S), P, N]
            if num_samples is None:
                return ops.transpose(samples)
            out = ops.empty((samples.shape[0], samples.shape[2], samples.shape[1]), like=samples)
            for s_ in range(samples.shape[0]):
                ops.transpose(samples[s_], out=out[s_])
            return out
        return sample_mvn(mean, cov, full_output_cov, num_samples, eps=eps, generator=generator)       # model.py:281-284

    def predict_y(self, Xnew, full_cov: bool = False, full_output_cov: bool = False):  # model.py:290-325
        if full_cov or full_output_cov:
            raise NotImplementedError("The predict_y method currently supports only the argument values "
                                      "full_cov=False and full_output_cov=False")
        Xnew = ops.to_device(Xnew)
        f_mean, f_var = self.predict_f(Xnew, full_cov=full_cov, full_output_cov=full_output_cov)
        return self.likelihood.predict_mean_and_var(Xnew, f_mean, f_var)

    def predict_log_density(self, data, full_cov: bool = False, full_output_cov: bool = False):  # :332-343
        if full_cov or full_output_cov:
            raise NotImplementedError("The predict_log_density method currently supports only the argument values "
                                      "full_cov=False and full_output_cov=False")
        X, Y = data
        X = ops.to_device(X)
        f_mean, f_var = self.predict_f(X, full_cov=full_cov, full_output_cov=full_output_cov)
        return self.likelihood.predict_log_density(X, f_mean, f_var, Y)


class LossClosure:
    """What `training_loss_closure()` returns: calling it evaluates the loss (as in the reference); models with a device
    backward pass also give the optimiser `value_and_gradients(variables)` -> (loss, [d loss / d unconstrained variable])
    in the order of `variables` (the pair gpflow/optimizers/scipy.py:300-316 obtains from a GradientTape).  For a model
    trained on external data, `batch()` supplies the data of one evaluation: `value_and_gradients` draws one batch and
    returns the loss and gradients of that same batch."""

    def __init__(self, model, loss_fn: Callable[[], Any], batch: Optional[Callable[[], Any]] = None):
        self._model, self._loss_fn, self._batch = model, loss_fn, batch
        if hasattr(model, "training_loss_and_gradients"):
            self.value_and_gradients = self._value_and_gradients

    def __call__(self):
        return self._loss_fn()

    def _value_and_gradients(self, variables=None):
        args = () if self._batch is None else (self._batch(),)
        loss, grads = self._model.training_loss_and_gradients(*args)
        params = self._model.trainable_parameters
        if variables is None:
            return loss, grads
        by_id = {id(p): g for p, g in zip(params, grads)}
        missing = [v for v in variables if id(v) not in by_id]
        if missing:
            raise ValueError("a variable passed to the optimiser is not a trainable parameter of the model")
        return loss, [by_id[id(v)] for v in variables]


class DeviceGradientMixin:
    """The optimiser's side of a model with a fused value + gradient call.  The model supplies `_objective_and_grad()`
    -> (objective, {Parameter: d objective / d constrained value}); a model trained on external data takes the batch
    as its argument (`_objective_and_grad(data)`)."""

    def _refuse_device_gradient(self, X) -> None:
        lik = self.likelihood
        # a likelihood without a noise variance (Bernoulli, Poisson, StudentT) has nothing heteroskedastic to refuse
        if getattr(lik, "heteroskedastic", False) or (hasattr(lik, "variance") and lik.variance is None):
            raise NotImplementedError("the device backward pass covers Gaussian(variance=...) with a constant variance")
        if ops.dtype_code(X) != _lib.GPK_F64:
            raise NotImplementedError("the device backward pass computes in float64")

    def _mean_gradients(self, ws, off: int, X, N: int, P: int):
        """[(Parameter, device gradient)] of a Constant / Linear mean function from d objective / d m [N, P], which the
        fused call leaves at byte `off` of its workspace `ws`, through mean_functions.gradients_from_adjoint; [] for
        other mean functions."""
        from .. import mean_functions as mf

        if not isinstance(self.mean_function, (mf.Constant, mf.Linear)):
            return []
        adjoint = ws[off:off + 8 * N * P].view(ops.torch().float64).view(N, P)
        return mf.gradients_from_adjoint(self.mean_function, X, adjoint)

    def _device_value_and_grad(self, X, P: int, *, layout: Callable[[], Tuple[int, int]], n_head: int, info_index: int,
                               scalars: Dict[Any, int], arrays: Sequence[Any], call: Callable[..., int], entry: str,
                               device_arrays: bool = False, kernels: Optional[Sequence[Kernel]] = None,
                               describe_info: Optional[Callable[[int], str]] = None):
        """One fused value + gradient call on the inputs X [N, D] with P outputs per row, and the steps every model
        shares around it: the refusals, the workspace, the output vector [n_head + leaf slots], one device array per
        Parameter of `arrays` for its gradient, the mean-function gradients, one host read, the Cholesky info check and
        the gradient dict.  With `device_arrays` the gradients of `arrays` stay the device tensors the call wrote (fp64,
        the parameters' shapes) instead of host copies: the device optimisers (NaturalGradient, Adam) consume them there.  The model
        supplies
          layout()  -> (workspace bytes, byte offset of d objective / d m(X) [N, P] in the workspace),
          scalars   {Parameter: index of its gradient in the output vector},
          call(kernel, out, n_out, array_grads, ws) -> status, `kernel` the compiled expression (nodes, n_nodes, dims,
                    ard) and `array_grads` the device arrays in the order of `arrays`.
        `kernels` (default: the model's kernel alone) lists the latent expressions of a multi-output model: `call` then
        gets the list of their compiled expressions, the output vector holds their slot ranges one after another, and a
        Parameter that appears in several ranges collects the sum.
        `describe_info(info)` names the failed factorisation of a non-zero out[info_index] in the error (default: the
        pivot).
        Returns (objective, {Parameter: d objective / d constrained value}), the objective out[0] checked against
        out[info_index]."""
        from ..kernels import gradient_slots, slot_gradients

        lib = _lib.load()
        N, D = X.shape
        exprs = [self.kernel] if kernels is None else list(kernels)
        slots = [gradient_slots(k, D) for k in exprs]  # NotImplementedError for materialised kernels
        self._refuse_device_gradient(X)
        need, dm_off = layout()
        if getattr(self, "_gws", None) is None or self._gws.numel() < need or self._gws.device != X.device:
            self._gws = ops.scratch_bytes(need)
        compiled = [compile_kernel(k, D) for k in exprs]
        offsets = [0]
        for c in compiled:
            n_slots = lib.gpk_gpr_lml_grad_slots(*c, D)
            _lib.check(min(n_slots, 0), "gpk_gpr_lml_grad_slots")
            offsets.append(offsets[-1] + n_slots)
        n_out = n_head + offsets[-1]
        T = ops.torch()
        out = T.empty((n_out,), dtype=T.float64, device=X.device)
        array_grads = [T.empty(tuple(p.shape), dtype=T.float64, device=X.device) for p in arrays]
        _lib.check(call(compiled[0] if kernels is None else compiled, out, n_out, array_grads, self._gws), entry)
        mean_dev = self._mean_gradients(self._gws, dm_off, X, N, P)
        h = out.cpu().numpy()
        if int(h[info_index]) != 0:
            where = f"pivot {int(h[info_index])}" if describe_info is None else describe_info(int(h[info_index]))
            raise ops.NonPositiveDefiniteError(f"Cholesky decomposition was not successful ({where} <= 0)")
        grads = {p: np.asarray(h[i]) for p, i in scalars.items()}
        for sl, o0, o1 in zip(slots, offsets[:-1], offsets[1:]):
            for p, g in slot_gradients(sl, h[n_head + o0:n_head + o1]).items():
                grads[p] = grads[p] + g if p in grads else g
        for p, g in zip(arrays, array_grads):
            grads[p] = g if device_arrays else g.cpu().numpy()
        for p, g in mean_dev:
            grads[p] = g.cpu().numpy().reshape(p.shape)
        return ops.objective(out, 0, info_index), grads

    def training_loss_and_gradients(self, *args):
        """(loss, gradients) for the optimiser contract of gpflow/optimizers/scipy.py:322-331: loss = -objective (float)
        and one gradient per TRAINABLE parameter w.r.t. its UNCONSTRAINED variable, in `trainable_parameters` order.
        `args` (the data batch of an external-data model) pass through to `_objective_and_grad`."""
        if any(p.prior is not None for p in self.trainable_parameters):
            raise NotImplementedError("parameter priors are outside the hot path: the device gradient covers the "
                                      "likelihood only")
        objective, grads = self._objective_and_grad(*args)
        out = []
        for p in self.trainable_parameters:
            if p not in grads:
                raise NotImplementedError("a trainable parameter has no device gradient (mean functions other than "
                                          "Constant / Linear, and data gradients, are outside the hot path)")
            out.append(-p.unconstrained_gradient(grads[p]))
        return -float(objective), out


class InternalDataTrainingLossMixin:
    """training_mixins.py:43-78."""

    def training_loss(self):
        return self._training_loss()

    def training_loss_closure(self, *, compile: bool = True) -> Callable[[], Any]:
        return LossClosure(self, self.training_loss)


class ExternalDataTrainingLossMixin:
    """training_mixins.py:81-147."""

    def training_loss(self, data):
        return self._training_loss(data)

    def training_loss_closure(self, data, *, compile: bool = True) -> Callable[[], Any]:
        """A LossClosure bound to `data`: a fixed (X, Y), or an iterator from which every evaluation draws the next
        batch."""
        if hasattr(data, "__next__"):
            it = data

            def batch():
                return next(it)
        else:
            def batch():
                return data

        return LossClosure(self, lambda: self._training_loss(batch()), batch)


def loss_model_and_batch(loss_fn, who: str) -> Tuple[Any, Optional[Callable[[], Any]]]:
    """(model, batch) behind the loss an optimiser's one-step `minimize` was given: a LossClosure (`batch()` draws the
    data of one evaluation) or the bound `training_loss` of an internal-data model (batch None).  A step evaluates
    `model._objective_and_grad(*(() if batch is None else (batch(),)))` once, so an iterator closure advances by exactly
    one batch.  Anything else is a ValueError naming `who`."""
    if isinstance(loss_fn, LossClosure):
        return loss_fn._model, loss_fn._batch
    model = getattr(loss_fn, "__self__", None)
    if not (isinstance(model, InternalDataTrainingLossMixin)
            and getattr(loss_fn, "__func__", None) is type(model).training_loss):
        raise ValueError(f"{who} takes a closure from training_loss_closure(...) or the bound training_loss of an "
                         "internal-data model (VGP)")
    return model, None
