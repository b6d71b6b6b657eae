"""Natural-gradient optimiser for the variational parameters (mirrors gpflow/optimizers/natgrad.py:43-367).

The reference takes steps in the natural parameters of q(u) = N(q_mu, q_sqrt q_sqrt^T) (Salimbeni et al., 2018): it
converts (q_mu, q_sqrt) to the expectation and natural parameters with TensorFlow ops and differentiates through the
conversions.  Here one fused device call, `gpk_natgrad_step` (csrc/natgrad.cu), applies the step of each latent GP from
the gradients the model's device backward pass returns, without forming Sig^-1 or a second Cholesky (include/gpk.h gives
the algebra).  q_mu, q_sqrt and their gradients never leave the device; the host values are refreshed with one
device-to-host copy per parameter."""
from __future__ import annotations

import ctypes
from typing import Any, Callable, Optional, Sequence, Tuple

import numpy as np

from .. import _lib, ops
from ..base import Parameter

__all__ = ["NaturalGradient", "XiNat", "XiSqrtMeanVar", "XiTransform"]


class XiTransform:
    """The parameterisation xi in which the natural-gradient step is taken (natgrad.py:43-98).  The device step covers
    the two transforms of the reference, XiNat and XiSqrtMeanVar; a user-defined transform has no device step."""

    _code: Optional[int] = None


class XiNat(XiTransform):
    """xi = the natural parameters (natgrad.py:101-136), the default: with a Gaussian likelihood one step of size 1
    reaches the optimal q."""

    _code = _lib.GPK_XI_NAT


class XiSqrtMeanVar(XiTransform):
    """xi = (q_mu, q_sqrt) themselves (natgrad.py:139-173): the natural gradient applied in the model's own
    parameterisation."""

    _code = _lib.GPK_XI_SQRT_MEAN_VAR


def _xi_code(xi: XiTransform) -> int:
    if type(xi) not in (XiNat, XiSqrtMeanVar):
        raise NotImplementedError(f"{type(xi).__name__}: the natural-gradient step covers XiNat and XiSqrtMeanVar; "
                                  "other xi transforms need autodiff through their conversions")
    return xi._code


class NaturalGradient:
    """natgrad.py:176-367: natural-gradient steps on (q_mu, q_sqrt) pairs of an SVGP (q_diag=False) or VGP.  Its only
    public method is `minimize(loss_fn, var_list)`, one step per call.  The usual setup makes q_mu and q_sqrt
    untrainable, so that another optimiser over the model's trainable parameters leaves them alone; the step takes
    their gradients either way."""

    def __init__(self, gamma: float, xi_transform: XiTransform = XiNat(), name: Optional[str] = None) -> None:
        gamma = float(gamma)
        if not (gamma > 0.0 and np.isfinite(gamma)):
            raise ValueError(f"NaturalGradient: gamma must be positive and finite, got {gamma}")
        _xi_code(xi_transform)
        self.name = self.__class__.__name__ if name is None else name
        self.gamma = gamma
        self.xi_transform = xi_transform
        self._ws = None

    def minimize(self, loss_fn: Callable[[], Any], var_list: Sequence[Tuple]) -> None:
        """One natural-gradient step on every (q_mu, q_sqrt) or (q_mu, q_sqrt, xi_transform) of `var_list`
        (natgrad.py:213-238), all from ONE evaluation of the model's fused value and gradient: an iterator closure
        draws exactly one batch.  `loss_fn` is a closure from `training_loss_closure(...)` or the bound `training_loss`
        of an internal-data model (VGP).  A step whose factorisation fails raises ops.NonPositiveDefiniteError and
        leaves q_mu and q_sqrt unchanged."""
        model, batch = self._model_and_batch(loss_fn)
        params = self._check_pairs(model, var_list)   # before the batch is drawn: a refused call consumes none
        _, grads = model._objective_and_grad(*(() if batch is None else (batch(),)), device_arrays=True)
        for q_mu, q_sqrt, xi in params:
            self._natgrad_apply_gradients(grads[q_mu], grads[q_sqrt], q_mu, q_sqrt, xi)

    @staticmethod
    def _model_and_batch(loss_fn) -> Tuple[Any, Optional[Callable[[], Any]]]:
        from ..models.model import InternalDataTrainingLossMixin, LossClosure

        if isinstance(loss_fn, LossClosure):
            model, batch = loss_fn._model, loss_fn._batch
        else:
            model = getattr(loss_fn, "__self__", None)
            if not (isinstance(model, InternalDataTrainingLossMixin)
                    and getattr(loss_fn, "__func__", None) is type(model).training_loss):
                raise ValueError("NaturalGradient.minimize takes a closure from training_loss_closure(...) or the bound "
                                 "training_loss of an internal-data model (VGP)")
            batch = None
        if not (hasattr(model, "_objective_and_grad") and hasattr(model, "q_mu") and hasattr(model, "q_sqrt")):
            raise NotImplementedError(f"{type(model).__name__} has no variational (q_mu, q_sqrt) with a device gradient "
                                      "for a natural-gradient step (SVGP and VGP have)")
        return model, batch

    def _check_pairs(self, model, var_list: Sequence[Tuple]):
        if not var_list:
            raise ValueError("NaturalGradient: var_list is empty; it holds the model's (q_mu, q_sqrt)")
        params = []
        for v in var_list:
            if len(v) not in (2, 3):
                raise ValueError("var_list holds (q_mu, q_sqrt) or (q_mu, q_sqrt, xi_transform) tuples")
            q_mu, q_sqrt = v[0], v[1]
            xi = v[2] if len(v) > 2 and v[2] is not None else self.xi_transform
            _xi_code(xi)
            if q_mu is not getattr(model, "q_mu", None) or q_sqrt is not getattr(model, "q_sqrt", None):
                raise ValueError("NaturalGradient: each pair must be the (q_mu, q_sqrt) of the loss function's model")
            if any(q is q_mu for q, _, _ in params):
                raise ValueError("NaturalGradient: a (q_mu, q_sqrt) pair is listed twice")
            if getattr(model, "q_diag", False):
                raise NotImplementedError("natural gradients need a full q_sqrt [P, M, M]; q_diag=True is not supported")
            if q_mu.prior is not None or q_sqrt.prior is not None:
                raise NotImplementedError("NaturalGradient: a prior on q_mu or q_sqrt is outside the device step")
            if q_mu.dtype != np.float64 or q_sqrt.dtype != np.float64:
                raise NotImplementedError("the natural-gradient step computes in float64")
            params.append((q_mu, q_sqrt, xi))
        return params

    def _natgrad_apply_gradients(self, q_mu_grad, q_sqrt_grad, q_mu: Parameter, q_sqrt: Parameter,
                                 xi_transform: Optional[XiTransform] = None) -> None:
        """natgrad.py:280-367 on the device.  q_mu_grad [M, P] and q_sqrt_grad [P, M, M] are device fp64 tensors of the
        gradients of the ELBO (not the loss) w.r.t. the constrained q_mu and q_sqrt, as the model's device backward
        pass returns them.  q_sqrt may hold negative diagonal entries: XiNat follows the chain rule through q_sqrt and
        returns the factor with a positive diagonal, where the reference would treat the gradient as one at
        chol(q_sqrt q_sqrt^T); the two agree whenever diag(q_sqrt) > 0 (include/gpk.h)."""
        xi = _xi_code(self.xi_transform if xi_transform is None else xi_transform)
        lib = _lib.load()
        T = ops.torch()
        m, S = ops.to_device(q_mu), ops.to_device(q_sqrt)
        M, P = m.shape
        need = lib.gpk_natgrad_step_ws(M, P, xi, _lib.GPK_F64)
        if self._ws is None or self._ws.numel() < need or self._ws.device != m.device:
            self._ws = ops.scratch_bytes(need)
        m_out, S_out = T.empty_like(m), T.empty_like(S)
        info = T.empty((P,), dtype=T.int32, device=m.device)
        _lib.check(lib.gpk_natgrad_step(xi, M, P, ops._p(m), ops._p(S), ops._p(q_mu_grad.contiguous()),
                                        ops._p(q_sqrt_grad.contiguous()), self.gamma, _lib.GPK_F64, ops._p(m_out),
                                        ops._p(S_out), ops._p(info), ops._p(self._ws), ops._stream()),
                   "gpk_natgrad_step")
        bad = [(p, int(k)) for p, k in enumerate(info.cpu().numpy()) if k != 0]
        if bad:
            p, k = bad[0]
            why = (f"q_sqrt[{p}] has a zero diagonal entry at {-k - 1}" if k < 0 else
                   f"latent {p}: the natural-gradient step is too long for the current q (pivot {k} <= 0 in the "
                   "Cholesky of I - 2 gamma H)")
            raise ops.NonPositiveDefiniteError(f"Cholesky decomposition was not successful: {why}")
        q_mu.assign_device(m_out)
        q_sqrt.assign_device(S_out)
