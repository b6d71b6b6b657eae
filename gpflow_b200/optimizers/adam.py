"""Adam on the device (mirrors tf_keras.optimizers.Adam as the reference uses it: the default optimiser of
gpflow/utilities/misc.py:76-109 `training_loop`, and the `adam.minimize(loss, model.trainable_variables)` of the SVGP
minibatch loops).

Keras updates the UNCONSTRAINED variable of each parameter.  Here the parameters whose gradient the model's device
backward pass leaves on the GPU (Z, q_mu, q_sqrt) are updated there, all in ONE launch of `gpk_adam_step`
(csrc/adam.cu), in place in their device mirrors; their gradients and moment estimates never reach the host, and the
host copy of the value is fetched only if someone asks for it (base.Parameter.device_updated).  The small parameters
(kernel hyperparameters, the likelihood parameter, Constant / Linear mean functions) reach the kernels as launch
arguments and their gradients arrive in the one small host read every gradient call makes; they take the same
formulas in NumPy."""
from __future__ import annotations

from typing import Any, Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from .. import _lib, ops
from ..base import Exp, FillTriangular, Parameter, Shifted, Softplus

__all__ = ["Adam"]


def _transform_code(p: Parameter) -> Tuple[int, float]:
    """(GPK_ADAM_* code, lower bound) of the parameter's bijector."""
    t, lower = p.transform, 0.0
    if t is None or isinstance(t, FillTriangular):
        return _lib.GPK_ADAM_IDENTITY, 0.0
    if isinstance(t, Shifted):
        t, lower = t.base, t.lower
    if type(t) is Softplus:
        return _lib.GPK_ADAM_SOFTPLUS, lower
    if type(t) is Exp:
        return _lib.GPK_ADAM_EXP, lower
    raise NotImplementedError(f"{type(p.transform).__name__}: the device Adam step covers the identity, Softplus and "
                              "Exp bijectors with a lower bound")


class Adam:
    """tf_keras.optimizers.Adam(learning_rate, beta_1, beta_2, epsilon): `minimize` and `apply_gradients` take ONE step
    per call and `iterations` counts them.  Moment estimates are kept per Parameter, created at its first step, on the
    device for the parameters stepped there."""

    def __init__(self, learning_rate: float = 0.001, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-07,
                 amsgrad: bool = False, name: Optional[str] = None) -> None:
        if amsgrad:
            raise NotImplementedError("Adam: amsgrad=True is not implemented")
        if callable(learning_rate) or not np.isscalar(learning_rate):
            raise NotImplementedError("Adam: learning-rate schedules are not implemented; pass a number")
        self.learning_rate, self.beta_1, self.beta_2 = float(learning_rate), float(beta_1), float(beta_2)
        self.epsilon = float(epsilon)
        if not (np.isfinite(self.learning_rate) and self.learning_rate >= 0.0):
            raise ValueError(f"Adam: learning_rate must be non-negative and finite, got {learning_rate}")
        if not (0.0 <= self.beta_1 < 1.0 and 0.0 <= self.beta_2 < 1.0):
            raise ValueError("Adam: beta_1 and beta_2 must lie in [0, 1)")
        if not self.epsilon > 0.0:
            raise ValueError("Adam: epsilon must be positive")
        self.name = self.__class__.__name__ if name is None else name
        self.iterations = 0
        self._moments: Dict[Parameter, Tuple[Any, Any]] = {}

    def minimize(self, loss: Callable[[], Any], var_list: Sequence[Parameter]) -> None:
        """One Adam step on the variables of `var_list` from ONE evaluation of the model's fused value and gradient (an
        iterator closure draws exactly one batch).  `loss` is a closure from `training_loss_closure(...)` or the bound
        `training_loss` of an internal-data model.  Variables that are not trainable, and parameters outside
        `var_list`, are left alone.  Priors, float32 parameters and variables that are not the model's are refused
        before a batch is drawn; a variable for which the model has no device gradient is refused after the evaluation
        and before anything is changed."""
        from ..models.model import loss_model_and_batch

        model, batch = loss_model_and_batch(loss, "Adam.minimize")
        if not hasattr(model, "_objective_and_grad"):
            raise NotImplementedError(f"{type(model).__name__} has no device gradient for an Adam step")
        variables = self._trainable(var_list)
        if any(p.prior is not None for p in model.trainable_parameters):
            raise NotImplementedError("parameter priors are outside the hot path: the device gradient covers the "
                                      "likelihood only")
        known = set(model.parameters)
        if any(p not in known for p in variables):
            raise ValueError("a variable passed to the optimiser is not a parameter of the model")
        _, grads = model._objective_and_grad(*(() if batch is None else (batch(),)), device_arrays=True)
        if any(p not in grads for p in variables):
            raise NotImplementedError("a trainable parameter has no device gradient (mean functions other than "
                                      "Constant / Linear, and data gradients, are outside the hot path)")
        on_device = [(p, grads[p]) for p in variables if hasattr(grads[p], "data_ptr")]
        # the model's gradients are those of the objective w.r.t. the constrained values: sign -1 on the device, and
        # the chain rule through the bijector on the host
        on_host = [(p, -p.unconstrained_gradient(grads[p])) for p in variables if not hasattr(grads[p], "data_ptr")]
        self._step(on_device, -1.0, on_host)

    def apply_gradients(self, grads_and_vars: Iterable[Tuple[Any, Parameter]]) -> None:
        """One Adam step from gradients of the LOSS w.r.t. the UNCONSTRAINED variables (what
        `closure.value_and_gradients(variables)` returns), NumPy arrays or device tensors.  A device gradient of a
        parameter without a constraining bijector (Z, q_mu, a dense q_sqrt) is consumed on the device; every other
        gradient takes the NumPy formulas."""
        pairs = [(g, p) for g, p in grads_and_vars]
        variables = self._trainable([p for _, p in pairs])
        on_device, on_host = [], []
        for g, p in pairs:
            if p not in variables:
                continue
            if hasattr(g, "data_ptr") and g.is_cuda and _transform_code(p)[0] == _lib.GPK_ADAM_IDENTITY:
                on_device.append((p, g))
            else:
                g = g.detach().cpu().numpy() if hasattr(g, "detach") else g
                on_host.append((p, np.asarray(g, dtype=np.float64).reshape(p.shape)))
        self._step(on_device, 1.0, on_host)

    @staticmethod
    def _trainable(var_list: Sequence[Parameter]) -> List[Parameter]:
        var_list = list(var_list)
        if not all(isinstance(p, Parameter) for p in var_list):
            raise TypeError("Adam: var_list is expected to only contain Parameter instances")
        if len(set(var_list)) != len(var_list):
            raise ValueError("Adam: a variable is listed twice")
        variables = [p for p in var_list if p.trainable]
        if any(p.dtype != np.float64 for p in variables):
            raise NotImplementedError("the device backward pass computes in float64")
        return variables

    def _step(self, on_device: List[Tuple[Parameter, Any]], sign: float,
              on_host: List[Tuple[Parameter, np.ndarray]]) -> None:
        """`on_device`: (parameter, device gradient w.r.t. its CONSTRAINED value, of sign * loss); `on_host`:
        (parameter, NumPy gradient of the loss w.r.t. its UNCONSTRAINED variable)."""
        t = self.iterations + 1
        lr_t = self.learning_rate * np.sqrt(1.0 - self.beta_2 ** t) / (1.0 - self.beta_1 ** t)
        if on_device:
            self._device_step(on_device, sign, lr_t)
        for p, g in on_host:
            m, v = self._state(p, None)
            m += (1.0 - self.beta_1) * (g - m)
            v += (1.0 - self.beta_2) * (g * g - v)
            p.assign_unconstrained(p.unconstrained_variable - lr_t * m / (np.sqrt(v) + self.epsilon))
        self.iterations = t

    def _state(self, p: Parameter, mirror: Any) -> Tuple[Any, Any]:
        """(m, v) of `p`: zeros at its first step; float64 tensors beside the device `mirror`, or NumPy arrays when
        `mirror` is None.  A parameter that changes sides between steps takes its moments along."""
        T = ops.torch()
        state = self._moments.get(p)
        if mirror is None:
            if state is None:
                state = (np.zeros(p.shape), np.zeros(p.shape))
            elif hasattr(state[0], "data_ptr"):
                state = tuple(s.cpu().numpy() for s in state)
        elif state is None:
            state = (T.zeros_like(mirror), T.zeros_like(mirror))
        elif not hasattr(state[0], "data_ptr") or state[0].device != mirror.device:
            state = tuple(T.as_tensor(s).to(mirror.device).contiguous() for s in state)
        self._moments[p] = state
        return state

    def _device_step(self, items: List[Tuple[Parameter, Any]], sign: float, lr_t: float) -> None:
        lib = _lib.load()
        T = ops.torch()
        dev = ops.require_cuda()
        segs, mirrors = [], []
        for p, g in items:
            value = p.device(dev)
            if g.dtype != T.float64 or g.device != value.device or g.numel() != value.numel():
                raise ValueError("Adam: a device gradient must be a float64 tensor of the parameter's size on its device")
            g = g.contiguous()
            state = self._state(p, value)
            code, lower = _transform_code(p)
            segs.append(_lib.AdamSeg(value.data_ptr(), g.data_ptr(), state[0].data_ptr(), state[1].data_ptr(),
                                     value.numel(), code, lower))
            mirrors.append((p, value))
        for k in range(0, len(segs), _lib.GPK_ADAM_MAX_SEGS):
            part = segs[k:k + _lib.GPK_ADAM_MAX_SEGS]
            _lib.check(lib.gpk_adam_step((_lib.AdamSeg * len(part))(*part), len(part), lr_t, self.beta_1, self.beta_2,
                                         self.epsilon, sign, _lib.GPK_F64, ops._stream()), "gpk_adam_step")
        for p, value in mirrors:
            p.device_updated(value)
