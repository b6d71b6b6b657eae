"""Parameter / Module scaffolding (mirrors gpflow/base.py:73-280, utilities/bijectors.py:27-52).

The forward value of a Parameter is its *constrained* value (gpflow/base.py:118-280); the
unconstrained value and the bijector are kept so optimiser drivers can be layered on later.
Values live on the host as NumPy arrays; large parameters (q_mu, q_sqrt, Z) are mirrored to the
device lazily and the mirror is invalidated by `assign`."""
from __future__ import annotations

from typing import Any, Dict, Iterator, Optional, Tuple

import numpy as np

from . import config


class Transform:
    """Bijector from unconstrained to constrained space."""

    def forward(self, x: np.ndarray) -> np.ndarray:
        return x

    def inverse(self, y: np.ndarray) -> np.ndarray:
        return y

    def forward_grad(self, x: np.ndarray) -> np.ndarray:
        """d forward(x) / dx, elementwise (chain rule from constrained to unconstrained gradients,
        what tf autodiff applies through the bijector; gpflow/base.py:118-280)."""
        return np.ones_like(np.asarray(x, dtype=np.float64))


class Softplus(Transform):
    def forward(self, x):
        return np.logaddexp(0.0, x)

    def inverse(self, y):
        y = np.asarray(y, dtype=np.float64)
        return y + np.log(-np.expm1(-y))

    def forward_grad(self, x):
        x = np.asarray(x, dtype=np.float64)
        return 1.0 / (1.0 + np.exp(-x))


class Exp(Transform):
    def forward(self, x):
        return np.exp(x)

    def inverse(self, y):
        return np.log(y)

    def forward_grad(self, x):
        return np.exp(np.asarray(x, dtype=np.float64))


class Sigmoid(Transform):
    """tfp.bijectors.Sigmoid(): the open interval (0, 1)."""

    def forward(self, x):
        x = np.asarray(x, dtype=np.float64)
        return np.exp(-np.logaddexp(0.0, -x))

    def inverse(self, y):
        y = np.asarray(y, dtype=np.float64)
        return np.log(y) - np.log1p(-y)

    def forward_grad(self, x):
        s = self.forward(x)
        return s * (1.0 - s)


class Shifted(Transform):
    """Chain([Shift(lower), base]) of gpflow/utilities/bijectors.py:41-44."""

    def __init__(self, base: Transform, lower: float):
        self.base, self.lower = base, float(lower)

    def forward(self, x):
        return self.base.forward(x) + self.lower

    def inverse(self, y):
        return self.base.inverse(np.asarray(y) - self.lower)

    def forward_grad(self, x):
        return self.base.forward_grad(x)


class FillTriangular(Transform):
    """triangular(): the constrained value is a (batch of) lower-triangular matrices; the forward
    value keeps whatever was assigned — consumers apply band_part(-1, 0) themselves
    (gpflow/conditionals/util.py:151, kullback_leiblers.py:120)."""


def positive(lower: Optional[float] = None, base: Optional[str] = None) -> Transform:
    name = (base if base is not None else config.default_positive_bijector()).lower()
    t: Transform = {"softplus": Softplus, "exp": Exp}[name]()
    lower_bound = lower if lower is not None else config.default_positive_minimum()
    if lower_bound != 0.0:
        t = Shifted(t, lower_bound)
    return t


def triangular() -> Transform:
    return FillTriangular()


class Parameter:
    def __init__(self, value: Any, *, transform: Optional[Transform] = None, prior: Any = None,
                 trainable: bool = True, dtype: Optional[type] = None, name: Optional[str] = None):
        if isinstance(value, Parameter):
            transform = transform or value.transform
            value = value.numpy()
        if hasattr(value, "detach"):  # torch tensor
            value = value.detach().cpu().numpy()
        self._dtype = np.dtype(dtype if dtype is not None else config.default_float())
        self.transform = transform
        self.prior = prior
        self.trainable = trainable
        self.name = name
        self._value = np.array(value, dtype=self._dtype)
        self._device_cache: Dict[Tuple[str, str], Any] = {}
        self._validate()

    def _validate(self) -> None:
        if isinstance(self.transform, (Softplus, Exp)) and np.any(self._value <= 0):
            raise ValueError("positive Parameter initialised with a non-positive value")
        if isinstance(self.transform, Shifted) and np.any(self._value <= self.transform.lower):
            raise ValueError(f"Parameter value must be greater than its lower bound {self.transform.lower}")
        if isinstance(self.transform, Sigmoid) and not np.all((self._value > 0) & (self._value < 1)):
            raise ValueError("a Sigmoid Parameter must lie in the open interval (0, 1)")

    @property
    def shape(self) -> Tuple[int, ...]:
        return self._value.shape

    @property
    def dtype(self) -> np.dtype:
        return self._dtype

    def numpy(self) -> np.ndarray:
        return self._value

    @property
    def unconstrained_variable(self) -> np.ndarray:
        return self._value if self.transform is None else self.transform.inverse(self._value)

    def assign_unconstrained(self, u: Any) -> None:
        """Sets the parameter from its unconstrained value (what an optimiser updates; gpflow/base.py:196-211)."""
        u = np.asarray(u, dtype=np.float64).reshape(self._value.shape)
        self.assign(u if self.transform is None else self.transform.forward(u))

    def unconstrained_gradient(self, g_constrained: Any) -> np.ndarray:
        """Chain rule: gradient w.r.t. the unconstrained variable from the gradient w.r.t. the constrained value."""
        g = np.asarray(g_constrained, dtype=np.float64).reshape(self._value.shape)
        if self.transform is None:
            return g
        return g * self.transform.forward_grad(self.unconstrained_variable)

    def assign(self, value: Any) -> None:
        if hasattr(value, "detach"):
            value = value.detach().cpu().numpy()
        new = np.array(value, dtype=self._dtype)
        if new.shape != self._value.shape:
            new = np.broadcast_to(new, self._value.shape).copy()
        self._value = new
        self._device_cache.clear()
        self._validate()

    def assign_device(self, t: Any) -> None:
        """Sets the value from the contiguous device tensor `t` (the parameter's shape and dtype) and keeps `t` itself
        as the device mirror, so the next evaluation reads it without an upload.  The host value is refreshed with one
        device-to-host copy.  `t` must not be written afterwards by anyone else."""
        host = t.detach().cpu().numpy()
        if host.shape != self._value.shape or host.dtype != self._dtype or not t.is_contiguous():
            raise ValueError(f"assign_device needs a contiguous {self._dtype.name} tensor of shape {self._value.shape}")
        old = self._value
        self._value = host
        try:
            self._validate()
        except ValueError:
            self._value = old
            raise
        self._device_cache.clear()
        self._device_cache[(str(t.device), self._dtype.name)] = t

    def device(self, device: Any, dtype: Optional[type] = None):
        """Contiguous device mirror (torch tensor used as a container only)."""
        import torch

        dt = np.dtype(dtype if dtype is not None else self._dtype)
        key = (str(device), dt.name)
        t = self._device_cache.get(key)
        if t is None:
            t = torch.from_numpy(np.ascontiguousarray(self._value.astype(dt))).to(device)
            self._device_cache[key] = t
        return t

    def __float__(self) -> float:
        return float(self._value)

    def __array__(self, dtype=None, copy=None):
        return self._value if dtype is None else self._value.astype(dtype)

    def __repr__(self) -> str:
        return f"Parameter(shape={self.shape}, dtype={self._dtype.name}, value={self._value!r})"


class Module:
    """Attribute-walking container (gpflow/base.py:73-110)."""

    def _walk(self, seen: set) -> Iterator[Parameter]:
        if id(self) in seen:
            return
        seen.add(id(self))
        for v in self.__dict__.values():
            yield from _walk_value(v, seen)

    @property
    def parameters(self) -> Tuple[Parameter, ...]:
        return tuple(self._walk(set()))

    @property
    def trainable_parameters(self) -> Tuple[Parameter, ...]:
        return tuple(p for p in self.parameters if p.trainable)

    @property
    def trainable_variables(self) -> Tuple[Parameter, ...]:
        """The handles an optimiser updates (tf.Module.trainable_variables in the reference): the trainable Parameters;
        their `unconstrained_variable` / `assign_unconstrained` are the unconstrained view."""
        return self.trainable_parameters


def _walk_value(v: Any, seen: set) -> Iterator[Parameter]:
    if isinstance(v, Parameter):
        if id(v) not in seen:
            seen.add(id(v))
            yield v
    elif isinstance(v, Module):
        yield from v._walk(seen)
    elif isinstance(v, (list, tuple)):
        for x in v:
            yield from _walk_value(x, seen)
    elif isinstance(v, dict):
        for x in v.values():
            yield from _walk_value(x, seen)
