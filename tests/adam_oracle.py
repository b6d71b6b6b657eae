"""NumPy oracle of the Adam step (tf_keras.optimizers.Adam.update_step, applied to the UNCONSTRAINED variable of each
parameter as the reference's minibatch loops do) and a host SVGP training loop driven by the gradient oracle
(tests/svgp_grad_oracle.py with the likelihoods of tests/lik_oracle.py).  The bijectors are restated here, independently
of gpflow_b200/base.py: identity, softplus and exp, each with the lower bound of gpflow.utilities.positive()."""
from typing import Dict, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as SV

IDENTITY, SOFTPLUS, EXP = "identity", "softplus", "exp"
KERAS_DEFAULTS = dict(lr=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-7)


def forward(kind: str, lower: float, u):
    u = np.asarray(u, dtype=np.float64)
    if kind == SOFTPLUS:
        return np.logaddexp(0.0, u) + lower
    if kind == EXP:
        return np.exp(u) + lower
    return u


def inverse(kind: str, lower: float, y):
    y = np.asarray(y, dtype=np.float64)
    if kind == SOFTPLUS:
        z = y - lower
        return z + np.log(-np.expm1(-z))
    if kind == EXP:
        return np.log(y - lower)
    return y


def forward_grad(kind: str, u):
    u = np.asarray(u, dtype=np.float64)
    if kind == SOFTPLUS:
        return 1.0 / (1.0 + np.exp(-u))
    if kind == EXP:
        return np.exp(u)
    return np.ones_like(u)


def lr_t(t: int, lr: float, beta_1: float, beta_2: float) -> float:
    """The bias-corrected step size of the 1-based step t."""
    return lr * np.sqrt(1.0 - beta_2 ** t) / (1.0 - beta_1 ** t)


def adam_step(u, g, m, v, t: int, *, lr, beta_1, beta_2, epsilon) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """One Keras Adam step on the variable u with the loss gradient g at the 1-based step t: (u', m', v')."""
    m = m + (1.0 - beta_1) * (g - m)
    v = v + (1.0 - beta_2) * (g * g - v)
    return u - lr_t(t, lr, beta_1, beta_2) * m / (np.sqrt(v) + epsilon), m, v


def constrained_step(value, grad, m, v, t: int, kind: str, lower: float, sign: float, **hyper):
    """The step as the device takes it: from the CONSTRAINED value and sign * (gradient of the loss w.r.t. it), through
    the bijector and back.  (value', m', v')."""
    u = inverse(kind, lower, value)
    u, m, v = adam_step(u, sign * np.asarray(grad, dtype=np.float64) * forward_grad(kind, u), m, v, t, **hyper)
    return forward(kind, lower, u), m, v


def svgp_loop(X, Y, params: Dict[str, Tuple[np.ndarray, str, float]], steps: int, *, lik: str, whiten: bool, num_data,
              jitter: float, train=None, **hyper) -> Dict[str, np.ndarray]:
    """`steps` Adam steps on the ELBO of an SVGP with a SquaredExponential kernel on the fixed batch (X, Y).  `params`
    maps "variance", "lengthscales", "Z", "q_mu", "q_sqrt" (and "lik", the Gaussian variance) to (value, bijector kind,
    lower bound); `train` names the ones Adam updates (default: all).  Returns the final values."""
    value = {k: np.array(p[0], dtype=np.float64) for k, p in params.items()}
    train = list(params) if train is None else list(train)
    state = {k: (np.zeros_like(value[k]), np.zeros_like(value[k])) for k in train}
    for t in range(1, steps + 1):
        kernel = O.SquaredExponential(float(value["variance"]), float(value["lengthscales"]))
        lo = LO.Gaussian(float(value["lik"])) if lik == "gaussian" else LO.make(lik)
        _, g = SV.svgp_elbo_and_grad(X, Y, [kernel], [value["Z"]], value["q_mu"], value["q_sqrt"], lo, whiten=whiten,
                                     num_data=num_data, jitter=jitter)
        grad = {"variance": g["leaves"][0]["variance"], "lengthscales": g["leaves"][0]["lengthscales"], "lik": g["lik"],
                "Z": g["Z"], "q_mu": g["q_mu"], "q_sqrt": g["q_sqrt"]}
        for k in train:
            _, kind, lower = params[k]
            gk = np.asarray(grad[k], dtype=np.float64).reshape(value[k].shape)
            value[k], *state[k] = constrained_step(value[k], gk, *state[k], t, kind, lower, -1.0, **hyper)
    return value
