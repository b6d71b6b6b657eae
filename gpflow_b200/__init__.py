"""gpflow_b200 — H100-native (sm_90a) implementation of GPflow's GP-inference hot path behind the
reference's Python API: kernels -> Kuu/Kuf -> Cholesky / triangular solves -> GPR LML, SGPR / SVGP
ELBO, posterior mean / variance.  Host code is Python over a C ABI (include/gpk.h); all arithmetic
runs in hand-written CUDA kernels (gpflow_b200/csrc).  There is no CPU fallback."""
from . import config
from .config import default_float, default_jitter
from .base import Module, Parameter
from . import (conditionals, covariances, inducing_variables, kernels, kullback_leiblers, likelihoods,
               logdensities, mean_functions, models, ops, optimizers, posteriors, sharding, utilities)
from .utilities import set_trainable

__version__ = "0.1.0"
__all__ = ["Module", "Parameter", "conditionals", "config", "covariances", "default_float", "default_jitter",
           "inducing_variables", "kernels", "kullback_leiblers", "likelihoods", "logdensities", "mean_functions",
           "models", "ops", "optimizers", "posteriors", "set_trainable", "sharding", "utilities"]
