"""gpflow.kernels surface for the hot path (RBF / Matern / Linear / White / Constant, Sum / Product,
independent multi-output wrappers)."""
from .base import (Combination, Kernel, Product, ReducingCombination, Sum, compile_kernel, gradient_slots, kernel_matrix,
                   slot_gradients)
from .linears import Linear, Polynomial
from .materialised import AnisotropicStationary, ArcCosine, ChangePoints, Coregion, Cosine, Periodic
from .multioutput import (IndependentLatent, LinearCoregionalization, MultioutputKernel, SeparateIndependent,
                          SharedIndependent)
from .statics import Bias, Constant, Static, White
from .stationaries import (
    Exponential,
    IsotropicStationary,
    Matern12,
    Matern32,
    Matern52,
    RationalQuadratic,
    SquaredExponential,
    Stationary,
)

RBF = SquaredExponential

__all__ = [
    "AnisotropicStationary", "ArcCosine", "Bias", "ChangePoints", "Combination", "Coregion", "Cosine", "Periodic", "Constant", "Exponential", "IsotropicStationary", "IndependentLatent", "Kernel", "Linear", "LinearCoregionalization", "Matern12", "Polynomial",
    "Matern32", "Matern52", "MultioutputKernel", "Product", "RBF", "RationalQuadratic", "ReducingCombination",
    "SeparateIndependent", "SharedIndependent", "SquaredExponential", "Static", "Stationary", "Sum", "White",
    "compile_kernel", "gradient_slots", "kernel_matrix", "slot_gradients",
]
