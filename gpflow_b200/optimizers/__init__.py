"""Optimiser drivers of the hot path (mirrors gpflow/optimizers/__init__.py: the Scipy driver and NaturalGradient)."""
from .natgrad import NaturalGradient, XiNat, XiSqrtMeanVar, XiTransform
from .scipy import Scipy

__all__ = ["NaturalGradient", "Scipy", "XiNat", "XiSqrtMeanVar", "XiTransform"]
