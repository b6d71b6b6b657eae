"""Optimiser drivers of the hot path (mirrors gpflow/optimizers/__init__.py: the Scipy driver and NaturalGradient; Adam
stands in for tf_keras.optimizers.Adam, which the reference's minibatch loops use)."""
from .adam import Adam
from .natgrad import NaturalGradient, XiNat, XiSqrtMeanVar, XiTransform
from .scipy import Scipy

__all__ = ["Adam", "NaturalGradient", "Scipy", "XiNat", "XiSqrtMeanVar", "XiTransform"]
