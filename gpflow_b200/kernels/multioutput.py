"""Multi-output kernels (mirrors gpflow/kernels/multioutput/kernels.py:118-400): SharedIndependent, SeparateIndependent and
LinearCoregionalization, with the full_output_cov=False forms ([P, N, N2] / [N, P]) that the independent posteriors use."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

from .. import ops
import numpy as np

from ..base import Parameter
from .base import Combination, Kernel, compile_kernel, kernel_matrix


class MultioutputKernel(Kernel):
    @property
    def num_latent_gps(self) -> int:
        raise NotImplementedError

    @property
    def latent_kernels(self) -> Tuple[Kernel, ...]:
        raise NotImplementedError


def latent_sets(kernel: MultioutputKernel, inducing_variable) -> Tuple[int, Tuple[Kernel, ...], tuple]:
    """(L, latent kernels, inducing sets) of a multi-output kernel with Shared- / SeparateIndependent inducing variables,
    as covariances._latent_pairs pairs them: L latent GPs, and one kernel or one inducing set shared by every latent, or
    L of them.  A ValueError if the counts do not match."""
    from ..covariances import _latent_pairs

    L = len(_latent_pairs(inducing_variable, kernel))
    return L, tuple(kernel.latent_kernels), tuple(inducing_variable.inducing_variables)


class SharedIndependent(MultioutputKernel):
    """One kernel shared by `output_dim` independent outputs (kernels.py:118-197)."""

    def __init__(self, kernel: Kernel, output_dim: int) -> None:
        super().__init__()
        self.kernel = kernel
        self.output_dim = output_dim

    @property
    def num_latent_gps(self) -> int:
        return self.output_dim

    @property
    def latent_kernels(self) -> Tuple[Kernel, ...]:
        return (self.kernel,)

    def K(self, X, X2=None, full_output_cov: bool = False):
        if full_output_cov:
            raise NotImplementedError("full_output_cov=True is outside the hot path")
        return self.kernel(X, X2)  # [N, N2], broadcast over outputs by the caller

    def K_diag(self, X, full_output_cov: bool = False):
        if full_output_cov:
            raise NotImplementedError("full_output_cov=True is outside the hot path")
        return self.kernel(X, full_cov=False)

    def __call__(self, X, X2=None, *, full_cov: bool = True, full_output_cov: bool = False, presliced=False):
        return self.K(X, X2, full_output_cov) if full_cov else self.K_diag(X, full_output_cov)


class SeparateIndependent(MultioutputKernel, Combination):
    """A different kernel per output (kernels.py:200-271): K -> [P, N, N2], K_diag -> [N, P]."""

    def __init__(self, kernels: Sequence[Kernel], name: Optional[str] = None) -> None:
        Kernel.__init__(self, name=name)
        self.kernels = list(kernels)

    @property
    def num_latent_gps(self) -> int:
        return len(self.kernels)

    @property
    def latent_kernels(self) -> Tuple[Kernel, ...]:
        return tuple(self.kernels)

    def K(self, X, X2=None, full_output_cov: bool = False):
        if full_output_cov:
            raise NotImplementedError("full_output_cov=True is outside the hot path")
        X = ops.to_device(X)
        X2d = None if X2 is None else ops.to_device(X2)
        N2 = X.shape[0] if X2d is None else X2d.shape[0]
        out = ops.empty((len(self.kernels), X.shape[0], N2), like=X)
        for p, k in enumerate(self.kernels):  # kernels.py:236-239
            if k.is_fusable():
                ops.kbuild(compile_kernel(k, X.shape[1]), X, X2d, out=out[p])
            else:
                ops.axpby(1.0, k(X, X2d), 0.0, out[p])
        return out

    def K_diag(self, X, full_output_cov: bool = False):
        if full_output_cov:
            raise NotImplementedError("full_output_cov=True is outside the hot path")
        X = ops.to_device(X)
        tmp = ops.empty((len(self.kernels), X.shape[0]), like=X)
        for p, k in enumerate(self.kernels):  # kernels.py:265-271
            if k.is_fusable():
                ops.kdiag(compile_kernel(k, X.shape[1]), X, out=tmp[p])
            else:
                ops.axpby(1.0, k(X, full_cov=False), 0.0, tmp[p])
        return ops.transpose(tmp)  # [N, P]

    def __call__(self, X, X2=None, *, full_cov: bool = True, full_output_cov: bool = False, presliced=False):
        return self.K(X, X2, full_output_cov) if full_cov else self.K_diag(X, full_output_cov)


class IndependentLatent(MultioutputKernel):
    """kernels.py:274-295: outputs are a transformation of independent latent GPs g."""

    def Kgg(self, X, X2):
        raise NotImplementedError


class LinearCoregionalization(IndependentLatent, SeparateIndependent):
    """f = W g with L independent latent GPs g_l ~ GP(0, k_l) and W [P, L] (kernels.py:298-400).  The posteriors work on
    the latent GPs (Kgg, [L, N, N2]) and mix afterwards (conditionals/util.py:518-563), so K / K_diag here return the
    LATENT covariances; `K_outputs_diag` gives the [N, P] output variances sum_l W[p, l]^2 k_l(x, x)."""

    def __init__(self, kernels: Sequence[Kernel], W, name: Optional[str] = None) -> None:
        SeparateIndependent.__init__(self, kernels, name=name)
        self.W = Parameter(W)
        if self.W.numpy().ndim != 2 or self.W.numpy().shape[1] != len(self.kernels):
            raise ValueError("W must have shape [P, L] with L = number of latent kernels")

    @property
    def num_latent_gps(self) -> int:
        return int(self.W.numpy().shape[-1])

    def Kgg(self, X, X2=None):  # kernels.py:320-323
        return SeparateIndependent.K(self, X, X2)

    def K_outputs_diag(self, X):  # kernels.py:382-400 with full_output_cov=False
        Kd = SeparateIndependent.K_diag(self, X)                       # [N, L]
        W2 = ops.to_device(np.square(self.W.numpy()))                   # [P, L]
        return ops.gemm(Kd, W2, transb=True)                            # [N, P]
