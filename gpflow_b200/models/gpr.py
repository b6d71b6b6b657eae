"""Gaussian-process regression (mirrors gpflow/models/gpr.py:36-196)."""
from __future__ import annotations

import ctypes
from typing import Any, Optional

from .. import _lib, ops, posteriors
from ..kernels import Kernel, compile_kernel
from ..likelihoods import Gaussian
from ..mean_functions import MeanFunction
from .model import DeviceGradientMixin, GPModel, InternalDataTrainingLossMixin, centred_targets, data_input_to_tensor


class GPR(GPModel, InternalDataTrainingLossMixin, DeviceGradientMixin):
    def __init__(self, data, kernel: Kernel, mean_function: Optional[MeanFunction] = None,
                 noise_variance: Any = None, likelihood: Optional[Gaussian] = None):
        assert (noise_variance is None) or (likelihood is None), "Cannot set both `noise_variance` and `likelihood`."
        if likelihood is None:
            if noise_variance is None:
                noise_variance = 1.0  # gpr.py:75-78
            likelihood = Gaussian(noise_variance)
        _, Y_data = data
        super().__init__(kernel, likelihood, mean_function, num_latent_gps=Y_data.shape[-1])
        self.data = data_input_to_tensor(data)
        self._ws = None
        self._out = None

    def maximum_log_likelihood_objective(self):  # gpr.py:85-86
        return self.log_marginal_likelihood()

    def log_marginal_likelihood(self):
        """gpr.py:91-107 in ONE fused call (gpk_gpr_lml): lower-triangle K-build with the noise on the
        diagonal, blocked Cholesky with (Y-m)^T riding along as extra rows, log-density reduction.
        Returns a device fp64 tensor of shape [] (float() it to synchronise)."""
        lib = _lib.load()
        X, Y = self.data
        N, D = X.shape
        P = Y.shape[1]
        dc = ops.dtype_code(X)
        Yc = centred_targets(self.mean_function, X, Y)
        if self.likelihood.heteroskedastic:   # per-point noise (scalar_continuous.py:92-111; model_utils.py:33-50)
            s2, svec = 0.0, self.likelihood.variance_at(X).reshape(-1).contiguous()
        else:
            s2, svec = self.likelihood._variance_value(), None
        # a fresh result vector per call: earlier results stay valid when the model is evaluated again
        self._out = ops.torch().empty((4,), dtype=ops.torch().float64, device=X.device)
        if not self.kernel.is_fusable():
            return self._lml_unfused(X, Yc, s2, svec)
        need = lib.gpk_gpr_lml_ws(N, P, dc)
        if self._ws is None or self._ws.numel() < need:
            self._ws = ops.scratch_bytes(need)
        nodes, n_nodes, dims, ard = compile_kernel(self.kernel, D)
        _lib.check(lib.gpk_gpr_lml(nodes, n_nodes, dims, ard, ops._p(X), N, ops._ld(X), D, ops._p(Yc), P, s2, ops._p(svec),
                                   dc, ops._p(self._out), ops._p(self._ws), ops._stream()), "gpk_gpr_lml")
        return ops.objective(self._out, 0, 3)

    def _lml_unfused(self, X, Yc, s2, svec):
        """gpr.py:91-107 composed from the individual operators for kernels without a fused K-build record (Cosine,
        Periodic, ArcCosine, Coregion, ChangePoints and combinations with them): K materialised, (Y - m)^T riding along
        the factorisation as extra rows, the same reductions."""
        import math
        from ..kernels import kernel_matrix

        T = ops.torch()
        N, P = Yc.shape
        A = ops.empty((N + P, N), like=X)
        K = kernel_matrix(self.kernel, X, None, diag_scalar=s2, diag_vec=svec)
        ops.axpby(1.0, K, 0.0, A[:N])
        ops.transpose(Yc, out=A[N:])
        info = T.empty((1,), dtype=T.int32, device=X.device)
        lib = _lib.load()
        ws = ops.scratch_bytes(lib.gpk_potrf_ws(N, N + P, ops.dtype_code(A)))
        _lib.check(lib.gpk_potrf(ops._p(A), N, N + P, ops._ld(A), ops.dtype_code(A), ops._p(info), ops._p(ws),
                                 ops._stream()), "gpk_potrf")
        out = self._out
        ops.fill(out.view(1, 4), 0.0)
        ops.reduce(ops.SUMSQ, A[N:], N * P, 1, out=out[1:2], accumulate=True)            # sum alpha^2
        ops.reduce(ops.SUMLOG, A, N, ops._ld(A) + 1, out=out[2:3], accumulate=True)       # sum log diag L
        ops.axpby(-0.5, out[1:2], 0.0, out[0:1])
        ops.axpby(-float(P), out[2:3], 1.0, out[0:1])
        ops.axpby(1.0, ops.full((1,), -0.5 * N * P * math.log(2.0 * math.pi), dtype="float64"), 1.0, out[0:1])
        self._info = info
        return ops.objective(out, 0, None, info_tensor=info)

    def log_marginal_likelihood_and_grad(self):
        """Value and gradient in ONE fused call (gpk_gpr_lml_grad_expr): the backward pass the reference gets from
        TensorFlow autodiff through gpr.py:91-107.  Returns (lml, grads): `lml` as log_marginal_likelihood(); `grads` a
        dict {Parameter: dLML/d(constrained value)} (NumPy, after one small device->host read) for every kernel
        parameter of a fused expression (Sum / Product of stationary, RationalQuadratic, Linear, Polynomial, White and
        Constant leaves), the likelihood variance and the Constant / Linear mean-function parameters; float64 only."""
        lib = _lib.load()
        X, Y = self.data
        N, D = X.shape
        P = Y.shape[1]

        def call(kernel, out, n_out, _, ws):
            Yc = centred_targets(self.mean_function, X, Y)
            status = lib.gpk_gpr_lml_grad_expr(*kernel, ops._p(X), N, ops._ld(X), D, ops._p(Yc), P,
                                               self.likelihood._variance_value(), _lib.GPK_F64, ops._p(out), n_out,
                                               ops._p(ws), ops._stream())
            if status == 0:
                self._out = out
            return status

        def layout():  # dLML/dm = alpha = K^-1 (Y - m)
            return lib.gpk_gpr_lml_grad_ws(N, P, _lib.GPK_F64), lib.gpk_gpr_lml_grad_alpha(N, P, _lib.GPK_F64)

        return self._device_value_and_grad(X, P, layout=layout, n_head=5, info_index=3,
                                           scalars={self.likelihood.variance: 4}, arrays=(), call=call,
                                           entry="gpk_gpr_lml_grad_expr")

    _objective_and_grad = log_marginal_likelihood_and_grad

    def cholesky_info(self) -> int:
        """0, or the 1-based index of the first non-positive pivot of the last evaluation."""
        if getattr(self, "_info", None) is not None and not self.kernel.is_fusable():
            return int(self._info.item())
        return int(self._out[3].item()) if self._out is not None else 0

    def posterior(self, precompute_cache=posteriors.PrecomputeCacheType.TENSOR) -> posteriors.GPRPosterior:
        """gpr.py:146-175."""
        return posteriors.GPRPosterior(kernel=self.kernel, data=self.data, likelihood=self.likelihood,
                                       mean_function=self.mean_function,
                                       precompute_cache=posteriors._validate_precompute_cache_type(precompute_cache))

    def predict_f(self, Xnew, full_cov: bool = False, full_output_cov: bool = False):  # gpr.py:178-190
        return self.posterior(posteriors.PrecomputeCacheType.NOCACHE).fused_predict_f(
            Xnew, full_cov=full_cov, full_output_cov=full_output_cov)
