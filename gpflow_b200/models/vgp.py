"""Variational GP with a full-rank whitened Gaussian q (mirrors gpflow/models/vgp.py:46-161), Gaussian likelihood, and
the Opper-Archambeau parametrisation of the full-data posterior (vgp.py:266-419), any device likelihood.

VGP is a sibling model on the same operators as the hot path (SURVEY.md 8(f) rank 3): kernel build, Cholesky, GEMM with the
lower-triangular / column-sum-of-squares flags, the whitened Gauss KL and the Gaussian variational expectations."""
from __future__ import annotations

from typing import Optional

import ctypes

import numpy as np

from .. import _lib, config, kullback_leiblers, ops
from ..base import Parameter, positive, triangular
from ..conditionals import conditional
from ..kernels import Kernel, MultioutputKernel
from ..likelihoods import (Bernoulli, Gaussian, HeteroskedasticTFPConditional, Likelihood, MultiClass, Poisson,
                           StudentT)
from ..mean_functions import Constant, Linear, MeanFunction, Zero
from .model import (DeviceGradientMixin, GPModel, InternalDataTrainingLossMixin, centred_targets, checked_mean_values,
                    data_input_to_tensor, likelihood_scalars)


class VGP(GPModel, InternalDataTrainingLossMixin, DeviceGradientMixin):
    def __init__(self, data, kernel: Kernel, likelihood: Likelihood, mean_function: Optional[MeanFunction] = None,
                 num_latent_gps: Optional[int] = None):
        X_data, Y_data = data_input_to_tensor(data)
        if num_latent_gps is None:
            num_latent_gps = Y_data.shape[-1]  # model.py:103-133 for a Gaussian likelihood
        super().__init__(kernel, likelihood, mean_function, num_latent_gps)
        self.data = X_data, Y_data
        self.num_data = X_data.shape[0]
        N, P = self.num_data, self.num_latent_gps
        self.q_mu = Parameter(np.zeros((N, P)), dtype=config.default_float())                   # vgp.py:92-95
        eye = np.eye(N, dtype=config.default_float())
        self.q_sqrt = Parameter(np.tile(eye[None], (P, 1, 1)), transform=triangular())          # vgp.py:96-102

    def maximum_log_likelihood_objective(self):  # vgp.py:106-107
        return self.elbo()

    def elbo(self):
        """vgp.py:111-143: E_q[log p(Y|F)] - KL[q(F) || p(F)] as a device fp64 scalar."""
        if not isinstance(self.likelihood, Gaussian):
            raise NotImplementedError("VGP.elbo covers the Gaussian likelihood")
        X, Y = self.data
        N, P = self.num_data, self.num_latent_gps
        q_mu, q_sqrt = ops.to_device(self.q_mu), ops.to_device(self.q_sqrt)
        KL = kullback_leiblers.gauss_kl(q_mu, q_sqrt)                                            # vgp.py:124
        K = self.kernel(X)
        ops.add_diag_(K, config.default_jitter())                                                # vgp.py:127
        L, _ = ops.cholesky(K)                                                                   # vgp.py:128
        fmean = ops.gemm(L, q_mu)                                                                # vgp.py:129
        if not isinstance(self.mean_function, Zero):
            ops.axpby(1.0, self.mean_function(X), 1.0, fmean)
        # fvar[n, p] = sum_k (L tril(q_sqrt_p))[n, k]^2  (vgp.py:130-135) = column sums of squares of
        # tril(q_sqrt_p)^T L^T, taken in the GEMM epilogue: LTA [P, N, N] is never materialised
        fvar_t = ops.full((P, N), 0.0, like=L)
        for p in range(P):
            ops.gemm(q_sqrt[p], L, transa=True, transb=True, out=fvar_t[p],
                     flags=_lib.GPK_GEMM_A_LOWER | _lib.GPK_GEMM_COLSUMSQ)
        fvar = ops.transpose(fvar_t)
        var_exp = self.likelihood.variational_expectations(X, fmean, fvar, Y)                    # vgp.py:140
        out = ops.copy(var_exp)
        ops.axpby(-1.0, KL, 1.0, out)                                                            # vgp.py:142
        return out[0]

    def elbo_and_grad(self, *, device_arrays: bool = False):
        """Value and gradient of the ELBO in ONE fused call (gpk_vgp_elbo_grad): the backward pass the reference gets
        from TensorFlow autodiff through vgp.py:111-143.  Returns (elbo, grads): `elbo` as elbo(); `grads` a dict
        {Parameter: dF/d(constrained value)} (NumPy, after one small device->host read) for every kernel parameter of a
        fused expression, the likelihood variance, q_mu, q_sqrt (its strict upper part 0) and the Constant / Linear
        mean-function parameters; float64.  `device_arrays=True` leaves the gradients of q_mu and q_sqrt as device
        tensors."""
        if isinstance(self.kernel, MultioutputKernel):
            raise NotImplementedError("the VGP device gradient covers single-output kernels")
        if not isinstance(self.likelihood, Gaussian):
            raise NotImplementedError("the VGP device gradient covers the Gaussian likelihood")
        if not isinstance(self.mean_function, (Zero, Constant, Linear)):
            raise NotImplementedError("the VGP device gradient covers the Zero, Constant and Linear mean functions")
        lib = _lib.load()
        X, Y = (ops.to_device(d) for d in self.data)
        N, D = X.shape
        P = self.num_latent_gps
        dc = _lib.GPK_F64

        def call(kernel, out, n_out, grads, ws):
            q_mu, q_sqrt = ops.to_device(self.q_mu), ops.to_device(self.q_sqrt)
            Yc = centred_targets(self.mean_function, X, Y)
            return lib.gpk_vgp_elbo_grad(*kernel, ops._p(X), N, ops._ld(X), D, ops._p(Yc), P, ops._p(q_mu),
                                         ops._p(q_sqrt), self.likelihood._variance_value(), config.default_jitter(), dc,
                                         ops._p(out), n_out, ops._p(grads[0]), ops._p(grads[1]), ops._p(ws),
                                         ops._stream())

        return self._device_value_and_grad(
            X, P, layout=lambda: (lib.gpk_vgp_elbo_grad_ws(N, P, dc), lib.gpk_vgp_elbo_grad_dm(N, P, dc)), n_head=5,
            info_index=3, scalars={self.likelihood.variance: 4}, arrays=(self.q_mu, self.q_sqrt), call=call,
            entry="gpk_vgp_elbo_grad", device_arrays=device_arrays)

    _objective_and_grad = elbo_and_grad

    def predict_f(self, Xnew, full_cov: bool = False, full_output_cov: bool = False):            # vgp.py:145-161
        if full_output_cov:
            raise NotImplementedError("The predict_f method currently supports only the argument values "
                                      "full_output_cov=False")
        X, _ = self.data
        mu, var = conditional(Xnew, X, self.kernel, self.q_mu, q_sqrt=self.q_sqrt, full_cov=full_cov, white=True)
        if not isinstance(self.mean_function, Zero):
            ops.axpby(1.0, self.mean_function(ops.to_device(Xnew)), 1.0, mu)
        return mu, var


class VGPOpperArchambeau(GPModel, InternalDataTrainingLossMixin, DeviceGradientMixin):
    """q(f_p) = N(K alpha_p + m(X), (K^-1 + diag(lambda_p^2))^-1) (mirrors gpflow/models/vgp.py:266-419): 2 N parameters
    per latent GP where VGP needs N + N^2, for any likelihood the device covers (Gaussian, Bernoulli, Poisson, StudentT,
    MultiClass, HeteroskedasticTFPConditional)."""

    def __init__(self, data, kernel: Kernel, likelihood: Likelihood, mean_function: Optional[MeanFunction] = None,
                 num_latent_gps: Optional[int] = None):
        X_data, Y_data = data_input_to_tensor(data)
        if num_latent_gps is None:
            num_latent_gps = Y_data.shape[-1]  # model.py:146-160; MultiClass and the heteroskedastic likelihood pass it
        super().__init__(kernel, likelihood, mean_function, num_latent_gps)
        self.data = X_data, Y_data
        self.num_data = X_data.shape[0]
        N, P = self.num_data, self.num_latent_gps
        self.q_alpha = Parameter(np.zeros((N, P)), dtype=config.default_float())                 # vgp.py:312
        self.q_lambda = Parameter(np.ones((N, P)), transform=positive(), dtype=config.default_float())  # :313-315

    def maximum_log_likelihood_objective(self):  # vgp.py:319-320
        return self.elbo()

    def elbo(self):
        """vgp.py:325-376: E_q[log p(Y|F)] - KL[q(F) || p(F)] as a device fp64 scalar, composed from the public
        operators; K carries no jitter."""
        if isinstance(self.kernel, MultioutputKernel):
            raise NotImplementedError("VGPOpperArchambeau covers single-output kernels")
        X, Y = self.data
        N, P = self.num_data, self.num_latent_gps
        alpha = ops.to_device(self.q_alpha)
        lam_t = ops.transpose(ops.to_device(self.q_lambda))                                      # [P, N]
        K = self.kernel(X)
        K_alpha = ops.gemm(K, alpha)                                                             # vgp.py:346
        f_mean = ops.copy(K_alpha)
        if not isinstance(self.mean_function, Zero):
            ops.axpby(1.0, self.mean_function(X), 1.0, f_mean)                                   # vgp.py:347
        f_var_t = ops.empty((P, N), like=K)
        A_logdet = ops.zeros_scalar()
        trAi = ops.zeros_scalar()
        eye = ops.full((N, N), 0.0, like=K)
        ops.add_diag_(eye, 1.0)
        for p in range(P):
            lam = lam_t[p]
            A = ops.copy(K)                                                                      # vgp.py:353-358
            ops.scale_rows_(A, lam)
            ops.scale_cols_(A, lam)
            ops.add_diag_(A, 1.0)
            L, dinv = ops.cholesky(A)
            Li = ops.trsm(L, ops.copy(eye), dinv=dinv)                                           # vgp.py:359-360
            ops.reduce(ops.SUMLOG, L, N, inc=N + 1, scale=2.0, out=A_logdet, accumulate=True)    # vgp.py:365
            ops.reduce(ops.SUMSQ, Li, N * N, out=trAi, accumulate=True)                          # vgp.py:366
            ops.scale_cols_(Li, lam, invert=True)                                                # vgp.py:361
            inv_sq = ops.full((1, N), 1.0, like=K)
            ops.scale_cols_(inv_sq, lam, invert=True)
            ops.scale_cols_(inv_sq, lam, invert=True)
            ops.colsumsq(Li, out=f_var_t[p])
            ops.axpby(1.0, inv_sq[0], -1.0, f_var_t[p])                                          # vgp.py:362
        f_var = ops.transpose(f_var_t)
        prod = ops.copy(K_alpha)
        ops.hadamard_(prod, alpha)
        KL = ops.reduce(ops.SUM, prod, N * P)                                                    # vgp.py:368-373
        ops.axpby(1.0, A_logdet, 1.0, KL)
        ops.axpby(1.0, trAi, 1.0, KL)
        ops.axpby(-float(N * P), ops.full((1,), 1.0, like=KL), 1.0, KL)
        ops.axpby(0.0, KL, 0.5, KL)
        var_exp = self.likelihood.variational_expectations(X, f_mean, f_var, Y)                  # vgp.py:375
        out = ops.copy(var_exp)
        ops.axpby(-1.0, KL, 1.0, out)                                                            # vgp.py:376
        return out[0]

    def elbo_and_grad(self, *, device_arrays: bool = False):
        """Value and gradient of the ELBO in ONE fused call (gpk_vgp_oa_elbo_grad): the backward pass the reference gets
        from TensorFlow autodiff through vgp.py:325-376.  Returns (elbo, grads): `elbo` as elbo(); `grads` a dict
        {Parameter: dF/d(constrained value)} (NumPy, after one small device->host read) for every kernel parameter of a
        fused expression, the likelihood's parameter (Gaussian variance, StudentT scale, RobustMax epsilon), q_alpha,
        q_lambda and the Constant / Linear mean-function parameters; float64.  `device_arrays=True` leaves the gradients
        of q_alpha and q_lambda as device tensors."""
        if isinstance(self.kernel, MultioutputKernel):
            raise NotImplementedError("the VGPOpperArchambeau device gradient covers single-output kernels")
        lik = self.likelihood
        if not isinstance(lik, (Gaussian, Bernoulli, Poisson, StudentT, MultiClass, HeteroskedasticTFPConditional)):
            raise NotImplementedError("the VGPOpperArchambeau device gradient covers the Gaussian, Bernoulli, Poisson, "
                                      "StudentT, MultiClass and HeteroskedasticTFPConditional likelihoods")
        if not isinstance(self.mean_function, (Zero, Constant, Linear)):
            raise NotImplementedError("the VGPOpperArchambeau device gradient covers the Zero, Constant and Linear mean "
                                      "functions")
        if any(p.prior is not None for p in self.trainable_parameters):
            raise NotImplementedError("parameter priors are outside the hot path: the device gradient covers the "
                                      "likelihood only")
        lib = _lib.load()
        X, Y = (ops.to_device(d) for d in self.data)
        N, D = X.shape
        P = self.num_latent_gps
        dc = _lib.GPK_F64

        def call(kernel, out, n_out, grads, ws):
            mX = checked_mean_values(lik, self.mean_function, X, Y, P)
            q_alpha, q_lambda = ops.to_device(self.q_alpha), ops.to_device(self.q_lambda)
            return lib.gpk_vgp_oa_elbo_grad(*kernel, ops._p(X), N, ops._ld(X), D, ops._p(Y), ops._p(mX), P,
                                            ops._p(q_alpha), ops._p(q_lambda), ctypes.byref(lik._lik_desc()), dc,
                                            ops._p(out), n_out, ops._p(grads[0]), ops._p(grads[1]), ops._p(ws),
                                            ops._stream())

        def describe_info(info: int) -> str:
            p, k = divmod(info - 1, N)
            return f"latent {p}, pivot {k + 1}"

        return self._device_value_and_grad(
            X, P, layout=lambda: (lib.gpk_vgp_oa_elbo_grad_ws(N, P, dc), lib.gpk_vgp_oa_elbo_grad_dm(N, P, dc)),
            n_head=5, info_index=3, scalars=likelihood_scalars(lik, 4), arrays=(self.q_alpha, self.q_lambda),
            call=call, entry="gpk_vgp_oa_elbo_grad", device_arrays=device_arrays, describe_info=describe_info)

    _objective_and_grad = elbo_and_grad

    def predict_f(self, Xnew, full_cov: bool = False, full_output_cov: bool = False):            # vgp.py:379-419
        """The mean K(Xnew, X) alpha + m(Xnew) and, per latent, the variance K(Xnew, Xnew) - K(Xnew, X)
        (K + diag(lambda_p^-2))^-1 K(X, Xnew): [N*, P], or [P, N*, N*] with full_cov."""
        if full_output_cov:
            raise NotImplementedError("The predict_f method currently supports only the argument values "
                                      "full_output_cov=False")
        X, _ = self.data
        Xnew = ops.to_device(Xnew)
        N, P, M = self.num_data, self.num_latent_gps, Xnew.shape[0]
        lam_t = ops.transpose(ops.to_device(self.q_lambda))                                      # [P, N]
        Kx = self.kernel(X, Xnew)
        K = self.kernel(X)
        f_mean = ops.gemm(Kx, ops.to_device(self.q_alpha), transa=True)                         # vgp.py:408
        if not isinstance(self.mean_function, Zero):
            ops.axpby(1.0, self.mean_function(Xnew), 1.0, f_mean)
        if full_cov:
            f_var = ops.empty((P, M, M), like=K)
        else:
            f_var_t = ops.empty((P, M), like=K)
            Kdiag = self.kernel(Xnew, full_cov=False)
        for p in range(P):
            inv_sq = ops.full((1, N), 1.0, like=K)
            ops.scale_cols_(inv_sq, lam_t[p], invert=True)
            ops.scale_cols_(inv_sq, lam_t[p], invert=True)
            A = ops.copy(K)
            ops.add_diag_(A, vec=inv_sq[0])                                                      # vgp.py:411
            L, dinv = ops.cholesky(A)
            LiKx = ops.trsm(L, ops.copy(Kx), dinv=dinv)                                          # vgp.py:412-414
            if full_cov:
                ops.axpby(1.0, self.kernel(Xnew), 0.0, f_var[p])
                ops.gemm(LiKx, LiKx, transa=True, alpha=-1.0, beta=1.0, out=f_var[p])           # vgp.py:416
            else:
                ops.colsumsq(LiKx, out=f_var_t[p])
                ops.axpby(1.0, Kdiag, -1.0, f_var_t[p])                                          # vgp.py:418
        return f_mean, (f_var if full_cov else ops.transpose(f_var_t))
