"""Variational GP with a full-rank whitened Gaussian q (mirrors gpflow/models/vgp.py:46-161), Gaussian likelihood.

A sibling model on the same operators as the hot path (SURVEY.md 8(f) rank 3): kernel build, Cholesky, GEMM with the
lower-triangular / column-sum-of-squares flags, the whitened Gauss KL and the Gaussian variational expectations."""
from __future__ import annotations

from typing import Optional

import numpy as np

from .. import _lib, config, kullback_leiblers, ops
from ..base import Parameter, triangular
from ..conditionals import conditional
from ..kernels import Kernel, MultioutputKernel
from ..likelihoods import Gaussian, Likelihood
from ..mean_functions import Constant, Linear, MeanFunction, Zero
from .model import DeviceGradientMixin, GPModel, InternalDataTrainingLossMixin, centred_targets, data_input_to_tensor


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
