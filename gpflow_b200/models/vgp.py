"""Variational GP with a full-rank whitened Gaussian q (mirrors gpflow/models/vgp.py:46-161), Gaussian likelihood.

A sibling model on the same operators as the hot path (SURVEY.md 8(f) rank 3): kernel build, Cholesky, GEMM with the
lower-triangular / column-sum-of-squares flags, the whitened Gauss KL and the Gaussian variational expectations."""
from __future__ import annotations

from typing import Optional

import numpy as np

from .. import _lib, config, kullback_leiblers, ops
from ..base import Parameter, triangular
from ..conditionals import conditional
from ..kernels import Kernel, MultioutputKernel, compile_kernel
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

    def elbo_and_grad(self):
        """Value and gradient of the ELBO in ONE fused call (gpk_vgp_elbo_grad): the backward pass the reference gets
        from TensorFlow autodiff through vgp.py:111-143.  Returns (elbo, grads): `elbo` as elbo(); `grads` a dict
        {Parameter: dF/d(constrained value)} (NumPy, after one small device->host read) for every kernel parameter of a
        fused expression, the likelihood variance, q_mu, q_sqrt (its strict upper part 0) and the Constant / Linear
        mean-function parameters; float64."""
        from ..kernels import gradient_slots, slot_gradients

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
        slots = gradient_slots(self.kernel, D)  # NotImplementedError for materialised kernels
        self._refuse_device_gradient(X)
        dc = _lib.GPK_F64
        need = lib.gpk_vgp_elbo_grad_ws(N, P, dc)
        if getattr(self, "_gws", None) is None or self._gws.numel() < need or self._gws.device != X.device:
            self._gws = ops.scratch_bytes(need)
        nodes, n_nodes, dims, ard = compile_kernel(self.kernel, D)
        n_slots = lib.gpk_gpr_lml_grad_slots(nodes, n_nodes, dims, ard, D)
        _lib.check(min(n_slots, 0), "gpk_gpr_lml_grad_slots")
        n_out = 5 + n_slots
        T = ops.torch()
        q_mu, q_sqrt = ops.to_device(self.q_mu), ops.to_device(self.q_sqrt)
        out = T.empty((n_out,), dtype=T.float64, device=X.device)
        dq_mu = T.empty(tuple(q_mu.shape), dtype=T.float64, device=X.device)
        dq_sqrt = T.empty(tuple(q_sqrt.shape), dtype=T.float64, device=X.device)
        Yc = centred_targets(self.mean_function, X, Y)
        _lib.check(lib.gpk_vgp_elbo_grad(nodes, n_nodes, dims, ard, ops._p(X), N, ops._ld(X), D, ops._p(Yc), P,
                                         ops._p(q_mu), ops._p(q_sqrt), self.likelihood._variance_value(),
                                         config.default_jitter(), dc, ops._p(out), n_out, ops._p(dq_mu),
                                         ops._p(dq_sqrt), ops._p(self._gws), ops._stream()), "gpk_vgp_elbo_grad")
        mean_dev = self._mean_gradients(self._gws, lib.gpk_vgp_elbo_grad_dm(N, P, dc), X, N, P)
        h = out.cpu().numpy()
        if int(h[3]) != 0:
            raise ops.NonPositiveDefiniteError(f"Cholesky decomposition was not successful (pivot {int(h[3])} <= 0)")
        grads = {self.likelihood.variance: np.asarray(h[4]), self.q_mu: dq_mu.cpu().numpy(),
                 self.q_sqrt: dq_sqrt.cpu().numpy(), **slot_gradients(slots, h[5:])}
        for p, g in mean_dev:
            grads[p] = g.cpu().numpy().reshape(p.shape)
        return ops.objective(out, 0, 3), grads

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
