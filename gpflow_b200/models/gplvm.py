"""Bayesian GPLVM (mirrors gpflow/models/gplvm.py:84-280): q(X) = N(X_data_mean, diag X_data_var) over the latent inputs,
the collapsed bound of Titsias & Lawrence (2010) with the RBF kernel expectations (psi statistics) computed on the device
(csrc/psi.cu), its gradient in one fused call, and prediction composed from the psi statistics and the device operators."""
from __future__ import annotations

from typing import Any, Optional

import numpy as np

from .. import _lib, config, covariances, ops
from ..base import Parameter, positive
from ..inducing_variables import InducingPoints, inducingpoint_wrapper
from ..kernels import Kernel, SquaredExponential, compile_kernel
from ..likelihoods import Gaussian
from .model import DeviceGradientMixin, GPModel, InternalDataTrainingLossMixin, data_input_to_tensor


class BayesianGPLVM(GPModel, InternalDataTrainingLossMixin, DeviceGradientMixin):
    def __init__(self, data: Any, X_data_mean: Any, X_data_var: Any, kernel: Kernel,
                 num_inducing_variables: Optional[int] = None, inducing_variable: Any = None,
                 X_prior_mean: Any = None, X_prior_var: Any = None):
        """gplvm.py:92-157.  `data` Y [N, P]; X_data_mean, X_data_var [N, Q]; exactly one of `inducing_variable` and
        `num_inducing_variables` (then Z is a random permutation of the rows of X_data_mean, first M kept).  The prior
        mean defaults to 0 and the prior variance to 1."""
        X_data_mean = np.asarray(X_data_mean.numpy() if isinstance(X_data_mean, Parameter) else X_data_mean)
        num_data, num_latent_gps = X_data_mean.shape
        super().__init__(kernel, Gaussian(), num_latent_gps=num_latent_gps)
        (self.data,) = data_input_to_tensor((data,))
        self.X_data_mean = Parameter(X_data_mean)
        self.X_data_var = Parameter(X_data_var, transform=positive())
        self.num_data = num_data
        self.output_dim = self.data.shape[-1]
        if (inducing_variable is None) == (num_inducing_variables is None):
            raise ValueError("BayesianGPLVM needs exactly one of `inducing_variable` and `num_inducing_variables`")
        if inducing_variable is None:
            inducing_variable = InducingPoints(np.random.permutation(X_data_mean)[:num_inducing_variables])
        self.inducing_variable = inducingpoint_wrapper(inducing_variable)
        assert X_data_mean.shape[1] == self.num_latent_gps
        shape = (self.num_data, self.num_latent_gps)
        self.X_prior_mean = np.broadcast_to(np.asarray(0.0 if X_prior_mean is None else X_prior_mean,
                                                       dtype=np.float64), shape).copy()
        self.X_prior_var = np.broadcast_to(np.asarray(1.0 if X_prior_var is None else X_prior_var,
                                                      dtype=np.float64), shape).copy()
        self._prior_dev = None

    def _check(self) -> None:
        """The device path covers one SquaredExponential leaf in float64 without priors."""
        if type(self.kernel) is not SquaredExponential:
            raise NotImplementedError(f"BayesianGPLVM on the device covers one SquaredExponential kernel, not "
                                      f"{type(self.kernel).__name__}: its expectations need quadrature or "
                                      "cross-expectations")
        if ops.dtype_code(self.data) != _lib.GPK_F64 or self.X_data_mean.dtype != np.float64:
            raise NotImplementedError("BayesianGPLVM: the psi statistics compute in float64")
        if any(p.prior is not None for p in self.parameters):
            raise NotImplementedError("BayesianGPLVM: parameter priors are outside the hot path")

    def _inputs(self):
        """Device mu, S [N, Q], Z [M, Q], the prior mean and variance [N, Q], and the compiled kernel."""
        self._check()
        dev = ops.require_cuda()
        mu = self.X_data_mean.device(dev)
        S = self.X_data_var.device(dev)
        Z = ops.to_device(self.inducing_variable.Z)
        if self._prior_dev is None or self._prior_dev[0].device != mu.device:
            self._prior_dev = (ops.to_device(self.X_prior_mean), ops.to_device(self.X_prior_var))
        return mu, S, Z, self._prior_dev[0], self._prior_dev[1], compile_kernel(self.kernel, mu.shape[1])

    def maximum_log_likelihood_objective(self):  # gplvm.py:159-160
        return self.elbo()

    def elbo(self):
        """gplvm.py:162-216 in one fused call (gpk_bgplvm_elbo); device fp64 scalar."""
        lib = _lib.load()
        mu, S, Z, m0, p0, kernel = self._inputs()
        N, Q = mu.shape
        M, P = Z.shape[0], self.data.shape[1]
        need = lib.gpk_bgplvm_elbo_ws(N, Q, M, P)
        if getattr(self, "_ws", None) is None or self._ws.numel() < need or self._ws.device != mu.device:
            self._ws = ops.scratch_bytes(need)
        T = ops.torch()
        out = T.empty((9,), dtype=T.float64, device=mu.device)
        _lib.check(lib.gpk_bgplvm_elbo(*kernel, ops._p(mu), ops._p(S), N, Q, ops._p(self.data), P, ops._p(Z), M,
                                       ops._ld(Z), ops._p(m0), ops._p(p0), self.likelihood._variance_value(),
                                       config.default_jitter(), ops._p(out), ops._p(self._ws), ops._stream()),
                   "gpk_bgplvm_elbo")
        return ops.objective(out, 0, 8)

    def elbo_and_grad(self, *, device_arrays: bool = False):
        """Value and gradient of the bound in ONE fused call (gpk_bgplvm_elbo_grad): (elbo, grads), `elbo` as elbo() and
        `grads` {Parameter: dF/d(constrained value)} for the likelihood variance, the kernel variance and
        lengthscale(s), X_data_mean, X_data_var and the inducing points Z.  `device_arrays=True` leaves the gradients
        of the three arrays device tensors."""
        lib = _lib.load()
        mu, S, Z, m0, p0, _ = self._inputs()
        N, Q = mu.shape
        M, P = Z.shape[0], self.data.shape[1]

        def call(kernel, out, n_out, grads, ws):
            return lib.gpk_bgplvm_elbo_grad(*kernel, ops._p(mu), ops._p(S), N, Q, ops._p(self.data), P, ops._p(Z), M,
                                            ops._ld(Z), ops._p(m0), ops._p(p0), self.likelihood._variance_value(),
                                            config.default_jitter(), ops._p(out), n_out, ops._p(grads[0]),
                                            ops._p(grads[1]), ops._p(grads[2]), ops._p(ws), ops._stream())

        return self._device_value_and_grad(
            mu, P, layout=lambda: (lib.gpk_bgplvm_elbo_grad_ws(N, Q, M, P), 0), n_head=10, info_index=8,
            scalars={self.likelihood.variance: 9},
            arrays=(self.X_data_mean, self.X_data_var, self.inducing_variable.Z), call=call,
            entry="gpk_bgplvm_elbo_grad", device_arrays=device_arrays)

    _objective_and_grad = elbo_and_grad

    def psi_statistics(self):
        """(psi0 [1], psi1 [N, M], psi2 [M, M]) of q(X) on the device (gpk_rbf_psi; psi2 summed over the points)."""
        lib = _lib.load()
        mu, S, Z, _, _, kernel = self._inputs()
        N, Q = mu.shape
        M = Z.shape[0]
        T = ops.torch()
        psi0 = T.empty((1,), dtype=T.float64, device=mu.device)
        psi1 = T.empty((N, M), dtype=T.float64, device=mu.device)
        psi2 = T.empty((M, M), dtype=T.float64, device=mu.device)
        ws = ops.scratch_bytes(lib.gpk_rbf_psi_ws(N, M))
        _lib.check(lib.gpk_rbf_psi(*kernel, ops._p(mu), ops._p(S), N, Q, ops._p(Z), M, ops._ld(Z), ops._p(psi0),
                                   ops._p(psi1), ops._p(psi2), ops._p(ws), ops._stream()), "gpk_rbf_psi")
        return psi0, psi1, psi2

    def predict_f(self, Xnew, full_cov: bool = False, full_output_cov: bool = False):
        """gplvm.py:218-274 composed from the psi statistics and the device operators."""
        if full_output_cov:
            raise NotImplementedError("BayesianGPLVM.predict_f does not support full_output_cov=True")
        _, psi1, psi2 = self.psi_statistics()
        Y = self.data
        s2 = self.likelihood._variance_value()
        iv = self.inducing_variable
        Xnew = ops.to_device(Xnew)
        Kus = covariances.Kuf(iv, self.kernel, Xnew)
        L, dinv = ops.cholesky(covariances.Kuu(iv, self.kernel, jitter=config.default_jitter()))
        A = ops.trsm(L, ops.transpose(psi1), dinv=dinv)
        tmp = ops.trsm(L, psi2, dinv=dinv)
        B = ops.trsm(L, ops.transpose(tmp), dinv=dinv)
        ops.axpby(0.0, B, 1.0 / s2, B)
        ops.add_diag_(B, 1.0)
        LB, dinvB = ops.cholesky(B)
        c = ops.trsm(LB, ops.gemm(A, Y, alpha=1.0 / s2), dinv=dinvB)
        tmp1 = ops.trsm(L, Kus, dinv=dinv)
        tmp2 = ops.trsm(LB, ops.copy(tmp1), dinv=dinvB)
        mean = ops.gemm(tmp2, c, transa=True)
        P = Y.shape[1]
        if full_cov:
            v = ops.copy(self.kernel(Xnew))
            ops.gemm(tmp2, tmp2, transa=True, alpha=1.0, beta=1.0, out=v)
            ops.gemm(tmp1, tmp1, transa=True, alpha=-1.0, beta=1.0, out=v)
            var = ops.empty((P,) + tuple(v.shape), like=v)
            for p in range(P):
                ops.axpby(1.0, v, 0.0, var[p])
            return mean, var
        v = ops.copy(self.kernel(Xnew, full_cov=False))
        ops.colsumsq(tmp2, scale=1.0, out=v, accumulate=True)
        ops.colsumsq(tmp1, scale=-1.0, out=v, accumulate=True)
        var_t = ops.empty((P, v.shape[0]), like=v)
        for p in range(P):
            ops.axpby(1.0, v, 0.0, var_t[p])
        return mean, ops.transpose(var_t)

    def predict_log_density(self, data, full_cov: bool = False, full_output_cov: bool = False):  # gplvm.py:276-280
        raise NotImplementedError
