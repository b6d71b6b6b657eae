"""Sparse variational GP (mirrors gpflow/models/svgp.py:36-261)."""
from __future__ import annotations

import ctypes
from typing import Any, Optional, Tuple

import numpy as np

from .. import _lib, config, kullback_leiblers, ops, posteriors
from ..base import Parameter, positive, triangular
from ..conditionals import conditional
from ..inducing_variables import InducingVariables, inducingpoint_wrapper
from ..kernels import Kernel, MultioutputKernel, compile_kernel
from ..likelihoods import Bernoulli, Gaussian, Likelihood, MultiClass, Poisson, StudentT
from ..mean_functions import Constant, Linear, MeanFunction, Zero
from .model import DeviceGradientMixin, ExternalDataTrainingLossMixin, GPModel


class SVGP(GPModel, ExternalDataTrainingLossMixin, DeviceGradientMixin):
    def __init__(self, kernel: Kernel, likelihood: Likelihood, inducing_variable, *,
                 mean_function: Optional[MeanFunction] = None, num_latent_gps: int = 1, q_diag: bool = False,
                 q_mu=None, q_sqrt=None, whiten: bool = True, num_data=None):
        super().__init__(kernel, likelihood, mean_function, num_latent_gps)
        self.num_data = num_data
        self.whiten = whiten
        self.inducing_variable: InducingVariables = inducingpoint_wrapper(inducing_variable)
        self.q_diag = q_diag
        self._init_variational_parameters(self.inducing_variable.num_inducing, q_mu, q_sqrt, q_diag)
        self._ws = None
        self._last = None

    def _init_variational_parameters(self, num_inducing: int, q_mu, q_sqrt, q_diag: bool) -> None:
        """svgp.py:91-148."""
        q_mu = np.zeros((num_inducing, self.num_latent_gps)) if q_mu is None else q_mu
        self.q_mu = Parameter(q_mu, dtype=config.default_float())
        if q_sqrt is None:
            if q_diag:
                self.q_sqrt = Parameter(np.ones((num_inducing, self.num_latent_gps)), transform=positive())
            else:
                eye = np.eye(num_inducing, dtype=config.default_float())
                self.q_sqrt = Parameter(np.tile(eye[None], (self.num_latent_gps, 1, 1)), transform=triangular())
        else:
            if q_diag:
                assert np.ndim(q_sqrt) == 2
                self.num_latent_gps = np.shape(q_sqrt)[1]
                self.q_sqrt = Parameter(q_sqrt, transform=positive())
            else:
                assert np.ndim(q_sqrt) == 3
                self.num_latent_gps = np.shape(q_sqrt)[0]
                self.q_sqrt = Parameter(q_sqrt, transform=triangular())

    def prior_kl(self):  # svgp.py:153-156
        return kullback_leiblers.prior_kl(self.inducing_variable, self.kernel, self.q_mu, self.q_sqrt,
                                          whiten=self.whiten)

    def maximum_log_likelihood_objective(self, data):  # svgp.py:159-160
        return self.elbo(data)

    def elbo(self, data, *, latent_range: Optional[Tuple[int, int]] = None, batch_total: Optional[int] = None,
             include_kl: bool = True):
        """svgp.py:166-181 in ONE fused call (gpk_svgp_elbo) for a single-output kernel and Gaussian
        likelihood.  Returns a device fp64 scalar.  Sharding over GPUs (SURVEY 8(e), see sharding.py):
        `latent_range=(p0, p1)` evaluates the share of latent GPs [p0, p1) (data term and KL of those latents);
        `batch_total=B` says that `data` holds only some ROWS of a minibatch of B rows (the data term is a sum over
        rows rescaled by num_data / B, svgp.py:173-181) and `include_kl=False` leaves the KL to another rank;
        in both cases the shares of all ranks sum to the full ELBO."""
        if isinstance(self.kernel, MultioutputKernel) or not self.kernel.is_fusable() or \
                not isinstance(self.likelihood, Gaussian) or self.likelihood.heteroskedastic:
            # multi-output / materialised kernels: composed from the public operators exactly as the reference composes
            # them (prior_kl, the posterior's predict_f, variational_expectations; svgp.py:166-181)
            if latent_range is not None or batch_total is not None or not include_kl:
                raise NotImplementedError("sharding options cover the fused single-output evaluation")
            return self.elbo_unfused(data)
        out = self._fused(data, latent_range, 0, None, batch_total)
        if include_kl:
            return ops.objective(out, 0, 3)
        share = ops.copy(out[1:2])                     # sum of variational expectations (unscaled)
        ops.axpby(0.0, share, self._scale(data, batch_total), share)
        return share[0]

    def _scale(self, data, batch_total):
        B = int(data[0].shape[0]) if batch_total is None else int(batch_total)
        return 1.0 if self.num_data is None else float(self.num_data) / B     # svgp.py:175-180

    def _fused(self, data, latent_range, stage, cols, batch_total=None):
        if isinstance(self.kernel, MultioutputKernel) or not isinstance(self.likelihood, Gaussian):
            raise NotImplementedError("fused SVGP.elbo covers single-output kernels with a Gaussian likelihood")
        lib = _lib.load()
        X, Y = (ops.to_device(d) for d in data)
        B, D = X.shape
        P = self.num_latent_gps
        mX = self._mean_values(X, Y)
        Z = ops.to_device(self.inducing_variable.Z)
        M = Z.shape[0]
        dc = ops.dtype_code(X)
        need = lib.gpk_svgp_elbo_ws(B, M, P, dc)
        if self._ws is None or self._ws.numel() < need:
            self._ws = ops.scratch_bytes(need)
        out = ops.torch().empty((4,), dtype=ops.torch().float64, device=X.device)
        q_mu, q_sqrt = ops.to_device(self.q_mu), ops.to_device(self.q_sqrt)
        scale = self._scale(data, batch_total)
        p0, p1 = (0, P) if latent_range is None else latent_range
        c0, c1 = (0, B) if cols is None else cols
        nodes, n_nodes, dims, ard = compile_kernel(self.kernel, D)
        _lib.check(lib.gpk_svgp_elbo_staged(nodes, n_nodes, dims, ard, ops._p(X), B, ops._ld(X), D, ops._p(Y),
                                            ops._p(mX), P, ops._p(Z), M, ops._ld(Z), ops._p(q_mu), ops._p(q_sqrt),
                                            int(self.q_diag), int(self.whiten),
                                            ctypes.byref(self.likelihood._lik_desc()), scale, config.default_jitter(),
                                            p0, p1, stage, c0, c1, dc, ops._p(out), ops._p(self._ws), ops._stream()),
                   "gpk_svgp_elbo")
        self._last = out
        return out

    def elbo_and_grad(self, data, *, device_arrays: bool = False):
        """Value and gradient of the ELBO on the batch `data` in ONE fused call (gpk_svgp_elbo_grad): the backward pass
        the reference gets from TensorFlow autodiff through svgp.py:166-181, including the num_data / B scale, for the
        Gaussian, Bernoulli, Poisson, StudentT and MultiClass (RobustMax) likelihoods.  Returns (elbo, grads): `elbo` as
        elbo(data); `grads` a dict {Parameter: dF/d(constrained value)} (NumPy, after one small device->host read) for
        every kernel parameter of a fused expression, the Gaussian variance, the StudentT scale or the RobustMax epsilon,
        the inducing points Z, q_mu, q_sqrt (its strict upper part 0) and the Constant / Linear mean-function
        parameters; float64, both whiten and both q_diag settings.  MultiClass takes the labels Y [B, 1] and one latent
        GP per class.  `device_arrays=True` leaves the gradients of Z, q_mu and q_sqrt as device tensors."""
        if isinstance(self.kernel, MultioutputKernel):
            raise NotImplementedError("the SVGP device gradient covers single-output kernels")
        lik = self.likelihood
        if not isinstance(lik, (Gaussian, Bernoulli, Poisson, StudentT, MultiClass)):
            raise NotImplementedError("the SVGP device gradient covers the Gaussian, Bernoulli, Poisson, StudentT and "
                                      "MultiClass likelihoods")
        if not isinstance(self.mean_function, (Zero, Constant, Linear)):
            raise NotImplementedError("the SVGP device gradient covers the Zero, Constant and Linear mean functions")
        lib = _lib.load()
        X, Y = (ops.to_device(d) for d in data)
        B, D = X.shape
        P = self.num_latent_gps
        mX = self._mean_values(X, Y)
        dc = _lib.GPK_F64
        iv = self.inducing_variable
        Z = ops.to_device(iv.Z)
        M = Z.shape[0]
        # out[4]: the gradient of the likelihood's parameter
        par = lik.variance if isinstance(lik, Gaussian) else (lik.scale if isinstance(lik, StudentT) else (
            lik.invlink.epsilon if isinstance(lik, MultiClass) else None))
        scalars = {par: 4} if isinstance(par, Parameter) else {}

        def layout():
            return (lib.gpk_svgp_elbo_grad_ws(B, M, P, ctypes.byref(lik._lik_desc()), dc),
                    lib.gpk_svgp_elbo_grad_dm(B, M, P, dc))

        def call(kernel, out, n_out, grads, ws):
            q_mu, q_sqrt = ops.to_device(self.q_mu), ops.to_device(self.q_sqrt)
            dZ, dq_mu, dq_sqrt = (ops._p(g) for g in grads)
            return lib.gpk_svgp_elbo_grad(*kernel, ops._p(X), B, ops._ld(X), D, ops._p(Y), ops._p(mX), P, ops._p(Z), M,
                                          ops._ld(Z), ops._p(q_mu), ops._p(q_sqrt), int(self.q_diag), int(self.whiten),
                                          ctypes.byref(lik._lik_desc()), self._scale(data, None),
                                          config.default_jitter(), dc, ops._p(out), n_out, dZ, dq_mu, dq_sqrt,
                                          ops._p(ws), ops._stream())

        return self._device_value_and_grad(X, P, layout=layout, n_head=5, info_index=3, scalars=scalars,
                                           arrays=(iv.Z, self.q_mu, self.q_sqrt), call=call, entry="gpk_svgp_elbo_grad",
                                           device_arrays=device_arrays)

    _objective_and_grad = elbo_and_grad

    def _mean_values(self, X, Y):
        """Checks the targets Y against the likelihood and returns m(X) [B, P] (None for a Zero mean): the device entries
        take Y raw and m(X) apart, which shifts fmean."""
        P, lik = self.num_latent_gps, self.likelihood
        if isinstance(lik, MultiClass):
            if Y.shape[1] != 1:
                raise ValueError(f"MultiClass takes the labels as Y [B, 1]; Y has {Y.shape[1]} columns")
            if P != lik.num_classes:
                raise ValueError(f"MultiClass needs one latent GP per class: the model has {P} latent GPs and the "
                                 f"likelihood {lik.num_classes} classes")
        elif Y.shape[1] != P:
            raise ValueError(f"Y has {Y.shape[1]} columns but the model has {P} latent GPs")
        if isinstance(self.mean_function, Zero):
            return None
        mX = ops.to_device(self.mean_function(X))
        if mX.shape[1] != P:  # one mean column shared by the latents
            mX = mX.expand(X.shape[0], P).contiguous()
        return mX

    def solve_columns(self, data, cols: Tuple[int, int]):
        """Stage 1 of the column-sharded evaluation: Kuu, chol(Kuu) and A[:, c0:c1] = Lm^-1 Kuf[:, c0:c1] for this rank's
        minibatch columns (conditionals/util.py:125).  Returns the workspace matrix A [M, B] (a strided view; only the
        columns [c0, c1) are valid) for the all-gather of sharding.svgp_elbo_latent_sharded."""
        self._fused(data, None, 1, cols)
        lib = _lib.load()
        X = data[0]
        B, M, P = int(X.shape[0]), int(self.inducing_variable.num_inducing), self.num_latent_gps
        ld = ctypes.c_int64(0)
        dt = ops.torch_dtype()
        off = lib.gpk_svgp_elbo_A(B, M, P, ops.dtype_code(ops.to_device(X)), ctypes.byref(ld))
        es = 8 if dt == ops.torch().float64 else 4
        flat = self._ws[off:off + M * ld.value * es].view(dt)
        return flat.view(M, ld.value)[:, :B]

    def elbo_from_columns(self, data, latent_range: Tuple[int, int]):
        """Stage 2: the share of latents [p0, p1) with A complete in the workspace (after the all-gather)."""
        return self._fused(data, latent_range, 2, None)[0]

    def elbo_unfused(self, data):
        """svgp.py:166-181 composed from the public operators (prior_kl, predict_f,
        variational_expectations) exactly as the reference composes them; device fp64 scalar."""
        X, Y = (ops.to_device(d) for d in data)
        kl = self.prior_kl()
        f_mean, f_var = self.predict_f(X, full_cov=False, full_output_cov=False)
        var_exp = self.likelihood.variational_expectations(X, f_mean, f_var, Y)
        scale = 1.0 if self.num_data is None else float(self.num_data) / X.shape[0]
        out = ops.copy(var_exp)
        ops.axpby(-1.0, kl, scale, out)
        return out[0]

    def posterior(self, precompute_cache=posteriors.PrecomputeCacheType.TENSOR) -> posteriors.BasePosterior:
        """svgp.py:210-240."""
        return posteriors.create_posterior(self.kernel, self.inducing_variable, self.q_mu, self.q_sqrt,
                                           whiten=self.whiten, mean_function=self.mean_function,
                                           precompute_cache=precompute_cache)

    def predict_f(self, Xnew, full_cov: bool = False, full_output_cov: bool = False):  # svgp.py:243-255
        return self.posterior(posteriors.PrecomputeCacheType.NOCACHE).fused_predict_f(
            Xnew, full_cov=full_cov, full_output_cov=full_output_cov)
