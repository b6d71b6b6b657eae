"""Conjugate Gradient Lower Bound (mirrors gpflow/models/cglb.py:36-295; Artemev, Burt & van der Wilk 2021).

SGPR's Nystrom approximation serves only as the preconditioner of conjugate gradients on the exact K^ = K(X, X) + s I;
the bound then lies within `cg_tolerance` of the quadratic term of the exact log marginal likelihood, at O(N^2) per CG
step and without factorising K^.  The device path never forms K^ either: every product with it is the matrix-free
`gpk_kmv` (csrc/kmv.cu), and the CG loop runs on the device (`gpk_cglb_elbo`), so memory stays O(N (M + P) + M^2).

The reference's module-level `NystromPreconditioner` and `cglb_conjugate_gradient` take a materialised K; they are not
mirrored here, since the model never builds K and a second, dense path would go unused.

`elbo_and_grad` gives the bound and its gradient in one device call (`gpk_cglb_elbo_grad`): every kernel parameter of
a fused expression, the noise variance, Z, the Constant / Linear mean-function parameters, and v when it is trainable.
The N x N part of the gradient is reduced tile by tile from the rank <= 2P weight 1/2 (v v^T + z v^T + v z^T), so it
too stays O(N P) in memory.  Scipy, Adam and `training_loop` train the model through it."""
from __future__ import annotations

from typing import Optional

import numpy as np

from .. import _lib, config, ops, posteriors
from ..base import Parameter
from ..kernels import compile_kernel
from ..mean_functions import Zero
from .model import centred_targets
from .sgpr import SGPR


class CGLB(SGPR):
    def __init__(self, data, *args, cg_tolerance: float = 1.0, max_cg_iters: int = 100, restart_cg_iters: int = 40,
                 v_grad_optimization: bool = False, **kwargs):
        """cglb.py:60-79.  `v_grad_optimization=False`: every evaluation of the bound runs CG from the stored auxiliary
        vector and stores the result; True: no CG runs and the vector is an ordinary trainable parameter."""
        super().__init__(data, *args, **kwargs)
        n, b = self.data[1].shape
        self._v = Parameter(np.zeros((b, n), dtype=np.float64), trainable=v_grad_optimization)
        self._cg_tolerance = cg_tolerance
        self._max_cg_iters = max_cg_iters
        self._restart_cg_iters = restart_cg_iters

    @property
    def aux_vec(self) -> Parameter:
        """The auxiliary vector v [P, N] of the quadratic term (cglb.py:81-86)."""
        return self._v

    def _check(self, run_cg: bool) -> None:
        X, Y = self.data
        if ops.dtype_code(X) != _lib.GPK_F64 or ops.dtype_code(Y) != _lib.GPK_F64:
            raise NotImplementedError("CGLB on the device computes in float64")
        if not self.kernel.is_fusable():
            raise NotImplementedError("CGLB needs a fused kernel expression: the matrix-free product evaluates K "
                                      "element by element and cannot take materialised kernel leaves")
        if getattr(self.likelihood, "heteroskedastic", False):
            raise NotImplementedError("CGLB covers Gaussian(variance=...) with a constant noise variance")
        if any(p.prior is not None for p in self.parameters):
            raise NotImplementedError("CGLB: parameter priors are outside the hot path")
        if run_cg and Y.shape[1] != 1:
            raise ValueError(f"CGLB runs conjugate gradients for one output only (P = {Y.shape[1]}): the reference's "
                             "CG step divides a [P] step size into a [P, N] direction, which does not broadcast for "
                             "P > 1; use v_grad_optimization=True or cg_tolerance=None")

    def _bound(self, v, run_cg: bool, cg_tolerance: float):
        """One gpk_cglb_elbo call on the device vector `v` [P, N] (overwritten with the CG result when run_cg);
        returns the device vector {elbo, const, logdet, quad, lb, r^T Q^-1 r, cg_iters, info}."""
        self._check(run_cg)
        lib = _lib.load()
        X, Y = self.data
        N, D = X.shape
        P = Y.shape[1]
        Z = ops.to_device(self.inducing_variable.Z)
        M = Z.shape[0]
        need = lib.gpk_cglb_elbo_ws(N, M, P)
        ws = getattr(self, "_cglb_ws", None)
        if ws is None or ws.numel() < need or ws.device != X.device:
            ws = self._cglb_ws = ops.scratch_bytes(need)
        T = ops.torch()
        out = T.empty((8,), dtype=T.float64, device=X.device)
        Yc = centred_targets(self.mean_function, X, Y).contiguous()
        _lib.check(lib.gpk_cglb_elbo(*compile_kernel(self.kernel, D), ops._p(X), N, ops._ld(X), D, ops._p(Yc), P,
                                     ops._p(Z), M, ops._ld(Z), self.likelihood._variance_value(),
                                     config.default_jitter(), ops._p(v), 1 if run_cg else 0, float(cg_tolerance),
                                     int(self._max_cg_iters), int(self._restart_cg_iters), ops._p(out), ops._p(ws),
                                     ops._stream()), "gpk_cglb_elbo")
        return out

    def elbo(self):
        """cglb.py:83-160 in one call; device fp64 scalar.  Without v_grad_optimization, CG runs from the stored v and
        the result is written back to the parameter's device mirror (cglb.py:155-156); it never travels to the host."""
        X, _ = self.data
        run_cg = not self._v.trainable
        v = self._v.device(X.device)
        self._last = self._bound(v, run_cg, self._cg_tolerance)
        if run_cg:
            self._v.device_updated(v)
        return ops.objective(self._last, 0, 7)

    def cg_iterations(self) -> int:
        """The number of CG steps the last evaluation of the bound ran (one small device->host read)."""
        if self._last is None:
            self.elbo()
        return int(self._last[6].item())

    def elbo_and_grad(self, *, device_arrays: bool = False):
        """Value and gradient of the bound in ONE device call (gpk_cglb_elbo_grad), the backward pass TensorFlow autodiff
        supplies to cglb.py:83-160: (elbo, grads), `elbo` as elbo() and `grads` {Parameter: dF/d(constrained value)}
        for every kernel parameter, the likelihood variance, the inducing points Z, the Constant / Linear mean-function
        parameters and, when it is trainable, the auxiliary vector.  Without v_grad_optimization CG runs first and v,
        stored as in elbo(), is held fixed (the reference's stop_gradient).  `device_arrays=True` leaves the gradients
        of Z and v device tensors."""
        lib = _lib.load()
        X, Y = self.data
        N, D = X.shape
        P = Y.shape[1]
        run_cg = not self._v.trainable
        self._check(run_cg)
        iv = self.inducing_variable
        Z = ops.to_device(iv.Z)
        M = Z.shape[0]
        v = self._v.device(X.device)

        def call(kernel, out, n_out, grads, ws):
            Yc = centred_targets(self.mean_function, X, Y).contiguous()
            status = lib.gpk_cglb_elbo_grad(*kernel, ops._p(X), N, ops._ld(X), D, ops._p(Yc), P, ops._p(Z), M,
                                            ops._ld(Z), self.likelihood._variance_value(), config.default_jitter(),
                                            ops._p(v), 1 if run_cg else 0, float(self._cg_tolerance),
                                            int(self._max_cg_iters), int(self._restart_cg_iters), ops._p(out), n_out,
                                            ops._p(grads[0]), ops._p(grads[1]) if len(grads) > 1 else None,
                                            ops._p(ws), ops._stream())
            if status == 0:
                self._last = out
                if run_cg:
                    self._v.device_updated(v)
            return status

        return self._device_value_and_grad(
            X, P, layout=lambda: (lib.gpk_cglb_elbo_grad_ws(N, M, P), lib.gpk_cglb_elbo_grad_dm(N, M, P)),
            n_head=9, info_index=7, scalars={self.likelihood.variance: 8},
            arrays=(iv.Z,) if run_cg else (iv.Z, self._v), call=call, entry="gpk_cglb_elbo_grad",
            device_arrays=device_arrays)

    _objective_and_grad = elbo_and_grad

    def _kmv(self, Xa, V, diag: float, X2=None):
        """(K(Xa, X2) + diag I) V on the device, matrix-free (gpk_kmv); X2 = None means X2 = Xa."""
        lib = _lib.load()
        N, D = Xa.shape
        P = V.shape[1]
        N2 = N if X2 is None else X2.shape[0]
        T = ops.torch()
        out = T.empty((N, P), dtype=T.float64, device=Xa.device)
        ws = ops.scratch_bytes(lib.gpk_kmv_ws(N, N2, P))
        _lib.check(lib.gpk_kmv(*compile_kernel(self.kernel, D), ops._p(Xa), N, ops._ld(Xa),
                               None if X2 is None else ops._p(X2), N2, ops._ld(Xa) if X2 is None else ops._ld(X2), D,
                               ops._p(V), P, ops._ld(V), diag, ops._p(out), P, ops._p(ws), ops._stream()), "gpk_kmv")
        return out

    def predict_f(self, Xnew, full_cov: bool = False, full_output_cov: bool = False,
                  cg_tolerance: Optional[float] = 1e-3):
        """cglb.py:162-240: mean = K(Xnew, X) v^T + the SGPR mean of the residual e - K^ v^T, plus m(Xnew); SGPR's
        variance.  With a tolerance, CG runs from the stored v to that tolerance and the result is NOT stored; None
        uses the stored v."""
        if full_output_cov:
            raise NotImplementedError("CGLB.predict_f does not support full_output_cov=True")
        X, Y = self.data
        self._check(cg_tolerance is not None)
        v = self._v.device(X.device)
        if cg_tolerance is not None:
            v = v.clone()
            self._bound(v, True, cg_tolerance)
        Xnew = ops.to_device(Xnew)
        Vt = ops.transpose(v)                                            # [N, P]
        cg_mean = self._kmv(Xnew, Vt, 0.0, X2=X)                         # K(Xnew, X) v^T
        res = centred_targets(self.mean_function, X, Y)
        res = ops.axpby(-1.0, self._kmv(X, Vt, self.likelihood._variance_value()), 1.0, ops.copy(res))
        post = posteriors.SGPRPosterior(kernel=self.kernel, data=(X, res), inducing_variable=self.inducing_variable,
                                        likelihood=self.likelihood, num_latent_gps=self.num_latent_gps,
                                        mean_function=Zero(output_dim=self.num_latent_gps),
                                        precompute_cache=None)
        mean, var = post.fused_predict_f(Xnew, full_cov=full_cov)
        ops.axpby(1.0, cg_mean, 1.0, mean)
        if not isinstance(self.mean_function, Zero):
            ops.axpby(1.0, self.mean_function(Xnew), 1.0, mean)
        return mean, var

    def predict_y(self, Xnew, full_cov: bool = False, full_output_cov: bool = False,
                  cg_tolerance: Optional[float] = 1e-3):  # cglb.py:242-263
        if full_cov or full_output_cov:
            raise NotImplementedError("The predict_y method currently supports only the argument values "
                                      "full_cov=False and full_output_cov=False")
        Xnew = ops.to_device(Xnew)
        f_mean, f_var = self.predict_f(Xnew, cg_tolerance=cg_tolerance)
        return self.likelihood.predict_mean_and_var(Xnew, f_mean, f_var)

    def predict_log_density(self, data, full_cov: bool = False, full_output_cov: bool = False,
                            cg_tolerance: Optional[float] = 1e-3):  # cglb.py:265-287
        if full_cov or full_output_cov:
            raise NotImplementedError("The predict_log_density method currently supports only the argument values "
                                      "full_cov=False and full_output_cov=False")
        X, Y = data
        X = ops.to_device(X)
        f_mean, f_var = self.predict_f(X, cg_tolerance=cg_tolerance)
        return self.likelihood.predict_log_density(X, f_mean, f_var, Y)
