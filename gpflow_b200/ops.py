"""Device operators: thin typed wrappers over the C ABI (include/gpk.h).

torch tensors are *containers* (allocation, lifetime, stream handle); every arithmetic step is a
libgpk kernel.  All matrices are 2-D row-major; a tensor's row stride is its leading dimension."""
from __future__ import annotations

import ctypes
from ctypes import c_void_p
from typing import Any, Optional, Sequence, Tuple

import numpy as np

from . import _lib, config
from ._lib import GPK_F32, GPK_F64, check


def torch():
    import torch as _t

    return _t


def require_cuda():
    t = torch()
    if not t.cuda.is_available():
        raise _lib.GpkError("gpflow_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    return t.device("cuda", t.cuda.current_device())


def dtype_code(t) -> int:
    T = torch()
    if t.dtype == T.float64:
        return GPK_F64
    if t.dtype == T.float32:
        return GPK_F32
    raise TypeError(f"unsupported dtype {t.dtype}; the path computes in float32 or float64")


def torch_dtype(np_dtype=None):
    T = torch()
    d = np.dtype(np_dtype if np_dtype is not None else config.default_float())
    return T.float64 if d == np.float64 else T.float32


def to_device(x: Any, dtype=None):
    """Host/any -> contiguous device tensor of the default float (gpflow/models/util.py:91-107)."""
    T = torch()
    dev = require_cuda()
    td = torch_dtype(dtype)
    if isinstance(x, T.Tensor):
        if x.device == dev and x.dtype == td and x.is_contiguous():
            return x
        return x.to(device=dev, dtype=td).contiguous()
    if hasattr(x, "device") and hasattr(x, "numpy") and not isinstance(x, np.ndarray):  # Parameter
        return x.device(dev, np.float64 if td == T.float64 else np.float32)
    arr = np.ascontiguousarray(np.asarray(x, dtype=np.float64 if td == T.float64 else np.float32))
    return T.from_numpy(arr).to(dev, non_blocking=False)


def empty(shape: Sequence[int], like=None, dtype=None):
    T = torch()
    if like is not None:
        return T.empty(tuple(shape), dtype=like.dtype, device=like.device)
    return T.empty(tuple(shape), dtype=torch_dtype(dtype), device=require_cuda())


def _p(t) -> c_void_p:
    return c_void_p(t.data_ptr()) if t is not None else c_void_p(None)


def _stream() -> c_void_p:
    return c_void_p(torch().cuda.current_stream().cuda_stream)


def _ld(t) -> int:
    if t.dim() == 1:
        return t.shape[0]
    if t.stride(-1) != 1 and t.shape[-1] > 1:  # a single column's stride is never used (x[:, None] has stride 0)
        raise ValueError("matrix must be row-major with unit column stride")
    return t.stride(-2) if t.shape[-2] > 1 else max(t.shape[-1], t.stride(-2))


def scratch_bytes(nbytes: int):
    return torch().empty((max(int(nbytes), 16),), dtype=torch().uint8, device=require_cuda())


def zeros_scalar(n: int = 1):
    """fp64 device scalars for reductions (zeroed by a memset kernel-free path)."""
    t = torch().empty((n,), dtype=torch().float64, device=require_cuda())
    fill(t.view(1, n), 0.0)
    return t


# ---- kernel expressions -------------------------------------------------------------------------
def kbuild(desc, X, X2=None, *, uplo: int = _lib.GPK_FULL, diag_scalar: float = 0.0, diag_vec=None, out=None):
    """K = kernel(X, X2) [+ diag]; `desc` = (nodes, n_nodes, dims, ard) from kernels.compile_kernel."""
    nodes, n_nodes, dims, ard = desc
    N, D = X.shape
    N2 = N if X2 is None else X2.shape[0]
    if out is None:
        out = empty((N, N2), like=X)
    check(_lib.load().gpk_kbuild(nodes, n_nodes, dims, ard, _p(X), N, _ld(X), _p(X2), N2,
                                 _ld(X2) if X2 is not None else 0, D, _p(out), _ld(out), dtype_code(X), uplo,
                                 float(diag_scalar), _p(diag_vec), _stream()), "gpk_kbuild")
    return out


def kdiag(desc, X, out=None):
    nodes, n_nodes, dims, ard = desc
    N, D = X.shape
    if out is None:
        out = empty((N,), like=X)
    check(_lib.load().gpk_kdiag(nodes, n_nodes, dims, ard, _p(X), N, _ld(X), D, _p(out), dtype_code(X), _stream()),
          "gpk_kdiag")
    return out


# ---- dense linear algebra -------------------------------------------------------------------------
class NonPositiveDefiniteError(_lib.GpkError):
    """Analogue of TF's InvalidArgumentError 'Cholesky decomposition was not successful'."""


_OBJECTIVE_CLS = None


def objective(out, value_idx: int = 0, info_idx: Optional[int] = None, info_tensor=None):
    """Scalar result of a fused objective: the 0-d DEVICE tensor out[value_idx] (no synchronisation), typed so that
    reading it on the host -- float(v), v.item(), v.cpu() -- also reads out[info_idx] in the same transfer and raises
    NonPositiveDefiniteError when the factorisation inside the evaluation met a non-positive pivot, as
    tf.linalg.cholesky raises InvalidArgumentError in the reference (gpflow/models/gpr.py:102).  `v.unchecked()`
    returns the plain tensor."""
    global _OBJECTIVE_CLS
    T = torch()
    if _OBJECTIVE_CLS is None:
        class Objective(T.Tensor):
            __torch_function__ = T._C._disabled_torch_function_impl  # ops on it yield plain tensors

            def unchecked(self):
                return self.as_subclass(T.Tensor)

            def _host_value(self):
                src = getattr(self, "_gpk_out", None)
                if src is None:
                    return T.Tensor.item(self.as_subclass(T.Tensor))
                out_, vi, ii, it = src
                h = out_.cpu()
                piv = int(h[ii]) if ii is not None else (int(it.cpu()[0]) if it is not None else 0)
                if piv != 0:
                    raise NonPositiveDefiniteError(f"Cholesky decomposition was not successful (pivot {piv} <= 0)")
                return float(h[vi])

            def item(self):
                return self._host_value()

            def __float__(self):
                return float(self._host_value())

            def cpu(self, *a, **k):
                self._host_value()
                return self.as_subclass(T.Tensor).cpu(*a, **k)

        _OBJECTIVE_CLS = Objective
    v = out[value_idx].as_subclass(_OBJECTIVE_CLS)
    v._gpk_out = (out, value_idx, info_idx, info_tensor)
    return v


def potrf(A, n: Optional[int] = None, *, check_info: bool = True):
    """In-place lower Cholesky of the leading n x n block of A [rows, >=n]; returns (A, dinv)."""
    rows = A.shape[0]
    n = A.shape[1] if n is None else n
    lib = _lib.load()
    dc = dtype_code(A)
    ws = scratch_bytes(lib.gpk_potrf_ws(n, rows, dc))
    info = torch().empty((1,), dtype=torch().int32, device=A.device)
    check(lib.gpk_potrf(_p(A), n, rows, _ld(A), dc, _p(info), _p(ws), _stream()), "gpk_potrf")
    if check_info:
        i = int(info.item())
        if i != 0:
            raise NonPositiveDefiniteError(f"Cholesky decomposition was not successful (pivot {i} <= 0)")
    return A, ws


def potrf_batched(A, *, check_info: bool = True):
    """In-place lower Cholesky of a batch A [L, n, n] (multi-output Kuu stacks); n <= 128 runs as ONE launch."""
    Lb, n = A.shape[0], A.shape[-1]
    lib = _lib.load()
    dc = dtype_code(A)
    ws = scratch_bytes(lib.gpk_potrf_batched_ws(n, Lb, dc))
    info = torch().empty((Lb,), dtype=torch().int32, device=A.device)
    check(lib.gpk_potrf_batched(_p(A), n, A.stride(-2), A.stride(0), Lb, dc, _p(info), _p(ws), _stream()), "gpk_potrf_batched")
    if check_info:
        bad = info.cpu().numpy()
        if bad.any():
            b = int(bad.nonzero()[0][0])
            raise NonPositiveDefiniteError(f"Cholesky decomposition was not successful (matrix {b}, pivot {int(bad[b])} <= 0)")
    return A, ws


def cholesky(K):
    """tf.linalg.cholesky semantics: new tensor, strict upper triangle zero."""
    L = empty(K.shape, like=K)
    axpby(1.0, K, 0.0, L)
    _, dinv = potrf(L)
    tril_(L)
    return L, dinv


def trsm(L, B, *, trans: bool = False, dinv=None):
    """B <- L^-1 B or L^-T B, in place; returns B."""
    lib = _lib.load()
    n = L.shape[0]
    dc = dtype_code(L)
    ws = None if dinv is not None else scratch_bytes(lib.gpk_trsm_ws(n, dc))
    nrhs = B.shape[1] if B.dim() == 2 else 1
    check(lib.gpk_trsm(1 if trans else 0, _p(L), n, _ld(L), _p(B), nrhs, _ld(B) if B.dim() == 2 else 1, dc,
                       _p(dinv), _p(ws), _stream()), "gpk_trsm")
    return B


def gemm(A, B, *, transa: bool = False, transb: bool = False, alpha: float = 1.0, beta: float = 0.0, out=None,
         flags: int = 0):
    m = A.shape[1] if transa else A.shape[0]
    k = A.shape[0] if transa else A.shape[1]
    n = B.shape[0] if transb else B.shape[1]
    kb = B.shape[1] if transb else B.shape[0]
    if k != kb:
        raise ValueError(f"gemm: inner dimensions differ ({k} vs {kb})")
    if out is None:
        # the column-sum-of-squares epilogue ACCUMULATES (atomicAdd) into its output: start from zero
        out = full((n,), 0.0, like=A) if flags & _lib.GPK_GEMM_COLSUMSQ else empty((m, n), like=A)
    ldc = 0 if flags & _lib.GPK_GEMM_COLSUMSQ else _ld(out)
    check(_lib.load().gpk_gemm(int(transa), int(transb), m, n, k, float(alpha), _p(A), _ld(A), _p(B), _ld(B),
                               float(beta), _p(out), ldc, dtype_code(A), flags, _stream()), "gpk_gemm")
    return out


# ---- reductions ------------------------------------------------------------------------------------
def colsumsq(A, *, scale: float = 1.0, out=None, accumulate: bool = False):
    m, n = A.shape
    if out is None:
        out = empty((n,), like=A)
        accumulate = False
    check(_lib.load().gpk_colsumsq(_p(A), m, n, _ld(A), float(scale), int(accumulate), _p(out), dtype_code(A),
                                   _stream()), "gpk_colsumsq")
    return out


SUM, SUMSQ, SUMLOG, SUMLOGSQ = 0, 1, 2, 3


def reduce(f: int, x, n: int, inc: int = 1, *, scale: float = 1.0, out=None, accumulate: bool = False):
    if out is None:
        out = torch().empty((1,), dtype=torch().float64, device=x.device)
        accumulate = False
    check(_lib.load().gpk_reduce(f, _p(x), n, inc, float(scale), int(accumulate), _p(out), dtype_code(x), _stream()),
          "gpk_reduce")
    return out


def tril_sumsq(A, *, scale: float = 1.0, out=None, accumulate: bool = False):
    """sum over batch of squares of the lower triangles of A [..., n, n]."""
    n = A.shape[-1]
    batch = 1 if A.dim() == 2 else A.shape[0]
    if out is None:
        out = torch().empty((1,), dtype=torch().float64, device=A.device)
        accumulate = False
    check(_lib.load().gpk_tril_sumsq(_p(A), n, n, n * n, batch, float(scale), int(accumulate), _p(out),
                                     dtype_code(A), _stream()), "gpk_tril_sumsq")
    return out


# ---- elementwise -------------------------------------------------------------------------------------
def axpby(a: float, X, b: float, Y):
    """Y = a X + b Y (2-D or 1-D).  X [N, 1] against Y [N, P] broadcasts along the columns (the reference's
    `Y - mean_function(X)` with a single-column mean, gpflow/models/gpr.py:98); any other shape mismatch raises."""
    if tuple(X.shape) != tuple(Y.shape):
        if X.dim() == 2 and Y.dim() == 2 and X.shape[0] == Y.shape[0] and X.shape[1] == 1:
            for p in range(Y.shape[1]):
                axpby(a, X, b, Y[:, p:p + 1])
            return Y
        if X.numel() != Y.numel() or (X.dim() > 1 and Y.dim() > 1):
            raise ValueError(f"axpby: shapes {tuple(X.shape)} and {tuple(Y.shape)} do not match")
    if X.dim() <= 1:
        m, n, ldx, ldy = 1, X.numel(), X.numel(), Y.numel()
    else:
        (m, n), ldx, ldy = X.shape, _ld(X), _ld(Y)
    check(_lib.load().gpk_axpby(m, n, float(a), _p(X), ldx, float(b), _p(Y), ldy, dtype_code(X), _stream()),
          "gpk_axpby")
    return Y


def hadamard_(Y, X):
    """Y *= X elementwise (2-D, same shape)."""
    if tuple(X.shape) != tuple(Y.shape) or X.dim() != 2:
        raise ValueError(f"hadamard_: shapes {tuple(X.shape)} and {tuple(Y.shape)} do not match")
    check(_lib.load().gpk_hadamard(X.shape[0], X.shape[1], _p(X), _ld(X), _p(Y), _ld(Y), dtype_code(X), _stream()),
          "gpk_hadamard")
    return Y


def copy(X):
    Y = empty(X.shape, like=X)
    return axpby(1.0, X, 0.0, Y)


def scale_cols_(A, s, invert: bool = False):
    check(_lib.load().gpk_scale_cols(_p(A), A.shape[0], A.shape[1], _ld(A), _p(s), int(invert), dtype_code(A),
                                     _stream()), "gpk_scale_cols")
    return A


def scale_rows_(A, s, invert: bool = False):
    check(_lib.load().gpk_scale_rows(_p(A), A.shape[0], A.shape[1], _ld(A), _p(s), int(invert), dtype_code(A),
                                     _stream()), "gpk_scale_rows")
    return A


def add_diag_(A, scalar: float = 0.0, vec=None):
    check(_lib.load().gpk_add_diag(_p(A), A.shape[0], _ld(A), float(scalar), _p(vec), dtype_code(A), _stream()),
          "gpk_add_diag")
    return A


def fill(A, value: float):
    if A.dim() > 2:
        if not A.is_contiguous():
            raise ValueError("fill: tensors with more than two dimensions must be contiguous")
        fill(A.view(-1, A.shape[-1]), value)
        return A
    if A.dim() <= 1:
        m, n, ld = 1, A.numel(), A.numel()
    else:
        (m, n), ld = A.shape, _ld(A)
    check(_lib.load().gpk_fill(_p(A), m, n, ld, float(value), dtype_code(A), _stream()), "gpk_fill")
    return A


def full(shape, value: float, like=None, dtype=None):
    return fill(empty(shape, like=like, dtype=dtype), value)


def tril_(A):
    n = A.shape[-1]
    batch = 1 if A.dim() == 2 else A.shape[0]
    check(_lib.load().gpk_tril(_p(A), n, n if A.dim() == 3 else _ld(A), n * n, batch, dtype_code(A), _stream()),
          "gpk_tril")
    return A


def transpose(A, out=None):
    m, n = A.shape
    if out is None:
        out = empty((n, m), like=A)
    check(_lib.load().gpk_transpose(_p(A), m, n, _ld(A), _p(out), _ld(out), dtype_code(A), _stream()),
          "gpk_transpose")
    return out


def lik_varexp_sum(desc, Fmu, Fvar, Y, *, scale: float = 1.0):
    """scale * sum_{n,p} E_q[log p(Y | f)] of the likelihood `desc` (_lib.LikDesc) -> device fp64 [1]."""
    Bn, P = Fmu.shape
    out = torch().empty((1,), dtype=torch().float64, device=Fmu.device)
    check(_lib.load().gpk_lik_varexp_sum(ctypes.byref(desc), _p(Fmu), _p(Fvar), _p(Y), Bn, P, float(scale), 0,
                                         _p(out), dtype_code(Fmu), _stream()), "gpk_lik_varexp_sum")
    return out


def lik_predict_mean_and_var(desc, Fmu, Fvar):
    """The predictive mean and variance of y under the likelihood `desc` -> two device tensors [N, P] ([N, 1] for the
    heteroskedastic likelihood, whose two latents describe one output)."""
    N, P = Fmu.shape
    cols = 1 if desc.type == _lib.LIK_HETEROSKEDASTIC else P
    mean, var = empty((N, cols), like=Fmu), empty((N, cols), like=Fmu)
    check(_lib.load().gpk_lik_predict_mean_and_var(ctypes.byref(desc), _p(Fmu), _p(Fvar), N, P, _p(mean), _p(var),
                                                   dtype_code(Fmu), _stream()), "gpk_lik_predict_mean_and_var")
    return mean, var


def lik_varexp_grad(desc, Fmu, Fvar, Y, *, scale: float = 1.0):
    """The adjoints of scale * sum E_q[log p(Y | f)] under the likelihood `desc` (fp64 device tensors, Fmu and Fvar [B,
    P]) -> (R [B, P] = d/dFmu, W [B, P] = d/dFvar, dpar [1] = d/d(likelihood parameter), 0 if it has none)."""
    T = torch()
    if any(t.dtype != T.float64 for t in (Fmu, Fvar, Y)):
        raise ValueError("lik_varexp_grad computes in float64: Fmu, Fvar and Y must be float64")
    Bn, P = Fmu.shape
    R, Wt = empty((Bn, P), like=Fmu), empty((P, Bn), like=Fmu)
    dpar = T.zeros((1,), dtype=T.float64, device=Fmu.device)
    fvar_t = Fvar.t().contiguous()
    check(_lib.load().gpk_lik_varexp_grad(ctypes.byref(desc), _p(Fmu), _p(fvar_t), _p(Y), Bn, P, float(scale), _p(R),
                                          _p(Wt), _p(dpar), _stream()), "gpk_lik_varexp_grad")
    return R, Wt.t(), dpar


def lik_predict_log_density(desc, Fmu, Fvar, Y):
    """out[n] = sum_p log E_q[p(Y[n,p] | f)] under the likelihood `desc` -> device vector [N]."""
    N, P = Fmu.shape
    out = torch().empty((N,), dtype=Fmu.dtype, device=Fmu.device)
    check(_lib.load().gpk_lik_predict_log_density(ctypes.byref(desc), _p(Fmu), _p(Fvar), _p(Y), N, P, _p(out),
                                                  dtype_code(Fmu), _stream()), "gpk_lik_predict_log_density")
    return out
