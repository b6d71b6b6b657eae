"""Kernel plugin API (mirrors gpflow/kernels/base.py:29-314).

A kernel is a Python object tree exactly as in the reference; evaluation does not materialise one
matrix per node: `compile_kernel` flattens the tree into `gpk_knode` records and ONE fused CUDA
pass (`gpk_kbuild`, csrc/kbuild.cu) evaluates leaves, Sum and Product per output element."""
from __future__ import annotations

import abc
import ctypes
from typing import Any, List, Optional, Sequence, Tuple, Union

import numpy as np

from .. import _lib, ops
from ..base import Module, Parameter

ActiveDims = Union[None, slice, Sequence[int]]


class Kernel(Module, metaclass=abc.ABCMeta):
    def __init__(self, active_dims: ActiveDims = None, name: Optional[str] = None) -> None:
        self.name = name
        self._active_dims = self._normalize_active_dims(active_dims)

    @staticmethod
    def _normalize_active_dims(value: ActiveDims):  # base.py:47-53
        if value is None:
            return slice(None, None, None)
        if isinstance(value, slice):
            return value
        return np.array(value, dtype=int)

    @property
    def active_dims(self):
        return self._active_dims

    @active_dims.setter
    def active_dims(self, value: ActiveDims) -> None:
        self._active_dims = self._normalize_active_dims(value)

    def on_separate_dims(self, other: "Kernel") -> bool:  # base.py:63-77
        if isinstance(self.active_dims, slice) or isinstance(other.active_dims, slice):
            return False
        this_dims = self.active_dims.reshape(-1, 1)
        other_dims = other.active_dims.reshape(1, -1)
        return not np.any(this_dims == other_dims)

    def _validate_ard_active_dims(self, ard_parameter: Any) -> None:  # base.py:152-168
        arr = np.asarray(ard_parameter.numpy() if isinstance(ard_parameter, Parameter) else ard_parameter)
        if isinstance(self.active_dims, slice):
            return
        if arr.ndim > 0 and arr.shape[0] != len(self.active_dims):
            raise ValueError(
                f"Size of `active_dims` {self.active_dims} does not match size of ard parameter ({arr.shape[0]})"
            )

    def _resolved_dims(self, D: int) -> Optional[np.ndarray]:
        """None for 'all columns', else explicit column indices (slice applied to range(D))."""
        ad = self.active_dims
        if isinstance(ad, slice):
            if ad == slice(None, None, None):
                return None
            return np.arange(D)[ad]
        return np.asarray(ad, dtype=int)

    # -- reference surface ------------------------------------------------------------------
    def K(self, X, X2=None):
        """[N, N2] covariance on a device tensor (inputs taken as already sliced is NOT supported by the
        fused builder: leaves always slice their own active_dims, base.py:281-291)."""
        return self(X, X2, full_cov=True)

    def K_diag(self, X):
        return self(X, full_cov=False)

    def __call__(self, X, X2=None, *, full_cov: bool = True, presliced: bool = False):  # base.py:195-214
        if (not full_cov) and (X2 is not None):
            raise ValueError("Ambiguous inputs: `not full_cov` and `X2` are not compatible.")
        if presliced:
            raise NotImplementedError("presliced=True is not supported: the fused builder slices per leaf")
        X = ops.to_device(X)
        X2 = None if X2 is None else ops.to_device(X2)
        if not self.is_fusable():
            # a leaf that is not a function of a Gram term (kernels/materialised.py): children are evaluated one by one
            # and combined with elementwise device ops, as the reference composes them (base.py:281-314)
            return self._materialise(X, X2, full_cov)
        desc = compile_kernel(self, X.shape[-1])
        if not full_cov:
            return ops.kdiag(desc, X)
        return ops.kbuild(desc, X, X2)

    def is_fusable(self) -> bool:
        """True when the whole expression compiles into ONE fused K-build (every leaf has a `gpk_knode` record)."""
        return True

    def _materialise(self, X, X2, full_cov: bool):
        raise NotImplementedError(f"{type(self).__name__} has no materialised evaluation")

    def __add__(self, other: "Kernel") -> "Kernel":
        return Sum([self, other])

    def __mul__(self, other: "Kernel") -> "Kernel":
        return Product([self, other])

    # leaf kernels fill one record
    def _leaf_record(self, D: int) -> dict:
        raise NotImplementedError(f"{type(self).__name__} has no fused K-build record")


class Combination(Kernel):
    """gpflow/kernels/base.py:223-302."""

    _op: int = -1

    def __init__(self, kernels: Sequence[Kernel], name: Optional[str] = None) -> None:
        super().__init__(name=name)
        if not all(isinstance(k, Kernel) for k in kernels):
            raise TypeError("can only combine Kernel instances")
        self.kernels: List[Kernel] = []
        for k in kernels:  # flatten same-class nesting, base.py:246-254
            if isinstance(k, self.__class__):
                self.kernels.extend(k.kernels)
            else:
                self.kernels.append(k)

    def is_fusable(self) -> bool:
        return all(k.is_fusable() for k in self.kernels)

    def _materialise(self, X, X2, full_cov: bool):
        """Sum / Product with at least one materialised child (base.py:305-314): children one by one, fusable runs of
        children still in one fused pass."""
        fus = [k for k in self.kernels if k.is_fusable()]
        parts = [k(X, X2, full_cov=full_cov) if full_cov else k(X, full_cov=False) for k in self.kernels if not k.is_fusable()]
        if fus:
            grp = fus[0] if len(fus) == 1 else self.__class__(fus)
            parts.append(grp(X, X2, full_cov=full_cov) if full_cov else grp(X, full_cov=False))
        acc = parts[0]
        for p in parts[1:]:
            if self._op == _lib.K_SUM:
                ops.axpby(1.0, p, 1.0, acc)
            else:
                ops.hadamard_(acc.view(acc.shape[0], -1), p.view(p.shape[0], -1))
        return acc

    @property
    def on_separate_dimensions(self) -> bool:  # base.py:256-278
        if any(isinstance(k.active_dims, slice) for k in self.kernels):
            return False
        dimlist = [k.active_dims for k in self.kernels]
        for i, di in enumerate(dimlist):
            for dj in dimlist[i + 1:]:
                if np.any(di.reshape(-1, 1) == dj.reshape(1, -1)):
                    return False
        return True


class ReducingCombination(Combination):
    pass


class Sum(ReducingCombination):
    _op = _lib.K_SUM


class Product(ReducingCombination):
    _op = _lib.K_PRODUCT


def kernel_matrix(kernel: Kernel, X, X2=None, *, uplo: int = _lib.GPK_FULL, diag_scalar: float = 0.0, diag_vec=None):
    """kernel(X, X2) [+ diag] on the device: ONE fused K-build when the expression compiles (then `uplo=LOWER` skips the
    tiles above the diagonal), else the materialised evaluation (full matrix) followed by the diagonal shift."""
    X = ops.to_device(X)
    X2 = None if X2 is None else ops.to_device(X2)
    if kernel.is_fusable():
        return ops.kbuild(compile_kernel(kernel, X.shape[-1]), X, X2, uplo=uplo, diag_scalar=diag_scalar, diag_vec=diag_vec)
    K = kernel(X, X2)
    if diag_scalar != 0.0 or diag_vec is not None:
        ops.add_diag_(K, diag_scalar, diag_vec)
    return K


# ------------------------------------------------------------------------------------------------
# expression tree -> gpk_knode[]
# ------------------------------------------------------------------------------------------------
def compile_kernel(kernel: Kernel, D: int) -> Tuple[Any, int, Any, Any]:
    """Flattens `kernel` for inputs with D columns.  Returns (nodes, n_nodes, dims, ard) ctypes arrays
    ready for gpk_kbuild / gpk_kdiag / the fused objectives."""
    records: List[dict] = []
    dims: List[int] = []
    ard: List[float] = []

    def visit(k: Kernel) -> int:
        if isinstance(k, Combination):
            if len(k.kernels) > _lib.GPK_MAX_CHILDREN:
                # split wide combinations into a chain of same-op nodes
                idx = [visit(c) for c in k.kernels]
                while len(idx) > _lib.GPK_MAX_CHILDREN:
                    head, idx = idx[: _lib.GPK_MAX_CHILDREN], idx[_lib.GPK_MAX_CHILDREN:]
                    records.append({"op": k._op, "children": head})
                    idx = [len(records) - 1] + idx
                records.append({"op": k._op, "children": idx})
                return len(records) - 1
            children = [visit(c) for c in k.kernels]
            records.append({"op": k._op, "children": children})
            return len(records) - 1
        rec = k._leaf_record(D)
        d = k._resolved_dims(D)
        rec["n_dims"], rec["dims_off"] = 0, 0
        if d is not None:
            if np.any(d < 0) or np.any(d >= D):
                raise ValueError(f"active_dims {d} out of range for inputs with {D} columns")
            rec["n_dims"], rec["dims_off"] = len(d), len(dims)
            dims.extend(int(v) for v in d)
        a = rec.pop("ard", None)
        rec["n_ard"], rec["ard_off"] = 0, 0
        if a is not None:
            n_act = len(d) if d is not None else D
            if len(a) != n_act:
                raise ValueError(f"Size of ARD parameter ({len(a)}) does not match active dims ({n_act})")
            rec["n_ard"], rec["ard_off"] = len(a), len(ard)
            ard.extend(float(v) for v in a)
        records.append(rec)
        return len(records) - 1

    visit(kernel)
    n = len(records)
    nodes = (_lib.KNode * n)()
    for i, r in enumerate(records):
        nd = nodes[i]
        nd.op = r["op"]
        ch = r.get("children", [])
        nd.n_children = len(ch)
        for j, c in enumerate(ch):
            nd.child[j] = c
        nd.variance = float(r.get("variance", 1.0))
        nd.lengthscale = float(r.get("lengthscale", 1.0))
        nd.alpha = float(r.get("alpha", 1.0))
        nd.n_dims, nd.dims_off = r.get("n_dims", 0), r.get("dims_off", 0)
        nd.n_ard, nd.ard_off = r.get("n_ard", 0), r.get("ard_off", 0)
    dims_arr = (ctypes.c_int32 * max(len(dims), 1))(*dims)
    ard_arr = (ctypes.c_double * max(len(ard), 1))(*ard)
    return nodes, n, dims_arr, ard_arr


def gradient_slots(kernel: Kernel, D: int) -> List[Tuple[Parameter, int, int]]:
    """The gradient slots of gpk_gpr_lml_grad_expr for `kernel` on inputs with D columns: one (Parameter, slot offset,
    count) per leaf parameter, leaves in the node order `compile_kernel` emits (children before parents, left to right).
    Per leaf: stationary: variance, lengthscales (1, or one per ARD entry) [, RationalQuadratic alpha]; Linear: variance
    (1 or per dim); Polynomial: variance, offset (the degree is no Parameter); White / Constant: variance.  The same
    Parameter may appear more than once (`k + k`): its gradient is the sum of its slots.  Kernels without a fused record
    raise NotImplementedError naming the class."""
    from .linears import Linear, Polynomial
    from .statics import Static
    from .stationaries import RationalQuadratic, Stationary

    out: List[Tuple[Parameter, int, int]] = []
    pos = 0

    def add(p: Parameter, n: int) -> None:
        nonlocal pos
        out.append((p, pos, n))
        pos += n

    def visit(k: Kernel) -> None:
        if isinstance(k, (Sum, Product)):
            for c in k.kernels:
                visit(c)
        elif not k.is_fusable():
            raise NotImplementedError(f"{type(k).__name__} has no device gradient (it is not a fused K-build leaf)")
        elif isinstance(k, Stationary):
            add(k.variance, 1)
            add(k.lengthscales, int(np.asarray(k.lengthscales.numpy()).size))
            if isinstance(k, RationalQuadratic):
                add(k.alpha, 1)
        elif isinstance(k, Linear):
            add(k.variance, int(np.asarray(k.variance.numpy()).size))
            if isinstance(k, Polynomial):
                add(k.offset, 1)
        elif isinstance(k, Static):
            add(k.variance, 1)
        else:
            raise NotImplementedError(f"{type(k).__name__} has no device gradient (it is not a fused K-build leaf)")

    visit(kernel)
    return out


def slot_gradients(slots: List[Tuple[Parameter, int, int]], h: np.ndarray) -> dict:
    """{Parameter: gradient} from the slot values `h` (host, slot 0 first) of a gradient_slots map; a Parameter in
    several leaves (k + k) collects the sum of its slots."""
    grads: dict = {}
    for p, off, n in slots:
        g = h[off:off + n].reshape(p.shape).copy()
        grads[p] = grads[p] + g if p in grads else g
    return grads
