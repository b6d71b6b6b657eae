"""Mean functions Zero / Constant / Linear (mirrors gpflow/functions.py:96-126,173-204)."""
from __future__ import annotations

from typing import Any

import numpy as np

from . import config, ops
from .base import Module, Parameter


class MeanFunction(Module):
    def __call__(self, X):
        raise NotImplementedError


class Zero(MeanFunction):
    def __init__(self, output_dim: int = 1) -> None:
        self.output_dim = output_dim

    def __call__(self, X):  # functions.py:201-204
        X = ops.to_device(X)
        return ops.full((X.shape[0], self.output_dim), 0.0, like=X)


class Constant(MeanFunction):
    def __init__(self, c: Any = None) -> None:
        c = np.zeros(1) if c is None else c
        self.c = Parameter(np.atleast_1d(np.asarray(c, dtype=config.default_float())))

    def __call__(self, X):  # functions.py:187-192
        X = ops.to_device(X)
        c = self.c.numpy()
        out = ops.empty((X.shape[0], c.shape[0]), like=X)
        for q in range(c.shape[0]):
            ops.fill(out[:, q:q + 1], float(c[q]))
        return out


class Linear(MeanFunction):
    def __init__(self, A: Any = None, b: Any = None) -> None:
        A = np.ones((1, 1), dtype=config.default_float()) if A is None else A
        b = np.zeros(1, dtype=config.default_float()) if b is None else b
        self.A = Parameter(np.atleast_2d(A))
        self.b = Parameter(np.atleast_1d(b))

    def __call__(self, X):  # functions.py:124-126
        X = ops.to_device(X)
        A = ops.to_device(self.A)
        out = ops.gemm(X, A)
        b = self.b.numpy()
        Q = out.shape[1]
        for q in range(Q):
            bq = float(b[q] if b.shape[0] > 1 else b[0])
            if bq != 0.0:
                col = out[:, q:q + 1]
                ones = ops.full(col.shape, bq, like=out)
                ops.axpby(1.0, ones, 1.0, col)
        return out


def gradients_from_adjoint(m: MeanFunction, X, adj) -> list:
    """[(Parameter, device gradient)] of a Constant / Linear mean function from d objective / d m = `adj` [N, P] (GPR:
    alpha = K^-1 (Y - m); SGPR: (Yc - A'^T v) / s): Constant.c and Linear.b get the column sums of `adj` (summed over P
    when the parameter has one entry), Linear.A gets X^T adj (X^T adj 1 when A has one column).  [] for other mean
    functions."""
    if not isinstance(m, (Constant, Linear)):
        return []
    N, P = adj.shape
    ones_n = ops.full((N, 1), 1.0, like=X)
    colsum = ops.gemm(ones_n, adj, transa=True)                    # [1, P]

    def per_output(p):
        if p.numpy().size == 1 and P > 1:
            return ops.gemm(colsum, ops.full((P, 1), 1.0, like=X))  # [1, 1]
        return colsum
    if isinstance(m, Constant):
        return [(m.c, per_output(m.c))]
    A = m.A.numpy()
    rhs = ops.gemm(adj, ops.full((P, 1), 1.0, like=X)) if (A.shape[1] == 1 and P > 1) else adj
    return [(m.A, ops.gemm(X, rhs, transa=True)), (m.b, per_output(m.b))]
