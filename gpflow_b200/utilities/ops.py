"""Host-side initialisers (mirrors gpflow/utilities/ops.py:153-167)."""
from __future__ import annotations

from typing import Any

import numpy as np


def pca_reduce(Y: Any, Q: int) -> np.ndarray:
    """Projects the centred rows of Y [N, D] onto the Q eigenvectors of largest eigenvalue of the sample covariance:
    the reference's initialiser of the GPLVM latent means.  A one-off initialisation, so it runs in NumPy on the host."""
    Y = np.asarray(Y.detach().cpu().numpy() if hasattr(Y, "detach") else Y, dtype=np.float64)
    if Q > Y.shape[1]:
        raise ValueError("Cannot have more latent dimensions than observed")
    Yc = Y - Y.mean(axis=0, keepdims=True)
    _, evecs = np.linalg.eigh(Yc.T @ Yc / Y.shape[0])
    return Yc @ evecs[:, -Q:]
