"""gpflow/utilities/misc.py:47-109 subset."""
from __future__ import annotations

from typing import Any, Callable, Iterable, Optional, Sequence, Union

import numpy as np

from .. import config
from ..base import Module, Parameter


def to_default_float(x: Any):
    if hasattr(x, "detach"):
        from .. import ops

        return ops.to_device(x)
    return np.asarray(x, dtype=config.default_float())


def set_trainable(model: Union[Module, Parameter, Iterable[Any]], flag: bool) -> None:
    if isinstance(model, Parameter):
        model.trainable = flag
        return
    if isinstance(model, Module):
        for p in model.parameters:
            p.trainable = flag
        return
    for m in model:
        set_trainable(m, flag)


def training_loop(closure: Callable[[], Any], optimizer: Optional[Any] = None,
                  var_list: Optional[Sequence[Parameter]] = None, maxiter: int = 1_000, compile: bool = False) -> None:
    """misc.py:76-109: `maxiter` calls of `optimizer.minimize(closure, var_list)`, one step (and, for a closure over an
    iterator, one minibatch) each.  `optimizer` defaults to `optimizers.Adam()` with its default settings, as in the
    reference.  `var_list=None` trains the trainable variables of the closure's model; the reference's default, an
    empty list, is an error in Keras.  `compile` is accepted for signature parity; nothing is traced here."""
    from ..models.model import loss_model_and_batch
    from ..optimizers import Adam

    optimizer = Adam() if optimizer is None else optimizer
    if var_list is None:
        var_list = loss_model_and_batch(closure, "training_loop")[0].trainable_variables
    for _ in range(maxiter):
        optimizer.minimize(closure, var_list)
