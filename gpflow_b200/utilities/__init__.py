from .multipledispatch import Dispatcher
from . import ops
from .misc import set_trainable, to_default_float, training_loop

__all__ = ["Dispatcher", "ops", "set_trainable", "to_default_float", "training_loop"]
