from .multipledispatch import Dispatcher
from .misc import set_trainable, to_default_float, training_loop

__all__ = ["Dispatcher", "set_trainable", "to_default_float", "training_loop"]
