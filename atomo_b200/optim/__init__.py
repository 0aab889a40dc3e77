"""PS-side optimizers (parity: ``/root/reference/src/optim/__init__.py``), and the layer-wise LARS and LAMB."""
from .sgd import SGD
from .adam import Adam
from .lars import LARS
from .lamb import LAMB

__all__ = ["SGD", "Adam", "LARS", "LAMB"]
