"""PS-side optimizers (parity: ``/root/reference/src/optim/__init__.py``), the layer-wise LARS and LAMB, and AdamW."""
from .sgd import SGD
from .adam import Adam
from .adamw import AdamW
from .lars import LARS
from .lamb import LAMB

__all__ = ["SGD", "Adam", "AdamW", "LARS", "LAMB"]
