"""PS-side optimizers (parity: ``/root/reference/src/optim/__init__.py``), the layer-wise LARS and LAMB, AdamW and Lion."""
from .sgd import SGD
from .adam import Adam
from .adamw import AdamW
from .lars import LARS
from .lamb import LAMB
from .lion import Lion

__all__ = ["SGD", "Adam", "AdamW", "LARS", "LAMB", "Lion"]
