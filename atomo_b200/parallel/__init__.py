"""Communication layer: transports (gloo / NCCL baseline) and the symmetric
NVLink peer-memory heap used by the fused H100 path."""
from .transport import Transport, TorchDistTransport, STOP_STEP
from . import wire
