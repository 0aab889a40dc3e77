"""Tiny driver for ncu: runs the subspace route (wgmma skinny GEMMs) and the fused BN kernels a few times."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from atomo_b200.data import SyntheticImageDataset
from atomo_b200.models import build_model, input_shape
from atomo_b200.runtime.engine import FusedEngine

torch.cuda.set_device(0)
torch.manual_seed(0)
net = sys.argv[1] if len(sys.argv) > 1 else "VGG11"
eng = FusedEngine(build_model(net, 10, "Cifar10"), 0, 1, code="svd", svd_rank=3, lr=0.01, momentum=0.9, dtype="bf16",
                  channels_last=True, use_graph=False, subspace=True)
x, y = SyntheticImageDataset(input_shape(net, "Cifar10"), 10, 1024).materialize(128)
eng.prepare(x.pin_memory(), y.pin_memory(), warmup=2)
for _ in range(3):
    eng.train_step()
torch.cuda.synchronize()
print("ok", eng.error_code(), float(eng.loss_buf[0]))
eng.close()
