from .synthetic import SyntheticImageDataset, synthetic_pair, SHAPES
from .datasets import (build_datasets, shard_dataset, shard_indices, SVHN, BatchDataset,
                       MNISTDataset, Cifar10Dataset, num_classes_of, real_transforms)
from .loader import DataLoader
from .gpu_loader import GpuLoader, UInt8ImageDataset
