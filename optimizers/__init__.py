"""Reference package name (optimizers/) -> CUDA implementations with the same class surface."""
from mlx_cuda_distributed_pretraining_b200.optimizers import (  # noqa: F401
    SGD, AdamW, HybridOptimizer, Lion, Muon, SGDEnhanced, Shampoo, ShampooParams)
