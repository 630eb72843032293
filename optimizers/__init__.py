"""Reference package name (optimizers/) -> CUDA implementations with the same class surface."""
from mlx_cuda_distributed_pretraining_b200.optimizers import AdamW, HybridOptimizer, Muon, Shampoo, ShampooParams  # noqa: F401
