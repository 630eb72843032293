"""Reference entry point name (core/training.py) -> CUDA implementation."""
from mlx_cuda_distributed_pretraining_b200.core.training import *  # noqa: F401,F403
from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer, main, train  # noqa: F401

if __name__ == "__main__":
    main()
