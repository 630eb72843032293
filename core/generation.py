"""Reference entry point name (core/generation.py) -> CUDA implementation."""
from mlx_cuda_distributed_pretraining_b200.core.generation import *  # noqa: F401,F403
from mlx_cuda_distributed_pretraining_b200.core.generation import generate, main  # noqa: F401

if __name__ == "__main__":
    main()
