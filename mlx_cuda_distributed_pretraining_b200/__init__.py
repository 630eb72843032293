"""H100-native (sm_90a) hot path of arthurcolle/mlx-cuda-distributed-pretraining (see DESIGN.md).

Importing the package is cheap and GPU-free; the C-ABI library is loaded on first use
(`_lib.lib()`), and every op raises if it is missing -- there is no CPU fallback.
"""
__version__ = "0.1.0"
