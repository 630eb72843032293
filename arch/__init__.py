"""Reference package name (arch/) -> CUDA implementations."""
