"""Drop-in shim: `python -m core.training --config <yaml>` resolves to the CUDA hot path."""
