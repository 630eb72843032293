"""Export a run trained with `model.misc.variant: mlx_lm` for mlx-lm / Hugging Face:

    python tools/convert-to-mlx-lm.py --run NAME --out-path DIR [--checkpoint step_N] [--runs-dir runs]

See mlx_cuda_distributed_pretraining_b200/tools/export.py."""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from mlx_cuda_distributed_pretraining_b200.tools.export import main  # noqa: E402

if __name__ == "__main__":
    main()
