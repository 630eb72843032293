"""Sliding-window attention on the host: the `model.attention.sliding_window` config key, the dense masks that define
the semantics (query q sees key k iff 0 <= q - k <= W, within its document), and the tile counts the benchmark
reports."""
import copy
import importlib.util
from pathlib import Path

import pytest
import torch
import yaml

ROOT = Path(__file__).resolve().parents[1]


def _c1():
    return yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())


@pytest.mark.parametrize("bad", [-1, 1.5, True, False, "64", [64]])
def test_config_rejects_bad_window(bad):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    d = _c1()
    d["model"]["attention"]["sliding_window"] = bad
    with pytest.raises(ValueError, match="sliding_window"):
        Config.from_dict(d)


@pytest.mark.parametrize("good", [None, 0, 1, 1024])
def test_config_accepts_window(good):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    d = _c1()
    d["model"]["attention"]["sliding_window"] = good
    assert Config.from_dict(copy.deepcopy(d)).model.attention["sliding_window"] == good
    assert "sliding_window" not in Config.from_dict(_c1()).model.attention


def _brute(pos, W):
    """[B, S, S] bool: 0 <= q - k <= W and k at or after q's document start (pos None: one document)."""
    B, S = pos.shape
    ok = torch.zeros(B, S, S, dtype=torch.bool)
    for b in range(B):
        for q in range(S):
            for k in range(S):
                d = q - k
                ok[b, q, k] = 0 <= d <= int(pos[b, q]) and (W is None or d <= W)
    return ok


def _layouts(S):
    rows = []
    for lens in ([S], [1, 2, 3, S - 6], [5, 17, 1, 40, S - 63], [S // 2, S - S // 2]):
        rows.append(torch.cat([torch.arange(n) for n in lens]))
    return torch.stack(rows).int()


@pytest.mark.parametrize("W", [None, 0, 1, 3, 16, 62, 63, 64, 100])
def test_dense_masks_match_brute_force(W):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import CausalMask, DocumentCausalMask
    S = 64
    pos = _layouts(S)
    want = _brute(pos, W)
    doc = DocumentCausalMask(pos, W).dense()[:, 0]
    assert torch.equal(doc == 0, want) and bool((doc[~want] == float("-inf")).all())
    causal = CausalMask(S, W).dense()[0, 0]
    assert torch.equal(causal == 0, want[0])
    # the identity the kernels rely on: the windowed mask is the document mask with pos clamped at W
    if W is not None:
        assert torch.equal(DocumentCausalMask(pos.clamp(max=W)).dense(), doc[:, None])
        assert torch.equal(DocumentCausalMask(torch.arange(S).clamp(max=W)[None].int()).dense()[0, 0], causal)
    # a window covering the row is the causal / document mask
    if W is not None and W >= S - 1:
        assert torch.equal(causal, CausalMask(S).dense()[0, 0])
        assert torch.equal(doc, DocumentCausalMask(pos).dense()[:, 0])


def test_masks_reject_bad_window():
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import CausalMask, DocumentCausalMask
    for bad in (-1, 2.0, True):
        with pytest.raises(ValueError):
            CausalMask(8, bad)
        with pytest.raises(ValueError):
            DocumentCausalMask(torch.zeros(1, 8, dtype=torch.int32), bad)


def _bench():
    spec = importlib.util.spec_from_file_location("window_bench", ROOT / "scripts" / "window_bench.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_forward_tile_counts():
    """Forward 128x128 tiles per (row, head) the window kernels execute, computed from the shapes."""
    b = _bench()
    assert b.fwd_tiles(2048, None) == 136 and b.fwd_tiles(2048, 512) == 70
    assert b.fwd_tiles(8192, None) == 2080 and b.fwd_tiles(8192, 1024) == 540
    assert b.fwd_tiles(2048, 4096) == b.fwd_tiles(2048, None)


def test_backward_items_and_pairs():
    b = _bench()
    S = 2048
    # causal: key tile kt has the 64-query items from 2 kt to the end
    assert b.bwd_items(S, None) == sum(S // 64 - 2 * kt for kt in range(S // 128))
    # W = 0: each key tile only its own two items
    assert b.bwd_items(S, 0) == 2 * (S // 128)
    assert b.visible_pairs(S, None) == S * (S + 1) // 2
    assert b.visible_pairs(S, 0) == S
    assert b.visible_pairs(S, 100) == sum(min(q, 100) + 1 for q in range(S))
