"""ALiBi on the host: the `model.attention.alibi` config key, the slopes of `alibi_slopes` against the paper's closed
form, the exporter's refusal and generation's length limit (past max_position_embeddings only for ALiBi without
RoPE)."""
import copy
import types
from pathlib import Path

import pytest
import torch
import yaml

ROOT = Path(__file__).resolve().parents[1]


def _c1():
    return yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())


@pytest.mark.parametrize("good", [True, False, None])
def test_config_accepts_alibi(good):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    d = _c1()
    d["model"]["attention"]["alibi"] = good
    assert Config.from_dict(copy.deepcopy(d)).model.attention["alibi"] is good
    assert "alibi" not in Config.from_dict(_c1()).model.attention


@pytest.mark.parametrize("bad", [1, 0, "true", 1.0, [True]])
def test_config_rejects_non_bool_alibi(bad):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    d = _c1()
    d["model"]["attention"]["alibi"] = bad
    with pytest.raises(ValueError, match="alibi"):
        Config.from_dict(d)


def _closed_form(H):
    """The ALiBi paper's slopes, written from its definition in exact powers of two: exponents -8 i / H for a power of
    two H; else the exponents -8 i / n (n = 2^floor(log2 H)) and then -8 (2 j - 1) / (2 n), j = 1 .. H - n."""
    n = 1
    while 2 * n <= H:
        n *= 2
    exps = [-8.0 * i / n for i in range(1, n + 1)] + [-8.0 * (2 * j - 1) / (2 * n) for j in range(1, H - n + 1)]
    return torch.tensor([2.0 ** e for e in exps], dtype=torch.float64)


@pytest.mark.parametrize("H", list(range(1, 65)))
def test_alibi_slopes_closed_form(H):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    s = alibi_slopes(H)
    assert s.dtype == torch.float32 and tuple(s.shape) == (H,)
    ref = _closed_form(H)
    assert torch.allclose(s.double(), ref, rtol=2 ** -23, atol=0), (H, s, ref)
    assert bool((s > 0).all()) and bool((s < 1).all()) and len(set(s.tolist())) == H


def test_alibi_slopes_examples():
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    assert alibi_slopes(8).tolist() == [2.0 ** -i for i in range(1, 9)]
    want12 = [2.0 ** -i for i in range(1, 9)] + [2.0 ** -0.5, 2.0 ** -1.5, 2.0 ** -2.5, 2.0 ** -3.5]
    assert torch.allclose(alibi_slopes(12).double(), torch.tensor(want12, dtype=torch.float64), rtol=2 ** -23)
    s20, s48 = alibi_slopes(20).double(), alibi_slopes(48).double()
    assert torch.allclose(s20[16:], torch.tensor([2.0 ** (-(2 * j - 1) / 4) for j in range(1, 5)],
                                                 dtype=torch.float64), rtol=2 ** -23)
    assert torch.allclose(s48[:32], torch.tensor([2.0 ** (-i / 4) for i in range(1, 33)], dtype=torch.float64),
                          rtol=2 ** -23)
    assert torch.allclose(s48[32:], torch.tensor([2.0 ** (-(2 * j - 1) / 8) for j in range(1, 17)],
                                                 dtype=torch.float64), rtol=2 ** -23)
    for bad in (0, -1, 2.0, True):
        with pytest.raises(ValueError):
            alibi_slopes(bad)


def test_slopes_are_not_parameters():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    base = dict(model_type="llama", hidden_size=64, num_hidden_layers=2, intermediate_size=128,
                num_attention_heads=4, head_dim=16, vocab_size=300)
    plain, alibi = Model(ModelArgs(**base)), Model(ModelArgs(**base, alibi=True))
    assert list(dict(plain.named_parameters())) == list(alibi.parameters_dict())
    assert list(plain.state_dict()) == list(alibi.state_dict())
    attn = alibi.layers[0].self_attn.attn
    assert attn.alibi and not plain.layers[0].self_attn.attn.alibi
    assert plain.layers[0].self_attn.attn.alibi_slopes("cpu") is None
    assert torch.equal(attn.alibi_slopes("cpu"), torch.tensor([2.0 ** -2, 2.0 ** -4, 2.0 ** -6, 2.0 ** -8]))


def test_exporter_refuses_alibi_runs():
    from mlx_cuda_distributed_pretraining_b200.tools.export import check_exportable
    m = types.SimpleNamespace(misc={"variant": "mlx_lm"}, rope={"traditional": False},
                              attention={"alibi": True})
    with pytest.raises(ValueError, match="alibi"):
        check_exportable(m)
    m.attention = {"alibi": False}
    check_exportable(m)


def _model(alibi, rope=False, variant=None, limit=64):
    return types.SimpleNamespace(args=types.SimpleNamespace(max_position_embeddings=limit, alibi=alibi,
                                                            apply_rope=rope, variant=variant))


def test_generation_length_limit():
    from mlx_cuda_distributed_pretraining_b200.core import generation as G
    assert G.position_limit(_model(True).args) is None
    assert G.position_limit(_model(True, rope=True).args) == 64
    assert G.position_limit(_model(True, variant="mlx_lm").args) == 64
    assert G.position_limit(_model(False).args) == 64
    for model in (_model(False), _model(True, rope=True), _model(True, variant="mlx_lm")):
        with pytest.raises(ValueError, match="max_position_embeddings"):
            G.generate(model, [[1] * 40], max_tokens=25)
