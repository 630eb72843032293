"""Host-side checks of attention dropout: the Philox oracle, the keep-mask quantisation, config validation, seed
derivation, the exporter field, and that the element-wise checker of the GPU tests rejects single mask faults."""
import math

import numpy as np
import pytest
import torch

from tests import dropout_oracle as do
from mlx_cuda_distributed_pretraining_b200 import ops


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    got = do.philox4x32_10(*[np.uint32(c) for c in ctr], *key)
    assert tuple(int(x) for x in got) == want


def test_threshold_quantisation():
    assert do.threshold(0.0) == 0
    assert do.threshold(0.1) == 6554
    assert do.threshold(0.5) == 32768
    assert do.threshold(0.99999999) == 65535
    assert do.scale(0.5) == 2.0
    assert do.scale(0.1) == 65536.0 / (65536 - 6554)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_rate(p):
    keep = do.keep_mask(0x1234_5678_9ABC_DEF0, p, 2, 4, 512)  # 2 * 4 * 512^2 = 2.1M elements
    n = keep.size
    pk = 1.0 - do.threshold(p) / 65536.0
    assert abs(keep.mean() - pk) < 5 * math.sqrt(pk * (1 - pk) / n)


def test_mask_depends_on_every_coordinate():
    keep = do.keep_mask(7, 0.5, 2, 2, 64)
    assert (keep[0] != keep[1]).any() and (keep[:, 0] != keep[:, 1]).any()
    assert (keep[..., :32, :] != keep[..., 32:, :]).any() and (keep != keep.transpose(0, 1, 3, 2)).any()
    assert (keep != do.keep_mask(8, 0.5, 2, 2, 64)).any()


def test_seed_chain():
    a = ops.dropout_seed(42, 0, 5)
    assert a == ops.dropout_seed(42, 0, 5) and 0 <= a < 1 << 64
    assert len({a, ops.dropout_seed(43, 0, 5), ops.dropout_seed(42, 1, 5), ops.dropout_seed(42, 0, 6)}) == 4
    assert ops.dropout_seed(a, 0) != ops.dropout_seed(a, 1)
    assert ops.splitmix64(0) == 0xE220A8397B1DCDAF  # splitmix64's first output from state 0


@pytest.mark.parametrize("bad", [True, "0.1", float("nan"), -0.1, 1.0, 1.5])
def test_ops_rejects_bad_p(bad):
    q = torch.zeros(1, 4, 2, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.attention(q, q, q, dropout=bad, seed=1)


@pytest.mark.parametrize("bad", [-1, 1 << 64, 1.0, True, "3"])
def test_ops_rejects_bad_seed(bad):
    q = torch.zeros(1, 4, 2, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.attention(q, q, q, dropout=0.1, seed=bad)


def test_ops_rejects_prefix():
    q = torch.zeros(1, 4, 2, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.attention(q, q, q, dropout=0.1, seed=1, prefix=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(ValueError):
        ops.attention_fp32(q.float()[..., :16], q.float()[..., :16], q.float()[..., :16], dropout=0.1,
                           prefix=torch.zeros(1, dtype=torch.int32))


def _model_config(attn_extra):
    from mlx_cuda_distributed_pretraining_b200.core.training import ModelConfig
    attn = {"num_heads": 2, "max_position_embeddings": 64, **attn_extra}
    return ModelConfig(architecture="llama", dimensions={"hidden_size": 32, "intermediate_size": 64,
                                                         "num_layers": 1},
                       attention=attn, normalization={}, rope={}, misc={})


@pytest.mark.parametrize("bad", [True, False, "0.1", float("nan"), -0.1, 1.0, 2])
def test_config_rejects(bad):
    with pytest.raises(ValueError):
        _model_config({"dropout": bad})


def test_config_rejects_prefix_lm():
    with pytest.raises(ValueError):
        _model_config({"dropout": 0.1, "prefix_lm": True})
    _model_config({"dropout": 0, "prefix_lm": True})
    _model_config({"dropout": None})
    _model_config({"dropout": 0.1})


def test_model_args_off_equals_absent():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    base = dict(model_type="llama", hidden_size=32, num_hidden_layers=2, intermediate_size=64, num_attention_heads=2)
    m = Model(ModelArgs(**base, attention_dropout=0.0))
    assert [l.self_attn.attn.layer_idx for l in m.layers] == [0, 1]
    assert all(l.self_attn.attn.dropout == 0.0 for l in m.layers)
    m = Model(ModelArgs(**base, attention_dropout=0.25))
    assert all(l.self_attn.attn.dropout == 0.25 for l in m.layers)
    m.train()
    assert m.layers[0].self_attn.attn.drops()
    with torch.no_grad():
        assert not m.layers[0].self_attn.attn.drops()
    m.eval()
    assert not m.layers[0].self_attn.attn.drops()


def test_exporter_field():
    from types import SimpleNamespace
    from mlx_cuda_distributed_pretraining_b200.tools.export import hf_config

    def cfg(attn_extra):
        m = SimpleNamespace(attention={"num_heads": 2, "num_kv_heads": 2, **attn_extra},
                            dimensions={"hidden_size": 32, "intermediate_size": 64, "num_layers": 1},
                            misc={"attention_bias": False, "mlp_bias": False, "tie_word_embeddings": True},
                            normalization={"rms_norm_eps": 1e-5}, rope={"theta": 10000.0, "scaling": None,
                                                                         "traditional": False})
        return SimpleNamespace(model=m, data=SimpleNamespace(preprocessing={"max_context_size": 64}))
    assert hf_config(cfg({"dropout": 0.1}), 100, 1, 2)["attention_dropout"] == 0.1
    assert hf_config(cfg({}), 100, 1, 2)["attention_dropout"] == 0.0


# the checker the GPU tests use (tests/attn_dropout_check.py) must reject single mask faults: outputs computed with
# the true mask and rounded to bf16 as the kernels' are, checked against a reference that takes the fault
def _outputs(p, seed, S=48, B=2, H=4, Hk=2, D=16):
    from tests import attn_dropout_check as dc
    g = torch.Generator().manual_seed(1)
    q, k, v, dout = (torch.randn(B, S, h, D, generator=g).to(torch.bfloat16) for h in (H, Hk, Hk, H))
    vis = torch.ones(S, S, dtype=torch.bool).tril().expand(B, S, S)
    o64 = dc.reference(q, k, v, torch.zeros(B, S, H, D), dout, None, D ** -0.5, vis, seed, p)["o"][0]
    o = o64.to(torch.bfloat16)
    true = dc.reference(q, k, v, o, dout, None, D ** -0.5, vis, seed, p)
    got = {n: true[n][0].to(torch.bfloat16) if n != "lse" else true[n][0].float() for n in true}
    return (q, k, v, o, dout, vis), got


def _rejects(args, got, seed, p, **fault):
    from tests import attn_dropout_check as dc
    q, k, v, o, dout, vis = args
    ref = dc.reference(q, k, v, o, dout, None, q.shape[-1] ** -0.5, vis, seed, p, **fault)
    for n in ("o", "dq", "dk", "dv"):
        try:
            dc.check(n, got[n], *ref[n])
        except AssertionError:
            return True
    return False


def test_checker_accepts_true_mask_and_rejects_faults():
    p, seed = 0.3, 99
    args, got = _outputs(p, seed)
    assert not _rejects(args, got, seed, p)

    def flipped(b, h):
        m = do.keep_mask_head(seed, p, b, h, 48)
        if (b, h) == (1, 2):
            m[3, 1] = ~m[3, 1]
        return m
    assert _rejects(args, got, seed, p, keep_fn=flipped)
    assert _rejects(args, got, seed, p, keep_fn=lambda b, h: do.keep_mask_head(seed, p, b, h, 48).T)
    assert _rejects(args, got, seed, p, keep_fn=lambda b, h: do.keep_mask_head(seed, p, b, h // 2, 48))


def test_checker_rejects_unquantised_scale():
    """1 / (1 - p) instead of 1 / (1 - p_eff).  Where p is a multiple of 2^-16 the two agree; near 1 they differ
    most (p = 0.9999: p_eff = 65529 / 65536, 6.8 % apart), far beyond any bf16 output's resolution elsewhere."""
    p, seed = 0.9999, 12345
    assert do.keep_mask(seed, p, 2, 4, 48).any()
    args, got = _outputs(p, seed)
    assert not _rejects(args, got, seed, p)
    assert _rejects(args, got, seed, p, sc=1.0 / (1.0 - p))
