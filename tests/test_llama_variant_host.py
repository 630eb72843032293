"""`model.misc.variant: mlx_lm` on the host: config validation, the fp64 oracle of the block pinned against
transformers' LlamaForCausalLM, and the mlx-lm exporter (tools/convert-to-mlx-lm.py)."""
import copy
import json
import os
from pathlib import Path

import pytest
import torch
import yaml

from oracle import reference_math as rm
from tests import llama_variant_oracle as vo

ROOT = Path(__file__).resolve().parents[1]
THETA = 10000.0  # rope.theta of every config here


def _c1():
    return yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())


def _cfg(d):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    return Config.from_dict(copy.deepcopy(d))


def test_variant_absent_leaves_config_unchanged():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import ModelArgs
    c = _cfg(_c1())
    assert "variant" not in c.model.misc
    assert ModelArgs(model_type="llama", hidden_size=8, num_hidden_layers=1, intermediate_size=8,
                     num_attention_heads=1).variant is None


@pytest.mark.parametrize("good", [None, "reference", "mlx_lm"])
def test_config_accepts_variant(good):
    d = _c1()
    d["model"]["misc"]["variant"] = good
    assert _cfg(d).model.misc["variant"] == good


@pytest.mark.parametrize("bad", ["mlx-lm", "MLX_LM", "", 1, True, ["mlx_lm"], {"a": 1}])
def test_config_rejects_bad_variant(bad):
    d = _c1()
    d["model"]["misc"]["variant"] = bad
    with pytest.raises(ValueError, match="variant"):
        _cfg(d)


def test_variant_rejects_rope_disabled_and_scaling():
    d = _c1()
    d["model"]["misc"]["variant"] = "mlx_lm"
    d["model"]["rope"]["enabled"] = False
    with pytest.raises(ValueError, match="rope.enabled"):
        _cfg(d)
    d["model"]["rope"]["enabled"] = True
    d["model"]["rope"]["scaling"] = {"type": "linear", "factor": 2.0}
    with pytest.raises(ValueError, match="rope.scaling"):
        _cfg(d)
    d["model"]["misc"]["variant"] = None   # the reference block ignores both, as before
    d["model"]["rope"]["enabled"] = False
    _cfg(d)


def test_config_yaml_round_trip_keeps_variant(tmp_path):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    d = _c1()
    d["model"]["misc"]["variant"] = "mlx_lm"
    p = tmp_path / "config.yaml"
    p.write_text(yaml.safe_dump(d))
    assert Config.from_yaml(str(p)).model.misc["variant"] == "mlx_lm"


def test_model_args_and_modules_follow_variant():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    kw = dict(model_type="llama", hidden_size=32, num_hidden_layers=1, intermediate_size=64, num_attention_heads=2,
              vocab_size=16)
    blk = Model(ModelArgs(**kw, variant="mlx_lm")).layers[0]
    assert blk.mlp.act == "silu" and blk.self_attn.apply_rope and blk.self_attn.rope_layout == "half"
    blk = Model(ModelArgs(**kw, variant="mlx_lm", rope_traditional=True)).layers[0]
    assert blk.self_attn.rope_layout == "interleaved"
    blk = Model(ModelArgs(**kw)).layers[0]
    assert blk.mlp.act == "sigmoid2" and not blk.self_attn.apply_rope and blk.self_attn.rope_layout == "interleaved"
    with pytest.raises(ValueError):
        Model(ModelArgs(**kw, variant="gpt2"))


def test_ops_validate_layout_and_act():
    from mlx_cuda_distributed_pretraining_b200 import ops
    x = torch.zeros(1, 2, 1, 16)
    with pytest.raises(ValueError, match="layout"):
        ops.rope(x, torch.zeros(2, 8), torch.zeros(2, 8), layout="split")
    with pytest.raises(ValueError, match="act"):
        ops.glu(torch.zeros(8), torch.zeros(8), act="gelu")
    with pytest.raises(ValueError, match="act"):
        ops.mlp(torch.zeros(2, 8), torch.zeros(8, 8), torch.zeros(8, 8), torch.zeros(8, 8), act="swiglu")
    with pytest.raises(ValueError, match="head_dim"):
        ops.rope(torch.zeros(1, 2, 1, 8), torch.zeros(2, 4), torch.zeros(2, 4), layout="half")
    # fp32 CPU tensors take the torch formulas
    g, u = torch.randn(8, dtype=torch.float64), torch.randn(8, dtype=torch.float64)
    assert torch.equal(ops.glu(g, u, "silu"), torch.nn.functional.silu(g) * u)
    assert torch.equal(ops.glu(g, u), g * torch.sigmoid(u) * 2)


def test_rope_half_is_rotate_half():
    """The oracle's half-split rotation is HF's q * cos + rotate_half(q) * sin with duplicated angles."""
    x = torch.randn(2, 5, 3, 16, dtype=torch.float64)
    D = 16
    inv = 10000.0 ** (-torch.arange(0, D, 2, dtype=torch.float64) / D)
    ang = torch.arange(5, dtype=torch.float64)[:, None] * inv
    emb = torch.cat([ang, ang], -1)[None, :, None]
    rot = torch.cat([-x[..., D // 2:], x[..., : D // 2]], -1)
    assert torch.allclose(vo.rope_half(x), x * emb.cos() + rot * emb.sin(), atol=1e-14, rtol=0)


# ---- the pin: transformers.LlamaForCausalLM ----------------------------------------------------------------------
def _dims(H, inter, L, nh, nkv, hd, V, tied):
    return rm.LlamaDims(hidden_size=H, intermediate_size=inter, num_layers=L, num_heads=nh, num_kv_heads=nkv,
                        head_dim=hd, vocab_size=V, rms_norm_eps=1e-5, rope_theta=10000.0, use_rope=True,
                        tie_word_embeddings=tied)


def _params(d, seed):
    p = rm.init_params(d, seed=seed, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed + 1)
    for k in p:
        if p[k].dim() == 1:   # non-trivial norm gains, so a swapped norm shows
            p[k] = 1 + 0.3 * torch.randn(p[k].shape, generator=g, dtype=torch.float64)
    return p


@pytest.fixture
def hf_fp64(monkeypatch):
    """transformers in full fp64: its RMSNorm variance and RoPE angles are always computed in fp32 (a precision
    choice, not part of the function); both are restated in fp64 here so the pin can hold to 1e-10."""
    pytest.importorskip("transformers")
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    from transformers.models.llama import modeling_llama as ml

    def norm(self, h):
        var = h.pow(2).mean(-1, keepdim=True)
        return self.weight * (h * torch.rsqrt(var + self.variance_epsilon))

    def rot(self, x, position_ids):
        D = self.inv_freq.numel() * 2
        inv = THETA ** (-torch.arange(0, D, 2, dtype=torch.float64) / D)
        ang = position_ids[:, :, None].double() * inv
        emb = torch.cat([ang, ang], -1)
        return emb.cos().to(x.dtype), emb.sin().to(x.dtype)

    monkeypatch.setattr(ml.LlamaRMSNorm, "forward", norm)
    monkeypatch.setattr(ml.LlamaRotaryEmbedding, "forward", rot)
    return ml


def _hf_config(d, V):
    from transformers import LlamaConfig
    return LlamaConfig(vocab_size=V, hidden_size=d.hidden_size, intermediate_size=d.intermediate_size,
                       num_hidden_layers=d.num_layers, num_attention_heads=d.num_heads,
                       num_key_value_heads=d.num_kv_heads, head_dim=d.head_dim, rms_norm_eps=d.rms_norm_eps,
                       rope_theta=d.rope_theta, tie_word_embeddings=d.tie_word_embeddings, hidden_act="silu",
                       max_position_embeddings=64, attention_bias=False, mlp_bias=False)


CASES = [  # (hidden, inter, layers, heads, kv heads, head_dim, vocab, tied)
    (64, 96, 2, 4, 2, 16, 40, True),     # GQA, tied, D 16
    (64, 96, 2, 4, 4, 16, 40, False),    # MHA, untied
    (128, 160, 2, 2, 1, 64, 50, False),  # GQA, D 64
    (128, 128, 1, 2, 2, 64, 33, True),   # MHA, tied, D 64
]


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_transformers_llama(hf_fp64, case):
    from transformers import LlamaForCausalLM
    from mlx_cuda_distributed_pretraining_b200.tools.export import hf_name
    *dims, V, tied = case
    d = _dims(*dims, V, tied)
    params = _params(d, seed=sum(dims))
    model = LlamaForCausalLM(_hf_config(d, V)).double().eval()
    sd = {hf_name(k): v for k, v in params.items()}
    if tied:
        sd["lm_head.weight"] = params["embed_tokens.weight"]
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and set(missing) <= {"lm_head.weight"}
    tokens = torch.randint(0, V, (2, 23), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = model(tokens).logits
    got = vo.forward(params, tokens, d)
    assert float((got - want).abs().max()) <= 1e-10


# ---- exporter ------------------------------------------------------------------------------------------------
def _fake_run(tmp_path, name="r", **over):
    from safetensors.torch import save_file
    d = _c1()
    d["name"] = name
    m = d["model"]
    m["misc"]["variant"] = "mlx_lm"
    m["dimensions"].update(hidden_size=64, intermediate_size=96, num_layers=2)
    m["attention"].update(num_heads=4, num_kv_heads=2, head_dim=16)
    for sec, kv in over.items():
        m[sec].update(kv)
    run = tmp_path / "runs" / name
    (run / "checkpoints").mkdir(parents=True)
    (run / "config.yaml").write_text(yaml.safe_dump(d))
    V = d["data"]["tokenizer"]["normal_vocab_size"] + len(d["data"]["tokenizer"]["special_tokens"])
    dims = _dims(64, 96, 2, 4, 2, 16, V, m["misc"]["tie_word_embeddings"])
    params = _params(dims, seed=11)
    save_file({k: v.float().contiguous() for k, v in params.items()},
              str(run / "checkpoints" / "step_final_model.safetensors"))
    return tmp_path / "runs", dims, {k: v.float().double() for k, v in params.items()}


@pytest.mark.parametrize("tied", [True, False])
def test_export_loads_in_transformers(tmp_path, hf_fp64, tied):
    from safetensors.torch import load_file
    from transformers import LlamaForCausalLM
    from mlx_cuda_distributed_pretraining_b200.tools.export import main
    runs, d, params = _fake_run(tmp_path, misc={"tie_word_embeddings": tied})
    out = tmp_path / "out"
    main(["--run", "r", "--out-path", str(out), "--runs-dir", str(runs)])
    cfg = json.loads((out / "config.json").read_text())
    assert cfg["architectures"] == ["LlamaForCausalLM"] and cfg["hidden_act"] == "silu"
    assert cfg["model_type"] == "llama" and cfg["num_key_value_heads"] == 2 and cfg["head_dim"] == 16
    assert cfg["torch_dtype"] == "float32" and cfg["max_position_embeddings"] == 1024
    w = load_file(str(out / "model.safetensors"))
    assert ("lm_head.weight" in w) == (not tied)
    assert all(t.dtype == torch.float32 for t in w.values())
    assert "model.layers.1.self_attn.k_proj.weight" in w and "model.layers.0.mlp.gate_proj.weight" in w
    assert not (out / "tokenizer.json").exists()   # byte-level run: weights and config only
    tokens = torch.randint(0, d.vocab_size, (2, 19), generator=torch.Generator().manual_seed(3))
    model = LlamaForCausalLM.from_pretrained(str(out), dtype=torch.float64).eval()
    with torch.no_grad():
        got = model(tokens).logits
    assert float((got - vo.forward(params, tokens, d)).abs().max()) <= 1e-10


@pytest.mark.parametrize("over,match", [
    ({"misc": {"variant": None}}, "variant"),
    ({"misc": {"variant": "reference"}}, "variant"),
    ({"rope": {"traditional": True}}, "traditional"),
    ({"attention": {"sliding_window": 64}}, "sliding_window"),
    ({"misc": {"logit_scale": 0.5}}, "logit_scale"),
])
def test_export_refuses_other_functions(tmp_path, over, match):
    from mlx_cuda_distributed_pretraining_b200.tools.export import export_run
    runs, _, _ = _fake_run(tmp_path, **over)
    with pytest.raises(ValueError, match=match):
        export_run("r", str(tmp_path / "out"), str(runs))
    assert not (tmp_path / "out" / "model.safetensors").exists()


def test_export_cli_script_runs(tmp_path):
    import subprocess
    import sys
    runs, _, _ = _fake_run(tmp_path)
    env = dict(os.environ, HF_HUB_OFFLINE="1")
    r = subprocess.run([sys.executable, str(ROOT / "tools" / "convert-to-mlx-lm.py"), "--run", "r", "--out-path",
                        str(tmp_path / "o"), "--runs-dir", str(runs), "--checkpoint", "step_final"],
                       capture_output=True, text=True, env=env, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "o" / "model.safetensors").is_file() and (tmp_path / "o" / "config.json").is_file()
