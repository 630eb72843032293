"""Export a run trained with `model.misc.variant: mlx_lm` as an mlx-lm / Hugging Face `LlamaForCausalLM` directory
(the reference's tools/convert-to-mlx-lm.py, with its CLI and config fields), or as `MixtralForCausalLM` when the run
has `model.misc.num_local_experts > 0`.

The run's checkpoint holds the fp32 master weights under the trainer's flat names; they are renamed to the mlx-lm /
HF names and written as fp32 `model.safetensors` next to `config.json`.  q / k weights are not permuted: the
variant trains in the half-split RoPE layout HF Llama uses.  Runs whose exported config would describe a different
function (the reference block, interleaved RoPE, a sliding window, ALiBi, prefix-LM, logit_scale) are refused.  Runs
on the CPU.
"""
from __future__ import annotations

import argparse
import json
import re
import shutil
from pathlib import Path
from typing import Dict, List, Optional

import torch

_LAYER = re.compile(r"layers\.(\d+)\.(.+)")
_LAYER_NAMES = {
    "self_attn.attn.q_proj": "self_attn.q_proj", "self_attn.attn.k_proj": "self_attn.k_proj",
    "self_attn.attn.v_proj": "self_attn.v_proj", "self_attn.attn.o_proj": "self_attn.o_proj",
    "mlp.gate_proj": "mlp.gate_proj", "mlp.up_proj": "mlp.up_proj", "mlp.down_proj": "mlp.down_proj",
    "input_layernorm": "input_layernorm", "post_attention_layernorm": "post_attention_layernorm",
}


_MOE = re.compile(r"block_sparse_moe\.switch_mlp\.(gate_proj|up_proj|down_proj)\.weight")
_MOE_HF = {"gate_proj": "w1", "down_proj": "w2", "up_proj": "w3"}


def hf_tensors(name: str, t: torch.Tensor) -> Dict[str, torch.Tensor]:
    """One trainer parameter -> its mlx-lm / HF tensors.  Stacked experts [E, out, in] are split into Mixtral's
    per-expert checkpoint names `block_sparse_moe.experts.J.w1|w2|w3.weight` (gate, down, up), the layout both
    transformers' MixtralForCausalLM.from_pretrained and mlx-lm's Mixtral loader convert from."""
    m = _LAYER.fullmatch(name)
    if m:
        e = _MOE.fullmatch(m.group(2))
        if e:
            w = _MOE_HF[e.group(1)]
            return {f"model.layers.{m.group(1)}.block_sparse_moe.experts.{j}.{w}.weight": t[j].contiguous()
                    for j in range(t.shape[0])}
        if m.group(2) == "block_sparse_moe.gate.weight":
            return {f"model.layers.{m.group(1)}.block_sparse_moe.gate.weight": t}
    return {hf_name(name): t}


def hf_name(name: str) -> str:
    """The trainer's flat parameter name -> the mlx-lm / HF Llama name."""
    if name in ("embed_tokens.weight", "norm.weight"):
        return "model." + name
    if name == "lm_head.weight":
        return name
    m = _LAYER.fullmatch(name)
    if m:
        mod, _, leaf = m.group(2).rpartition(".")
        if mod in _LAYER_NAMES:
            return f"model.layers.{m.group(1)}.{_LAYER_NAMES[mod]}.{leaf}"
    raise ValueError(f"no mlx-lm name for parameter {name!r}")


def check_exportable(model_cfg) -> None:
    """ValueError unless the run's block is exactly what an HF LlamaForCausalLM config describes."""
    misc, rope, attn = model_cfg.misc, model_cfg.rope, model_cfg.attention
    if misc.get("variant") != "mlx_lm":
        raise ValueError("only runs trained with model.misc.variant: mlx_lm can be exported: the reference block "
                         "(gate * sigmoid(up) * 2, no or interleaved RoPE) is not LlamaForCausalLM"
                         + (" or MixtralForCausalLM" if misc.get("num_local_experts") else ""))
    if rope.get("traditional"):
        raise ValueError("rope.traditional: true (interleaved RoPE) has no LlamaForCausalLM config")
    if attn.get("sliding_window") is not None:
        raise ValueError("runs with model.attention.sliding_window cannot be exported as LlamaForCausalLM")
    if attn.get("prefix_lm"):
        raise ValueError("runs with model.attention.prefix_lm cannot be exported: LlamaForCausalLM and "
                         "MixtralForCausalLM attend causally over the prompt")
    if attn.get("alibi"):
        raise ValueError("runs with model.attention.alibi cannot be exported: LlamaForCausalLM and "
                         "MixtralForCausalLM have no ALiBi")
    if misc.get("logit_scale") is not None:
        raise ValueError("runs with model.misc.logit_scale cannot be exported as LlamaForCausalLM")


def hf_config(cfg, vocab_size: int, bos: int, eos: int) -> dict:
    """config.json: the reference exporter's fields, plus num_key_value_heads, head_dim and model_type "llama"; a
    MoE run (model.misc.num_local_experts > 0) is a MixtralForCausalLM config with its expert fields."""
    m = cfg.model
    d = _llama_config(cfg, vocab_size, bos, eos)
    E = m.misc.get("num_local_experts") or 0
    if E:
        d.pop("mlp_bias")
        d.update(architectures=["MixtralForCausalLM"], model_type="mixtral", num_local_experts=E,
                 num_experts_per_tok=m.misc["num_experts_per_tok"],
                 router_aux_loss_coef=float(m.misc.get("router_aux_loss_coef", 0.001)), router_jitter_noise=0.0,
                 output_router_logits=False, sliding_window=None)
    return d


def _llama_config(cfg, vocab_size: int, bos: int, eos: int) -> dict:
    m = cfg.model
    heads = m.attention["num_heads"]
    return {
        "architectures": ["LlamaForCausalLM"],
        "attention_bias": m.misc["attention_bias"],
        "attention_dropout": float(m.attention.get("dropout") or 0.0),
        "bos_token_id": bos,
        "eos_token_id": [eos],
        "hidden_act": "silu",
        "hidden_size": m.dimensions["hidden_size"],
        "intermediate_size": m.dimensions["intermediate_size"],
        "max_position_embeddings": cfg.data.preprocessing["max_context_size"],
        "mlp_bias": m.misc["mlp_bias"],
        "model_type": "llama",
        "num_attention_heads": heads,
        "num_hidden_layers": m.dimensions["num_layers"],
        "num_key_value_heads": m.attention.get("num_kv_heads") or heads,
        "head_dim": m.attention.get("head_dim") or m.dimensions["hidden_size"] // heads,
        "rms_norm_eps": m.normalization["rms_norm_eps"],
        "rope_scaling": m.rope["scaling"],
        "rope_theta": m.rope["theta"],
        "tie_word_embeddings": m.misc["tie_word_embeddings"],
        "torch_dtype": "float32",
        "use_cache": True,
        "vocab_size": vocab_size,
    }


def _bos_post_processor(bos_token: str, bos_id: int) -> dict:
    """The reference exporter's post-processor: every sequence starts with BOS."""
    special = lambda t: {"SpecialToken": {"id": bos_token, "type_id": t}}  # noqa: E731
    seq = lambda s, t: {"Sequence": {"id": s, "type_id": t}}  # noqa: E731
    return {"type": "Sequence", "processors": [{
        "type": "TemplateProcessing",
        "single": [special(0), seq("A", 0)],
        "pair": [special(0), seq("A", 0), special(1), seq("B", 1)],
        "special_tokens": {bos_token: {"id": bos_token, "ids": [bos_id], "tokens": [bos_token]}},
    }]}


def export_run(run: str, out_path: str, runs_dir: str = "runs", checkpoint: Optional[str] = None,
               log=print) -> Path:
    from safetensors.torch import load_file, save_file

    from ..core.generation import resolve_checkpoint
    from ..core.training import Config, TokenizerManager

    run_dir = Path(runs_dir) / run
    cfg_path = run_dir / "config.yaml"
    if not cfg_path.is_file():
        raise ValueError(f"Config not found for run: {run} ({cfg_path})")
    cfg = Config.from_yaml(str(cfg_path))
    check_exportable(cfg.model)
    ck = resolve_checkpoint(run_dir, checkpoint)
    synthetic = cfg.data.input_file.startswith("synthetic")
    tok = TokenizerManager(cfg.data, run_dir, synthetic=synthetic)

    weights = load_file(str(ck))
    out: Dict[str, torch.Tensor] = {}
    for name, t in weights.items():
        out.update(hf_tensors(name, t.float().contiguous()))
    tied = bool(cfg.model.misc["tie_word_embeddings"])
    if tied:
        out.pop("lm_head.weight", None)
    elif "lm_head.weight" not in out:
        raise ValueError(f"{ck.name}: untied run without lm_head.weight")

    out_dir = Path(out_path)
    out_dir.mkdir(parents=True, exist_ok=True)
    log(f"Writing {len(out)} tensors from {ck} to {out_dir / 'model.safetensors'}")
    save_file(out, str(out_dir / "model.safetensors"))
    with open(out_dir / "config.json", "w") as f:
        json.dump(hf_config(cfg, tok.VOCAB_SIZE, tok.BOS_TOKEN, tok.EOS_TOKEN), f, indent=4)

    if tok.external_tokenizer is None:
        log("byte-level tokenizer: wrote weights and config.json only (there is no tokenizer.json to export)")
        return out_dir
    src = run_dir / "tokenizer" / "tokenizer.json"
    if not src.is_file():
        src = Path(cfg.data.tokenizer_path) / "tokenizer.json"
    sp = cfg.data.tokenizer["special_tokens"]
    tokenizer_config = {
        "bos_token": sp["bos"], "eos_token": sp["eos"], "model_input_names": ["input_ids", "attention_mask"],
        "model_max_length": cfg.data.preprocessing["max_context_size"], "tokenizer_class": "PreTrainedTokenizerFast",
    }
    with open(out_dir / "tokenizer_config.json", "w") as f:
        json.dump(tokenizer_config, f, indent=4)
    shutil.copy2(src, out_dir / "tokenizer.json")
    with open(out_dir / "tokenizer.json") as f:
        data = json.load(f)
    data["post_processor"] = _bos_post_processor(sp["bos"], tok.BOS_TOKEN)
    with open(out_dir / "tokenizer.json", "w") as f:
        json.dump(data, f, indent=4)
    return out_dir


def parse_args(argv: Optional[List[str]] = None) -> argparse.Namespace:
    p = argparse.ArgumentParser(description="Convert a model to MLX format")
    p.add_argument("--run", type=str, required=True, help="Name of the training run to use")
    p.add_argument("--out-path", type=str, default="output", help="Path for MLX-LM Model output directory")
    p.add_argument("--checkpoint", type=str, default=None, help="checkpoint to export, e.g. step_1000 (default: final)")
    p.add_argument("--runs-dir", type=str, default="runs", help="directory holding the run directories")
    return p.parse_args(argv)


def main(argv: Optional[List[str]] = None) -> None:
    a = parse_args(argv)
    export_run(a.run, a.out_path, a.runs_dir, a.checkpoint)


if __name__ == "__main__":
    main()
