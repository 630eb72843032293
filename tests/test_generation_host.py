"""Host-side generation logic (no GPU): the sampling filters and the repetition processor against the reference's
own make_sampler / make_logits_processors (tests/golden/sampler_vectors.npz), the CLI's arguments, checkpoint
lookup, the max_position_embeddings guard and the trainer's saved config.yaml."""
from __future__ import annotations

import types
from pathlib import Path

import numpy as np
import pytest
import torch
import yaml

from mlx_cuda_distributed_pretraining_b200.core import generation as G
from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer

ROOT = Path(__file__).resolve().parents[1]
Z = np.load(ROOT / "tests" / "golden" / "sampler_vectors.npz")
SAMPLER_KEYS = sorted({k.split("_")[0] for k in Z.files if k.startswith("s")})
PROC_KEYS = sorted({k.split("_")[0] for k in Z.files if k.startswith("r")})


def fixture_distribution(key):
    """The fixture's filtered distribution in vocabulary order (min-p / top-p are recorded in sorted order)."""
    dist = Z[f"{key}_dist"].astype(np.float64)
    p = np.exp(dist - dist.max())
    p = p / p.sum()
    if str(Z[f"{key}_kind"]) == "plain":
        return p
    out = np.zeros_like(p)
    out[Z[f"{key}_order"]] = p
    return out


def test_fixture_covers_the_required_cases():
    kinds = {str(Z[f"{k}_kind"]) for k in SAMPLER_KEYS}
    assert kinds == {"min_p", "top_p", "plain"}
    assert len({float(Z[f"{k}_temp"]) for k in SAMPLER_KEYS}) >= 3
    peaked = [k for k in SAMPLER_KEYS if str(Z[f"{k}_case"]) == "peaked" and str(Z[f"{k}_kind"]) == "min_p"]
    assert any((fixture_distribution(k) > 0).sum() == 1 for k in peaked)   # min_p keeps only the top token
    lens = {len(Z[f"{k}_tokens"]) - 1 for k in PROC_KEYS}
    assert any(n < int(Z[f"{k}_context"]) for k in PROC_KEYS for n in lens)
    assert any(len(Z[f"{k}_tokens"]) - 1 > int(Z[f"{k}_context"]) for k in PROC_KEYS)


@pytest.mark.parametrize("key", SAMPLER_KEYS)
def test_filters_match_reference_sampler(key):
    lp = torch.tensor(Z[f"{key}_logprobs"])
    kind, temp, param = str(Z[f"{key}_kind"]), float(Z[f"{key}_temp"]), float(Z[f"{key}_param"])
    got = G.sampling_distribution(lp, temp, min_p=param if kind == "min_p" else None,
                                  top_p=param if kind == "top_p" else None)
    np.testing.assert_allclose(got.numpy(), fixture_distribution(key), rtol=0, atol=1e-6)


@pytest.mark.parametrize("key", PROC_KEYS)
def test_repetition_penalty_matches_reference_processor(key):
    toks = Z[f"{key}_tokens"].tolist()
    got = G.apply_repetition_penalty(torch.tensor(Z[f"{key}_logits"])[None],
                                     [G.repetition_window(toks, int(Z[f"{key}_context"]))],
                                     float(Z[f"{key}_penalty"]))[0]
    np.testing.assert_allclose(got.numpy(), Z[f"{key}_out"], rtol=1e-6, atol=1e-6)


def test_repetition_window_is_the_literal_slice():
    assert G.repetition_window([1, 2, 3, 4, 5], 2) == [3, 4]      # leaves out the token just fed
    assert G.repetition_window([1, 2, 3], 20) == [1, 2]
    assert G.repetition_window([9], 20) == []


def test_temperature_zero_is_argmax():
    logits = torch.tensor([[0.1, 3.0, -1.0], [2.0, 0.0, 2.5]])
    assert G.sample(logits, 0.0, 0.05, None, None).tolist() == [1, 2]


def test_cli_defaults_and_extensions():
    a = G.parse_args(["--run", "r", "--prompt", "p"])
    assert (a.max_tokens, a.temperature, a.min_p, a.repetition_penalty, a.repetition_context_size) == \
        (256, 1.0, 0.05, 1.1, 20)
    assert (a.top_p, a.seed, a.num_samples, a.checkpoint, a.runs_dir) == (None, None, 1, None, "runs")
    a = G.parse_args(["--run", "r", "--prompt", "p", "--top-p", "0.9", "--seed", "3", "--num-samples", "4",
                      "--checkpoint", "step_10", "--runs-dir", "/x"])
    assert (a.top_p, a.seed, a.num_samples, a.checkpoint, a.runs_dir) == (0.9, 3, 4, "step_10", "/x")
    with pytest.raises(SystemExit):
        G.parse_args(["--prompt", "p"])


def test_checkpoint_resolution(tmp_path):
    ck = tmp_path / "run" / "checkpoints"
    ck.mkdir(parents=True)
    with pytest.raises(ValueError):
        G.resolve_checkpoint(tmp_path / "run")
    (ck / "step_final.safetensors").write_bytes(b"")
    assert G.resolve_checkpoint(tmp_path / "run").name == "step_final.safetensors"
    (ck / "step_final_model.safetensors").write_bytes(b"")
    assert G.resolve_checkpoint(tmp_path / "run").name == "step_final_model.safetensors"
    (ck / "step_10_model.safetensors").write_bytes(b"")
    assert G.resolve_checkpoint(tmp_path / "run", "step_10").name == "step_10_model.safetensors"
    with pytest.raises(ValueError):
        G.resolve_checkpoint(tmp_path / "run", "step_11")


def test_prompt_plus_max_tokens_beyond_max_positions_raises():
    model = types.SimpleNamespace(args=types.SimpleNamespace(max_position_embeddings=64))
    with pytest.raises(ValueError, match="max_position_embeddings"):
        G.generate(model, [[1] * 40], max_tokens=25)


def _config_dict(input_file):
    d = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
    d["data"]["input_file"] = input_file
    d["training"]["hyperparameters"]["iters"] = 7   # a CLI override
    return d


@pytest.mark.parametrize("input_file,synthetic,saved", [("synthetic:markov", True, "synthetic:markov"),
                                                         ("data/train.jsonl", True, "synthetic"),
                                                         ("data/train.jsonl", False, "data/train.jsonl")])
def test_saved_config_round_trips(tmp_path, input_file, synthetic, saved):
    cfg = Config.from_dict(_config_dict(input_file))
    stub = types.SimpleNamespace(config=cfg, synthetic=synthetic, run_dir=tmp_path)
    path = Trainer.save_config(stub)
    assert path == tmp_path / "config.yaml"
    back = Config.from_yaml(str(path))
    assert back.data.input_file == saved
    assert back.training.hyperparameters["iters"] == 7
    assert back.model == cfg.model and back.system == cfg.system and back.name == cfg.name
