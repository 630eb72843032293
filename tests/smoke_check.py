"""smoke(): one tiny invocation of the whole hot path on cuda:0, checked against the oracle.

Runs (1) batched Newton-Schulz, (2) fused attention fwd+bwd, (3) one full Llama+Muon training
step through the public Trainer API, each compared with oracle/reference_math.py (CPU fp32).
Used by __graft_entry__.smoke(); the oracle is the checker here, never the thing shipped.
"""
from __future__ import annotations

import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def tiny_config(name="smoke", optimizer="muon", mixed=True, **over):
    cfg = {
        "name": name, "overwrite": True,
        "data": {"input_file": "synthetic", "preprocessing": {"max_context_size": 128, "chunk_overlap": 0},
                 "tokenizer": {"normal_vocab_size": 256,
                               "special_tokens": {"pad": "<pad>", "bos": "<bos>", "eos": "<eos>"}}},
        "model": {"architecture": "llama",
                  "dimensions": {"hidden_size": 128, "intermediate_size": 256, "num_layers": 2},
                  "attention": {"num_heads": 4, "num_kv_heads": 2, "head_dim": 32, "max_position_embeddings": 1024},
                  "normalization": {"rms_norm_eps": 1e-5},
                  "rope": {"theta": 10000, "traditional": False, "scaling": None},
                  "misc": {"attention_bias": False, "mlp_bias": False, "tie_word_embeddings": True}},
        "training": {"epochs": None,
                     "hyperparameters": {"batch_size": 2, "learning_rate": 2e-2, "weight_decay": 0.01, "iters": 100},
                     "scheduler": {"type": "cosine", "min_lr_ratio": 0.01},
                     "optimization": {"optimizer": optimizer}},
        "logging": {"log_dir": "logs", "checkpoint_dir": "checkpoints",
                    "steps": {"logging_interval": 10 ** 9, "checkpoint_interval": 0, "validation_interval": 0},
                    "metrics": {}},
        "system": {"seed": 42, "device": "gpu", "distributed": False, "mixed_precision": mixed,
                   "precision": "bfloat16"},
    }
    for k, v in over.items():
        sec, key = k.split("__")
        cfg["training" if sec == "hp" else sec]["hyperparameters" if sec == "hp" else key] = (
            {**cfg["training"]["hyperparameters"], key: v} if sec == "hp" else v)
    return cfg


def smoke(verbose: bool = True) -> dict:
    sys.path.insert(0, str(ROOT))
    from oracle import reference_math as R
    from mlx_cuda_distributed_pretraining_b200 import ops
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer

    ops.require_device()
    out = {}
    torch.manual_seed(0)
    # 1. Newton-Schulz (wide + tall) vs oracle
    for shape in ((2, 128, 256), (1, 384, 128)):
        g = torch.randn(*shape) * 0.02
        x = ops.zeropower_via_newtonschulz5(g.cuda())
        out[f"ns{shape}"] = _rel(x, R.newton_schulz5(g))
        assert out[f"ns{shape}"] < 3e-2, out
    # 2. attention fwd/bwd vs oracle (GQA, causal, padded head dim)
    B, S, H, Hk, D = 2, 160, 4, 2, 32
    q, k, v = (torch.randn(B, S, h, D).to(torch.bfloat16) for h in (H, Hk, Hk))
    qc, kc, vc = (t.cuda().requires_grad_(True) for t in (q, k, v))
    o = ops.attention(qc, kc, vc, D ** -0.5, True)
    do = torch.randn(B, S, H, D).to(torch.bfloat16)
    o.backward(do.cuda())
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    orf = R.attention(qr, kr, vr, D ** -0.5, R.causal_mask(S))
    orf.backward(do.float())
    out["attn_o"] = _rel(o, orf)
    out["attn_dq"], out["attn_dk"], out["attn_dv"] = _rel(qc.grad, qr.grad), _rel(kc.grad, kr.grad), _rel(vc.grad, vr.grad)
    assert max(out["attn_o"], out["attn_dq"], out["attn_dk"], out["attn_dv"]) < 2e-2, out
    # 3. one full training step through the Trainer vs the oracle's step
    with tempfile.TemporaryDirectory(prefix="smoke_runs_") as run_root:
        tr = Trainer(Config.from_dict(tiny_config()), synthetic=True, quiet=True, run_root=run_root)
        tr._accum_step, tr._accum_tokens = 0, 0
        d = R.LlamaDims(128, 256, 2, 4, 2, 32, 259)
        params = {n: t.detach().cpu().clone() for n, t in tr.store.named_master().items()}
        batch = tr.data_manager.generate_batch(0)
        loss, ntoks, _ = tr.train_step(0, batch)
    loss_ref, _, grads = R.loss_and_grads(params, batch, d, pad_token=256)
    out["loss"], out["loss_ref"] = float(loss), float(loss_ref)
    assert abs(out["loss"] - out["loss_ref"]) < 2e-2, out
    opt = R.MuonOracle(tr.lr_schedule)
    ref = dict(params)
    opt.update(ref, grads)
    new = {n: t.detach().cpu() for n, t in tr.store.named_master().items()}
    worst = 0.0
    for n in params:
        delta, delta_ref = new[n] - params[n], ref[n] - params[n]
        if delta_ref.norm() > 0:
            worst = max(worst, _rel(delta, delta_ref))
    out["worst_param_delta_rel"] = worst
    assert worst < 0.15, out   # bf16 fwd/bwd gradients through NS5; DESIGN.md §5 tolerances
    if verbose:
        print("smoke ok:", {k: (round(v, 5) if isinstance(v, float) else v) for k, v in out.items()})
    return out
