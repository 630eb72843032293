"""KV-cached generation on the GPU: the decode-attention kernel against fp64, its determinism, the cache append, the
model's prefill / decode steps against Model.forward and the fp64 oracle, greedy decoding, device sampling, and the
`python -m core.generation` CLI end to end."""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden" / "sampler_vectors.npz"
LENS = [1, 2, 255, 256, 257, 1000, 2048, 4095]
S_MAX = 4160
CANARY = 64


def _ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


def _decode_raw(q, kc, vc, lens, scale):
    """b200_attn_decode with o and lse inside canary-filled buffers; returns (o, lse, canaries intact)."""
    from mlx_cuda_distributed_pretraining_b200._lib import check, lib
    ops = _ops()
    B, H, D = q.shape
    Hk = kc.shape[2]
    obuf = torch.full((B * H * D + 2 * CANARY,), 1234.5, device=q.device, dtype=q.dtype)
    lbuf = torch.full((B * H + 2 * CANARY,), 1234.5, device=q.device, dtype=torch.float32)
    ws = torch.empty(ops.attention_decode_workspace_bytes(B, H, kc.shape[1], D), device=q.device, dtype=torch.uint8)
    check(lib().b200_attn_decode(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), lens.data_ptr(),
                                 obuf[CANARY:].data_ptr(), lbuf[CANARY:].data_ptr(), B, kc.shape[1], H, Hk, D,
                                 float(scale), int(q.dtype == torch.bfloat16), ws.data_ptr(), ws.numel(),
                                 torch.cuda.current_stream().cuda_stream), "b200_attn_decode")
    o = obuf[CANARY:CANARY + B * H * D].view(B, H, D)
    lse = lbuf[CANARY:CANARY + B * H].view(B, H)
    intact = bool((obuf[:CANARY] == 1234.5).all() and (obuf[-CANARY:] == 1234.5).all() and
                  (lbuf[:CANARY] == 1234.5).all() and (lbuf[-CANARY:] == 1234.5).all())
    return o, lse, intact


def _make_cache(lens, s_max, H, Hk, D, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B = len(lens)
    q = torch.randn(B, H, D, device="cuda", generator=g).to(dtype)
    kc = torch.randn(B, s_max, Hk, D, device="cuda", generator=g).to(dtype)
    vc = torch.randn(B, s_max, Hk, D, device="cuda", generator=g).to(dtype)
    for b, n in enumerate(lens):  # keys at or beyond lens[b] must never be read
        kc[b, n:] = float("nan")
        vc[b, n:] = float("nan")
    return q, kc, vc, torch.tensor(lens, device="cuda", dtype=torch.int32)


def _reference(q, kc, vc, lens, scale):
    """fp64 softmax(q K^T scale) V per row, plus sum_j |p_j| |v_j| for the error bound and the LSE."""
    B, H, D = q.shape
    Hk = kc.shape[2]
    out, absterm, lses = [], [], []
    for b, n in enumerate(lens):
        k = kc[b, :n].double().repeat_interleave(H // Hk, dim=1)  # [n, H, D]
        v = vc[b, :n].double().repeat_interleave(H // Hk, dim=1)
        s = torch.einsum("hd,nhd->hn", q[b].double(), k) * scale
        lse = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - lse[:, None])
        out.append(torch.einsum("hn,nhd->hd", p, v))
        absterm.append(torch.einsum("hn,nhd->hd", p.abs(), v.abs()))
        lses.append(lse)
    return torch.stack(out), torch.stack(absterm), torch.stack(lses)


# c of the bound 2^-8 |R| + c 2^-24 sum |p||v| (first term, the bf16 output rounding, for bf16 outputs only).  On an
# H100 the largest fp32 error/bound ratio was 0.077 (c ~ 5 would do); bf16 ratios reach 0.99, the rounding term.
C_BOUND = 64.0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("D", [16, 32, 64, 128])
@pytest.mark.parametrize("H,Hk", [(1, 1), (4, 1), (16, 8), (16, 16)])
def test_decode_attention_matches_fp64(dtype, D, H, Hk):
    scale = D ** -0.5
    q, kc, vc, lens = _make_cache(LENS, S_MAX, H, Hk, D, dtype, seed=D + H)
    o, lse, intact = _decode_raw(q, kc, vc, lens, scale)
    torch.cuda.synchronize()
    assert intact, "decode attention wrote outside o / lse"
    R, absterm, lse_ref = _reference(q, kc, vc, LENS, scale)
    err = (o.double() - R).abs()
    bound = C_BOUND * 2.0 ** -24 * absterm + (2.0 ** -8 * R.abs() if dtype == torch.bfloat16 else 0)
    ratio = float((err / bound).max())
    print(f"max error/bound {ratio:.3f} ({dtype}, D={D}, H={H}, Hk={Hk})")
    assert torch.isfinite(o).all()
    assert ratio <= 1.0
    assert float((lse.double() - lse_ref).abs().max()) < 1e-4 * max(1.0, float(lse_ref.abs().max()))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_decode_attention_batch_invariant_and_repeatable(dtype):
    ops = _ops()
    H, Hk, D = 16, 8, 64
    lens = [2048, 5, 257, 1000, 4095, 256, 31]
    q, kc, vc, lt = _make_cache(lens, S_MAX, H, Hk, D, dtype, seed=3)
    o_batch = ops.attention_decode(q, kc, vc, lt)
    again = ops.attention_decode(q, kc, vc, lt)
    assert torch.equal(o_batch, again)
    for b in range(len(lens)):
        alone = ops.attention_decode(q[b:b + 1].contiguous(), kc[b:b + 1].contiguous(), vc[b:b + 1].contiguous(),
                                     lt[b:b + 1].contiguous())
        assert torch.equal(alone[0], o_batch[b]), f"row {b} differs alone vs in the batch"
    # a smaller cache (s_max only changes the grid, never a row's chunks)
    small = ops.attention_decode(q[:1].contiguous(), kc[:1, :2048].contiguous(), vc[:1, :2048].contiguous(),
                                 lt[:1].contiguous())
    assert torch.equal(small[0], o_batch[0])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("rope", [False, True], ids=["norope", "rope"])
def test_kv_append_matches_rope(dtype, rope):
    ops = _ops()
    B, H, Hk, D, s_max = 5, 8, 2, 64, 300
    pos = [0, 7, 299, 128, 31]
    g = torch.Generator(device="cuda").manual_seed(11)
    q = torch.randn(B, H, D, device="cuda", generator=g).to(dtype)
    k = torch.randn(B, Hk, D, device="cuda", generator=g).to(dtype)
    v = torch.randn(B, Hk, D, device="cuda", generator=g).to(dtype)
    kc = torch.full((B, s_max, Hk, D), 7.0, device="cuda", dtype=dtype)
    vc = torch.full((B, s_max, Hk, D), 7.0, device="cuda", dtype=dtype)
    lens = torch.tensor([p + 1 for p in pos], device="cuda", dtype=torch.int32)
    tables = ops.rope_tables(512, D, 10000.0, "cuda") if rope else None
    q_in = q.clone()
    ops.kv_append(q, k, v, kc, vc, lens, tables)
    torch.cuda.synchronize()
    written = torch.zeros(B, s_max, dtype=torch.bool)
    for b, p in enumerate(pos):
        if rope:
            cos_t, sin_t = tables
            want_k = ops.rope(k[b][None, None], cos_t[p:p + 1], sin_t[p:p + 1])[0, 0]
            want_q = ops.rope(q_in[b][None, None], cos_t[p:p + 1], sin_t[p:p + 1])[0, 0]
            assert torch.equal(q[b], want_q)
        else:
            want_k = k[b]
        assert torch.equal(kc[b, p], want_k)
        assert torch.equal(vc[b, p], v[b])
        written[b, p] = True
    if not rope:
        assert torch.equal(q, q_in)
    rest = ~written.cuda()
    assert bool((kc[rest] == 7.0).all()) and bool((vc[rest] == 7.0).all()), "append wrote outside [b, pos[b]]"


# -- model level ----------------------------------------------------------------------------------------------------
def _cfg(kind: str):
    from tests.smoke_check import tiny_config
    if kind == "c1_fp32":   # C1's shape: hidden 128, 4 layers, 8 heads of 16, fp32
        c = tiny_config(name="gen-c1", optimizer="adamw", mixed=False)
        c["model"]["dimensions"].update(hidden_size=128, intermediate_size=256, num_layers=4)
        c["model"]["attention"].update(num_heads=8, num_kv_heads=8, head_dim=16, max_position_embeddings=1024)
        return c
    c = tiny_config(name=f"gen-{kind}", optimizer="adamw", mixed=True)
    c["model"]["attention"].update(num_heads=4, num_kv_heads=2, head_dim=64, max_position_embeddings=1024)
    c["model"]["rope"]["enabled"] = kind == "bf16_rope"
    return c


def _trainer(kind: str):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    tmp = tempfile.mkdtemp(prefix="gen_runs_")
    return Trainer(Config.from_dict(_cfg(kind)), for_training=False, synthetic=True, quiet=True, run_root=tmp)


def _oracle_logits(tr, tokens):
    from oracle import reference_math as R
    a = tr.model_args
    d = R.LlamaDims(a.hidden_size, a.intermediate_size, a.num_hidden_layers, a.num_attention_heads,
                    a.num_key_value_heads, a.head_dim, a.vocab_size, a.rms_norm_eps, a.rope_theta, a.apply_rope, True)
    params = {n: t.detach().double().cpu() for n, t in tr.store.named_master().items()}
    return R.llama_forward(params, tokens.cpu(), d)


# logits tolerance, relative to the row's largest |logit|.  bf16: activations rounded to bf16 at every layer.  fp32:
# the training forward's bf16x3 attention itself sits ~2e-3 from the fp64 oracle (the cached path ~1.4e-3).
TOL = {"c1_fp32": 5e-3, "bf16_gqa": 3e-2, "bf16_rope": 3e-2}


def _rel_rows(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float(((a - b).abs().amax(-1) / b.abs().amax(-1).clamp_min(1e-6)).max())


@pytest.mark.parametrize("kind", ["c1_fp32", "bf16_gqa", "bf16_rope"])
def test_prefill_decode_match_forward_and_oracle(kind):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    tr = _trainer(kind)
    model = tr.model
    T, t0 = 300, 260      # prompt crosses the 256-key chunk boundary during decoding
    g = torch.Generator().manual_seed(5)
    tokens = torch.randint(0, 256, (2, T), generator=g)
    with torch.no_grad():
        full = model(tokens.cuda()).float()
    oracle = _oracle_logits(tr, tokens)
    cache = KVCache(model, 2, T)
    got = [model.prefill(tokens[:, :t0].cuda(), [t0, t0], cache)]
    for t in range(t0, T - 1):
        got.append(model.decode_step(tokens[:, t].cuda(), cache))
    got = torch.stack(got, dim=1)                          # logits after positions t0-1 .. T-2
    e_fwd = _rel_rows(got, full[:, t0 - 1:T - 1])
    e_orc = _rel_rows(got, oracle[:, t0 - 1:T - 1])
    e_fwd_orc = _rel_rows(full[:, t0 - 1:T - 1], oracle[:, t0 - 1:T - 1])
    print(f"{kind}: cached vs forward {e_fwd:.2e}, cached vs fp64 oracle {e_orc:.2e}, forward vs oracle {e_fwd_orc:.2e}")
    assert e_fwd < TOL[kind]
    assert e_orc < max(TOL[kind], 2 * e_fwd_orc)


@pytest.mark.parametrize("kind", ["c1_fp32", "bf16_rope"])
def test_ragged_batch_rows_match_alone(kind):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    tr = _trainer(kind)
    model = tr.model
    g = torch.Generator().manual_seed(9)
    prompts = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (3, 40, 300)]
    steps = 6
    cont = torch.randint(0, 256, (len(prompts), steps), generator=g)

    def run(rows):
        S = max(len(prompts[r]) for r in rows)
        toks = torch.zeros((len(rows), S), dtype=torch.int64)
        for i, r in enumerate(rows):
            toks[i, :len(prompts[r])] = torch.tensor(prompts[r])
        cache = KVCache(model, len(rows), S + steps)
        out = [model.prefill(toks.cuda(), [len(prompts[r]) for r in rows], cache)]
        for s in range(steps):
            out.append(model.decode_step(cont[rows, s].cuda(), cache))
        return torch.stack(out, 1)

    batch = run([0, 1, 2])
    for r in range(3):
        alone = run([r])[0]
        err = _rel_rows(batch[r], alone)
        print(f"{kind} row {r}: batch vs alone {err:.2e}")
        assert err < TOL[kind] / 4


def test_greedy_cache_matches_full_forward():
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    tr = _trainer("bf16_gqa")
    model = tr.model
    prompt = [tr.tokenizer.BOS_TOKEN] + list(range(40, 80))
    n = 48
    out = generate(model, [prompt], max_tokens=n, temperature=0, repetition_penalty=1.0, min_p=None)[0]
    seq = list(prompt)
    skipped = 0
    for i, t in enumerate(out):
        with torch.no_grad():
            logits = model(torch.tensor([seq], device="cuda")).float()[0, -1]
        top2 = torch.topk(logits, 2).values
        if float(top2[0] - top2[1]) <= TOL["bf16_gqa"] * float(logits.abs().max()):
            skipped += 1       # near-tie: either choice is within the logits tolerance
        else:
            assert t == int(torch.argmax(logits)), f"step {i}"
        seq.append(t)        # follow the cached run's choice either way
    print(f"greedy: {n} steps, {skipped} skipped as near-ties")
    assert skipped < n // 2


def test_device_sampling_matches_fixture_and_seed_reproduces():
    from mlx_cuda_distributed_pretraining_b200.core import generation as G
    z = np.load(GOLDEN)
    keys = sorted({k.split("_")[0] for k in z.files if k.startswith("s")})
    for key in keys:
        lp = torch.tensor(z[f"{key}_logprobs"], device="cuda")
        kind, temp, param = str(z[f"{key}_kind"]), float(z[f"{key}_temp"]), float(z[f"{key}_param"])
        got = G.sampling_distribution(lp, temp, min_p=param if kind == "min_p" else None,
                                      top_p=param if kind == "top_p" else None).cpu().numpy()
        np.testing.assert_allclose(got, _fixture_distribution(z, key), rtol=0, atol=1e-6, err_msg=key)
    tr = _trainer("bf16_gqa")
    runs = [G.generate(tr.model, [[1, 2, 3], [4, 5]], max_tokens=20, temperature=1.0, seed=123) for _ in range(2)]
    assert runs[0] == runs[1]


def _fixture_distribution(z, key):
    """The fixture's filtered distribution in vocabulary order."""
    dist = z[f"{key}_dist"].astype(np.float64)
    order = z[f"{key}_order"]
    p = np.exp(dist - dist.max())
    p = p / p.sum()
    if str(z[f"{key}_kind"]) == "plain":
        return p
    out = np.zeros_like(p)
    out[order] = p
    return out


def test_cli_end_to_end():
    env = dict(os.environ, PYTHONPATH=str(ROOT) + os.pathsep + os.environ.get("PYTHONPATH", ""))
    with tempfile.TemporaryDirectory(prefix="gen_e2e_") as tmp:
        cfg = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
        cfg["name"] = "gen-e2e"
        cfg["data"]["input_file"] = "synthetic:markov"
        cfg["data"]["preprocessing"]["max_context_size"] = 128
        cfg["training"]["hyperparameters"]["iters"] = 4
        cfg["logging"]["steps"]["logging_interval"] = 1
        cfg_path = Path(tmp) / "cfg.yaml"
        cfg_path.write_text(yaml.safe_dump(cfg))
        subprocess.run([sys.executable, "-m", "core.training", "--config", str(cfg_path)], cwd=tmp, env=env,
                       check=True, timeout=600)
        saved = Path(tmp) / "runs" / "gen-e2e" / "config.yaml"
        assert saved.is_file()
        assert yaml.safe_load(saved.read_text())["data"]["input_file"] == "synthetic:markov"
        base = [sys.executable, "-m", "core.generation", "--run", "gen-e2e", "--runs-dir", str(Path(tmp) / "runs"),
                "--prompt", "hello", "--max-tokens", "24"]
        outs = [subprocess.run(base + ["--seed", "0", "--temperature", "0"], cwd=ROOT, env=env, check=True,
                               capture_output=True, text=True, timeout=600).stdout for _ in range(2)]
        lines = [l for l in outs[0].splitlines() if l.startswith("Greedy Output: ")]
        assert len(lines) == 1 and outs[0] == outs[1]
        four = subprocess.run(base + ["--seed", "1", "--num-samples", "4"], cwd=ROOT, env=env, check=True,
                              capture_output=True, text=True, timeout=600).stdout
        assert sum(l.startswith("Greedy Output: ") for l in four.splitlines()) == 4
