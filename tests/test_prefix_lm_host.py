"""Prefix-LM on the host: the `model.attention.prefix_lm` config key and the combinations it rejects, the prompt /
completion and split-point prefix sources, the target masking, PrefixCausalMask.dense() against the definition, the
exporter's refusal, and the fp64 attention checkers (tests/attn_fwd_check.py, tests/attn_bwd_check.py) under the prefix
mask: they accept the exact result and reject single faults of the mask."""
import copy
import json
import types
from pathlib import Path

import pytest
import torch
import yaml

from tests import attn_bwd_check as ac
from tests import attn_fwd_check as fc

ROOT = Path(__file__).resolve().parents[1]


def _c1():
    return yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())


# ---- config ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("good", [True, False, None])
def test_config_accepts_prefix_lm(good):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    d = _c1()
    d["model"]["attention"]["prefix_lm"] = good
    assert Config.from_dict(copy.deepcopy(d)).model.attention["prefix_lm"] is good
    assert "prefix_lm" not in Config.from_dict(_c1()).model.attention


@pytest.mark.parametrize("bad", [1, 0, "true", 1.0, [True]])
def test_config_rejects_non_bool_prefix_lm(bad):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    d = _c1()
    d["model"]["attention"]["prefix_lm"] = bad
    with pytest.raises(ValueError, match="prefix_lm"):
        Config.from_dict(d)


@pytest.mark.parametrize("key", ["sliding_window", "alibi", "pack_sequences"])
def test_config_rejects_combinations(key):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    d = _c1()
    d["model"]["attention"]["prefix_lm"] = True
    if key == "pack_sequences":
        d["data"]["preprocessing"]["pack_sequences"] = True
    else:
        d["model"]["attention"][key] = 64 if key == "sliding_window" else True
    with pytest.raises(ValueError, match=key):
        Config.from_dict(d)
    d2 = copy.deepcopy(d)
    d2["model"]["attention"]["prefix_lm"] = False
    Config.from_dict(d2)


# ---- data -----------------------------------------------------------------------------------------------------------
def _data_manager(tmp_path, lines, prefix_lm=True, ctx=64, overlap=0, bs=2, val=False):
    from mlx_cuda_distributed_pretraining_b200.core.training import DataConfig, DataManager, TokenizerManager
    f = tmp_path / "d.jsonl"
    f.write_text("".join(json.dumps(x) + "\n" for x in lines))
    cfg = DataConfig(input_file=str(f), validation_file=str(f) if val else None,
                     preprocessing={"max_context_size": ctx, "chunk_overlap": overlap},
                     tokenizer={"normal_vocab_size": 256,
                                "special_tokens": {"pad": "<pad>", "bos": "<bos>", "eos": "<eos>"}})
    tok = TokenizerManager(cfg)
    return DataManager(cfg, tok, bs, prefix_lm=prefix_lm), tok


def test_prompt_completion_rows_and_prefix(tmp_path):
    dm, tok = _data_manager(tmp_path, [{"prompt": "ab", "completion": "xyz"}, {"prompt": "hello", "completion": "!"}])
    assert sorted(dm.train_docs) == [("ab", "xyz"), ("hello", "!")]
    b = dm._create_batch([("ab", "xyz"), ("hello", "!")])
    B, E, PAD = tok.BOS_TOKEN, tok.EOS_TOKEN, tok.PAD_TOKEN
    assert b[:, 0].tolist() == [3, 6]
    assert b[0, 1:].tolist() == [B, 97, 98, 120, 121, 122, E, PAD]
    assert b[1, 1:].tolist() == [B, 104, 101, 108, 108, 111, 33, E]


def test_pairs_are_not_chunked_and_prefix_is_clipped(tmp_path):
    prompt, comp = "p" * 30, "c" * 30
    dm, _ = _data_manager(tmp_path, [{"prompt": prompt, "completion": comp}, {"text": "t" * 50}], ctx=16, overlap=0)
    assert ("p" * 30, "c" * 30) in dm.train_docs
    assert sum(isinstance(d, str) for d in dm.train_docs) == 4          # the text line is chunked by 16
    b = dm._create_batch([(prompt, comp)])
    assert b.shape == (1, 1 + 16) and int(b[0, 0]) == 16                # row truncated, P = 31 clipped to it


def test_text_rows_without_prefix_lm_are_unchanged(tmp_path):
    lines = [{"text": "the quick brown fox"}, {"text": "jumps"}]
    on, _ = _data_manager(tmp_path, lines, prefix_lm=True)
    off, _ = _data_manager(tmp_path, lines, prefix_lm=False)
    docs = ["the quick brown fox", "jumps"]
    a, b = on._create_batch(docs, 123), off._create_batch(docs)
    assert torch.equal(a[:, 1:], b)
    n_in = [min(len(x), b.shape[1] - 1) for x in ([0] * 21, [0] * 7)]
    assert all(0 <= int(a[i, 0]) <= n_in[i] for i in range(2))


def test_prefix_targets_mask_before_p_minus_1():
    from mlx_cuda_distributed_pretraining_b200.core.training import prefix_targets
    t = torch.arange(10).repeat(4, 1) + 100
    out = prefix_targets(t, torch.tensor([0, 1, 2, 7]), -1)
    assert out[0].tolist() == t[0].tolist() and out[1].tolist() == t[1].tolist()
    assert out[2].tolist() == [-1] + t[2, 1:].tolist()                    # target at P - 1 = 1 is kept
    assert out[3, :6].eq(-1).all() and out[3, 6:].tolist() == t[3, 6:].tolist()


def test_split_points_reproducible_and_uniform():
    from mlx_cuda_distributed_pretraining_b200.core.training import split_points, train_split_seed, val_split_seed
    a = split_points([50] * 8, train_split_seed(3, 1))
    assert torch.equal(a, split_points([50] * 8, train_split_seed(3, 1)))
    assert not torch.equal(a, split_points([50] * 8, train_split_seed(3, 0)))
    assert not torch.equal(a, split_points([50] * 8, train_split_seed(4, 1)))
    assert torch.equal(split_points([9] * 4, val_split_seed(2)), split_points([9] * 4, val_split_seed(2)))
    big = split_points([4] * 20000, 7)
    counts = torch.bincount(big, minlength=5).double() / 20000
    assert int(big.min()) == 0 and int(big.max()) == 4 and float((counts - 0.2).abs().max()) < 0.02
    assert split_points([0, 0], 1).tolist() == [0, 0]


def test_validation_split_points_follow_the_batch_index(tmp_path):
    lines = [{"text": "x" * (10 + i)} for i in range(6)]
    dm, _ = _data_manager(tmp_path, lines, val=True)
    first = [dm.generate_validation_batch(i) for i in range(3)]
    dm.val_ptr = 0
    again = [dm.generate_validation_batch(i) for i in range(3)]
    assert all(torch.equal(x, y) for x, y in zip(first, again))


@pytest.mark.parametrize("kind", ["uniform", "markov"])
def test_synthetic_stream_identical_with_prefix_lm(kind):
    from mlx_cuda_distributed_pretraining_b200.core.training import SyntheticData
    on = SyntheticData(300, 4, 64, rank=1, kind=kind, prefix_lm=True)
    off = SyntheticData(300, 4, 64, rank=1, kind=kind)
    for step in (0, 5):
        a, b = on.generate_batch(step), off.generate_batch(step)
        assert a.shape == (4, 1 + 65) and torch.equal(a[:, 1:], b)
        assert bool(((a[:, 0] >= 0) & (a[:, 0] <= 64)).all())
        assert torch.equal(a, on.generate_batch(step))


# ---- mask and exporter ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 7, 130])
def test_prefix_mask_dense_matches_definition(S):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import PrefixCausalMask
    Ps = [0, 1, S - 1, S]
    m = PrefixCausalMask(torch.tensor(Ps, dtype=torch.int32), S).dense()
    assert m.shape == (4, 1, S, S)
    for b, P in enumerate(Ps):
        for q in range(S):
            for k in range(S):
                want = 0.0 if (k <= q or k < P) else float("-inf")
                assert float(m[b, 0, q, k]) == want
    causal = torch.triu(torch.full((S, S), float("-inf")), diagonal=1)
    assert torch.equal(m[0, 0], causal) and torch.equal(m[1, 0], causal)
    assert torch.equal(m[3, 0], torch.zeros(S, S))


def test_exporter_refuses_prefix_lm_runs():
    from mlx_cuda_distributed_pretraining_b200.tools.export import check_exportable
    m = types.SimpleNamespace(misc={"variant": "mlx_lm"}, rope={"traditional": False}, attention={"prefix_lm": True})
    with pytest.raises(ValueError, match="prefix_lm"):
        check_exportable(m)
    m.attention = {"prefix_lm": False}
    check_exportable(m)


# ---- the fp64 checkers under the prefix mask ------------------------------------------------------------------------
def visible(S, prefix):
    P = torch.as_tensor(prefix, dtype=torch.int64).clamp(0, S)
    s = torch.arange(S)
    return (s[None, :] <= s[:, None])[None] | (s[None, None, :] < P[:, None, None])


def _inputs(B, S, H, Hk, D, seed):
    g = torch.Generator().manual_seed(seed)
    return tuple(torch.randn(B, S, h, D, generator=g).to(torch.bfloat16) for h in (H, Hk, Hk))


PREFIX = [0, 100, 129, 200]
S_CHK, D_CHK = 260, 64


def _faulty_masks():
    """Single faults of a prefix kernel's mask, each as the mask it would apply."""
    S = S_CHK
    s = torch.arange(S)
    good = visible(S, PREFIX)
    off_by_one = visible(S, [p + 1 for p in PREFIX])                      # k <= P instead of k < P
    first_tile = good & ~((s[None, None, :] >= 128) & (s[None, None, :] > s[None, :, None]))  # prefix on tile 0 only
    crossing = good.clone()                                               # causal mask kept on the tile crossing P
    for b, P in enumerate(PREFIX):
        t0 = (P // 128) * 128
        if 0 < P < S and P % 128:
            cols = torch.arange(t0, P)
            crossing[b][:, cols] = (cols[None, :] <= s[:, None])
    return {"k<=P": off_by_one, "first tile only": first_tile, "crossing tile causal": crossing}


def test_fwd_checker_accepts_exact_and_rejects_mask_faults():
    q, k, v = _inputs(len(PREFIX), S_CHK, 4, 2, D_CHK, seed=1)
    good = visible(S_CHK, PREFIX)
    ref = fc.reference(q, k, v, D_CHK ** -0.5, good)
    o, lse = fc.forward64(q, k, v, D_CHK ** -0.5, good)
    assert fc.check("exact o", o.to(torch.bfloat16), *ref["o"]) < 1.0
    assert fc.check("exact lse", lse.float(), *ref["lse"]) < 1.0
    for name, bad in _faulty_masks().items():
        ob, lb = fc.forward64(q, k, v, D_CHK ** -0.5, bad)
        with pytest.raises(AssertionError):
            fc.check(name, ob.to(torch.bfloat16), *ref["o"])
            fc.check(name, lb.float(), *ref["lse"])


def test_bwd_checker_rejects_a_causal_query_range_below_p():
    """A backward whose key tiles below P start their query range at the causal k0 / BQ misses the dK / dV terms of
    the earlier queries that see those keys; the reference with that range dropped must fall outside the bound."""
    B, H, Hk = len(PREFIX), 4, 2
    q, k, v = _inputs(B, S_CHK, H, Hk, D_CHK, seed=2)
    g = torch.Generator().manual_seed(3)
    do = torch.randn(B, S_CHK, H, D_CHK, generator=g).to(torch.bfloat16)
    good = visible(S_CHK, PREFIX)
    o, lse = fc.forward64(q, k, v, D_CHK ** -0.5, good)
    o, lse = o.to(torch.bfloat16), lse.float()
    ref = ac.reference(q, k, v, o, do, lse, D_CHK ** -0.5, False, mask=good)
    for name in ("dq", "dk", "dv"):
        assert ac.check(f"exact {name}", ref[name][0].to(torch.bfloat16), *ref[name]) < 1.0
    s = torch.arange(S_CHK)
    kt0 = (s // 128) * 128                          # first key of each key's 128-key tile
    causal_range = (s[:, None] >= (kt0 // 64 * 64)[None, :])              # query tile >= k0 / BQ
    bad = good & causal_range[None]
    faulty = ac.reference(q, k, v, o, do, lse, D_CHK ** -0.5, False, mask=bad)
    with pytest.raises(AssertionError):
        for name in ("dk", "dv"):
            ac.check(f"causal range {name}", faulty[name][0].to(torch.bfloat16), *ref[name])


def test_line_without_text_or_pair_names_the_keys(tmp_path):
    with pytest.raises(ValueError, match='"prompt" and "completion"'):
        _data_manager(tmp_path, [{"prompt": "only a prompt"}])
    with pytest.raises(ValueError, match='expected "text"'):
        _data_manager(tmp_path, [{"prompt": "a", "completion": "b"}], prefix_lm=False)


class _TinyLM(torch.nn.Module):
    """A CPU stand-in for Model on compute_loss's unfused path: logits from the inputs alone."""

    def __init__(self, vocab=259):
        super().__init__()
        self.emb = torch.nn.Embedding(vocab, 8)
        self.out = torch.nn.Linear(8, vocab)

    def forward(self, inputs, prefix_lens=None):
        return self.out(self.emb(inputs))


def test_batches_without_targets_give_a_finite_loss_and_gradient(tmp_path):
    """A prompt that fills the row (P clipped to it) and a text row whose split point is its input length keep no
    target.  A micro-batch of such rows has loss 0, zero finite gradients and ntoks 0; mixed with an ordinary row the
    loss is that row's alone."""
    from mlx_cuda_distributed_pretraining_b200.core.training import Trainer
    dm, tok = _data_manager(tmp_path, [{"text": "x"}], ctx=16)
    long_pair = dm._create_batch([("p" * 30, "c" * 30)])
    assert int(long_pair[0, 0]) == 16
    # [BOS] hello [EOS] padded by a longer row: 7 non-PAD inputs, the last one EOS with a PAD target
    text = dm._create_batch(["hello", "hello world!"])[:1].clone()
    text[0, 0] = 7                                        # the split point at n_b
    ordinary = dm._create_batch([("ab", "cdef")])
    cfg = types.SimpleNamespace(model=types.SimpleNamespace(attention={"max_position_embeddings": 64}))
    fake = types.SimpleNamespace(config=cfg, tokenizer=tok, model_args=None)
    model = _TinyLM()
    for rows, want_tokens in (([long_pair], 0), ([text], 0), ([long_pair, text], 0), ([ordinary], 5)):
        width = max(r.shape[1] for r in rows)
        batch = torch.cat([torch.nn.functional.pad(r, (0, width - r.shape[1]), value=tok.PAD_TOKEN) for r in rows])
        P, toks = batch[:, 0], batch[:, 1:]
        model.zero_grad(set_to_none=True)
        loss, ntoks = Trainer.compute_loss(fake, model, toks[:, :-1], toks[:, 1:], prefix=P)
        loss.backward()
        assert int(ntoks) == want_tokens and torch.isfinite(loss)
        grads = [p.grad for p in model.parameters()]
        assert all(torch.isfinite(g).all() for g in grads)
        if want_tokens == 0:
            assert float(loss.detach()) == 0.0 and all(float(g.abs().max()) == 0.0 for g in grads)
    mixed = torch.cat([ordinary, torch.nn.functional.pad(long_pair, (0, 0))[:, :ordinary.shape[1]]])
    loss_m, n_m = Trainer.compute_loss(fake, model, mixed[:, 1:-1], mixed[:, 2:], prefix=mixed[:, 0])
    loss_o, n_o = Trainer.compute_loss(fake, model, ordinary[:, 1:-1], ordinary[:, 2:], prefix=ordinary[:, 0])
    assert int(n_m) == int(n_o) == 5 and torch.allclose(loss_m, loss_o)
