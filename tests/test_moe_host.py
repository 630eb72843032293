"""Sparse MoE MLP (`model.misc.num_local_experts`) on the host: config validation and round trip, parameter names
and the flat store's grouping, the fp64 oracle (tests/moe_oracle.py) pinned against transformers' Mixtral, the
Mixtral export, and a CPU emulation of the routing kernels' index arithmetic with the faults it must reject."""
import copy
import json

import pytest
import torch
import yaml

from tests import moe_oracle as mo
from tests.test_llama_variant_host import THETA, _c1, _dims, _params


def _moe_dict(E=8, k=2, **misc):
    d = _c1()
    d["model"]["misc"].update(num_local_experts=E, num_experts_per_tok=k, **misc)
    d["system"]["mixed_precision"] = True
    return d


def _cfg(d):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    return Config.from_dict(copy.deepcopy(d))


# ---- config -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E,k", [(None, None), (0, 0), (0, None), (2, 1), (2, 2), (8, 2), (64, 8), (16, 8)])
def test_config_accepts(E, k):
    c = _cfg(_moe_dict(E, k))
    assert c.model.misc["num_local_experts"] == E


@pytest.mark.parametrize("E,k,match", [
    (1, 1, "num_local_experts"), (65, 2, "num_local_experts"), (-2, 1, "num_local_experts"),
    (8, 0, "num_experts_per_tok"), (8, 9, "num_experts_per_tok"), (4, 5, "num_experts_per_tok"),
    (0, 2, "num_experts_per_tok"), (True, 1, "num_local_experts"), (8.0, 2, "num_local_experts"),
    ("8", 2, "num_local_experts"), (8, 2.0, "num_experts_per_tok"), (8, True, "num_experts_per_tok"),
    (8, "2", "num_experts_per_tok"),
])
def test_config_rejects(E, k, match):
    with pytest.raises(ValueError, match=match):
        _cfg(_moe_dict(E, k))


@pytest.mark.parametrize("c", [0, 0.0, 0.001, 1, 2.5])
def test_config_accepts_aux_coef(c):
    assert _cfg(_moe_dict(router_aux_loss_coef=c)).model.misc["router_aux_loss_coef"] == c


@pytest.mark.parametrize("c", [-0.1, float("nan"), float("inf"), "0.01", True, None])
def test_config_rejects_aux_coef(c):
    with pytest.raises(ValueError, match="router_aux_loss_coef"):
        _cfg(_moe_dict(router_aux_loss_coef=c))


def test_config_rejects_bias_shampoo_and_fp32():
    with pytest.raises(ValueError, match="mlp_bias"):
        _cfg(_moe_dict(mlp_bias=True))
    d = _moe_dict()
    d["training"]["optimization"]["optimizer"] = "shampoo"
    with pytest.raises(ValueError, match="[Ss]hampoo"):
        _cfg(d)
    d["training"]["optimization"].update(optimizer="hybrid", matrix_optimizer="shampoo")
    with pytest.raises(ValueError, match="[Ss]hampoo"):
        _cfg(d)
    d = _moe_dict(4, 2)
    d["training"]["optimization"]["optimizer"] = "muon"   # E % 8 != 0: the router goes to Muon's elementwise side
    _cfg(d)
    d["model"]["dimensions"]["intermediate_size"] = 96
    with pytest.raises(ValueError, match="multiple of 64"):
        _cfg(d)
    d = _moe_dict()
    d["system"]["mixed_precision"] = False
    with pytest.raises(ValueError, match="mixed_precision"):
        _cfg(d)
    d = _c1()   # a dense config keeps every one of these
    d["model"]["misc"]["mlp_bias"] = True
    d["training"]["optimization"]["optimizer"] = "shampoo"
    _cfg(d)


def test_config_yaml_round_trip(tmp_path):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    from dataclasses import asdict
    d = _moe_dict(4, 2, router_aux_loss_coef=0.02)
    c = _cfg(d)
    p = tmp_path / "config.yaml"
    p.write_text(yaml.safe_dump(asdict(c), sort_keys=False))
    misc = Config.from_yaml(str(p)).model.misc
    assert (misc["num_local_experts"], misc["num_experts_per_tok"], misc["router_aux_loss_coef"]) == (4, 2, 0.02)


# ---- model and flat store -------------------------------------------------------------------------------------
def _model(E=4, k=2, variant="mlx_lm"):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    return Model(ModelArgs(model_type="llama", hidden_size=32, num_hidden_layers=2, intermediate_size=24,
                           num_attention_heads=2, vocab_size=16, variant=variant, num_local_experts=E,
                           num_experts_per_tok=k))


def test_parameter_names_and_shapes():
    m = _model()
    shapes = {n: tuple(p.shape) for n, p in m.named_parameters()}
    assert shapes["layers.1.block_sparse_moe.gate.weight"] == (4, 32)
    assert shapes["layers.1.block_sparse_moe.switch_mlp.gate_proj.weight"] == (4, 24, 32)
    assert shapes["layers.1.block_sparse_moe.switch_mlp.up_proj.weight"] == (4, 24, 32)
    assert shapes["layers.1.block_sparse_moe.switch_mlp.down_proj.weight"] == (4, 32, 24)
    assert not any(".mlp." in n for n in shapes)
    assert m.layers[0].block_sparse_moe.act == "silu" and _model(variant=None).layers[0].block_sparse_moe.act == \
        "sigmoid2"
    dense = _model(E=0, k=0)
    assert not any("block_sparse_moe" in n for n, _ in dense.named_parameters())


def test_init_matches_dense_linear_bound():
    from mlx_cuda_distributed_pretraining_b200.core.training import init_model_
    m = _model()
    init_model_(m, m.args, seed=1)
    w = m.layers[0].block_sparse_moe.switch_mlp.down_proj.weight
    w = w.detach()
    assert float(w.abs().max()) <= 24 ** -0.5 and float(w.abs().max()) > 0.9 * 24 ** -0.5
    assert float(w[0].std()) > 0 and not torch.equal(w[0], w[1])


def test_param_store_groups_experts_as_matrices():
    from mlx_cuda_distributed_pretraining_b200.flat import ParamStore
    m = _model()
    st = ParamStore(m, torch.float32, "cpu")
    g = next(g for g in st.mat_groups if (g.rows, g.cols) == (24, 32))
    name = "layers.0.block_sparse_moe.switch_mlp.gate_proj.weight"
    assert g.names.count(name) == 4 and g.batch == 16     # gate and up of 2 layers, 4 experts each
    assert st.index[name][1] == (4, 24, 32)
    p = dict(m.named_parameters())[name]
    assert p.shape == (4, 24, 32) and p.grad.shape == (4, 24, 32)
    gv = st.group_view(st.grad, g)
    p.grad[2, 5, 7] = 3.0                                 # the .grad view aliases the flat buffer, expert by expert
    i = g.names.index(name)
    assert float(gv[i + 2, 5, 7]) == 3.0
    assert p.data.data_ptr() == st.group_view(st.master, g)[i].data_ptr()
    router = "layers.0.block_sparse_moe.gate.weight"           # E = 4 rows: kept with the elementwise parameters
    assert tuple(st.index[router][1]) == (4, 32) and any(e.name == router for e in st.vec_entries)
    st8 = ParamStore(_model(E=8), torch.float32, "cpu")       # E = 8: a matrix like every other [rows, hidden]
    assert not any(e.name == router for e in st8.vec_entries) and any(g.rows == 8 for g in st8.mat_groups)


# ---- the pin: transformers' Mixtral --------------------------------------------------------------------------------
@pytest.fixture
def mixtral_fp64(monkeypatch):
    """transformers' Mixtral in full fp64: its router softmax (`.float()`), RMSNorm variance and RoPE angles are
    computed in fp32 even in an fp64 model; the three are restated in fp64 so the pin can hold to 1e-10."""
    pytest.importorskip("transformers")
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    from transformers.models.mixtral import modeling_mixtral as mm

    def router(self, h):
        h = h.reshape(-1, self.hidden_dim)
        p = torch.softmax(torch.nn.functional.linear(h, self.weight), dim=-1)
        top, idx = torch.topk(p, self.top_k, dim=-1)
        return p, top / top.sum(-1, keepdim=True), idx

    def norm(self, h):
        return self.weight * (h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + self.variance_epsilon))

    def rot(self, x, position_ids):
        D = self.inv_freq.numel() * 2
        inv = THETA ** (-torch.arange(0, D, 2, dtype=torch.float64) / D)
        emb = torch.cat([position_ids[:, :, None].double() * inv] * 2, -1)
        return emb.cos().to(x.dtype), emb.sin().to(x.dtype)

    monkeypatch.setattr(mm.MixtralTopKRouter, "forward", router)
    monkeypatch.setattr(mm.MixtralRMSNorm, "forward", norm)
    monkeypatch.setattr(mm.MixtralRotaryEmbedding, "forward", rot)
    return mm


def _mixtral_config(H, I, L, nh, nkv, hd, V, tied, E, k):
    from transformers import MixtralConfig
    return MixtralConfig(vocab_size=V, hidden_size=H, intermediate_size=I, num_hidden_layers=L, num_attention_heads=nh,
                         num_key_value_heads=nkv, head_dim=hd, rms_norm_eps=1e-5, rope_theta=THETA,
                         tie_word_embeddings=tied, num_local_experts=E, num_experts_per_tok=k, router_jitter_noise=0.0,
                         max_position_embeddings=64, sliding_window=None, experts_implementation="eager")


def _expert_params(E, I, H, seed):
    g = torch.Generator().manual_seed(seed)
    s = H ** -0.5
    return (torch.randn(E, H, generator=g, dtype=torch.float64) * 2 * s,
            torch.randn(E, I, H, generator=g, dtype=torch.float64) * s,
            torch.randn(E, I, H, generator=g, dtype=torch.float64) * s,
            torch.randn(E, H, I, generator=g, dtype=torch.float64) * I ** -0.5)


@pytest.mark.parametrize("E,k", [(2, 1), (2, 2), (8, 1), (8, 2), (8, 8), (64, 2), (64, 8)])
def test_oracle_block_matches_mixtral_block(mixtral_fp64, E, k):
    H, I, T = 32, 24, 37
    cfg = _mixtral_config(H, I, 1, 2, 2, 16, 16, True, E, k)
    blk = mixtral_fp64.MixtralSparseMoeBlock(cfg).double().eval()
    wr, wg, wu, wd = _expert_params(E, I, H, E * 10 + k)
    with torch.no_grad():
        blk.gate.weight.copy_(wr)
        blk.experts.gate_up_proj.copy_(torch.cat([wg, wu], 1))
        blk.experts.down_proj.copy_(wd)
    x = torch.randn(1, T, H, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    with torch.no_grad():
        want = blk(x)
    got, _lg, _ids = mo.moe_block(x, wr, wg, wu, wd, k, "silu")
    assert float((got - want).abs().max()) <= 1e-10


@pytest.mark.parametrize("E,k", [(2, 1), (8, 2), (8, 8), (64, 1), (64, 8)])
@pytest.mark.parametrize("masked", [False, True])
def test_oracle_aux_matches_load_balancing_loss_func(mixtral_fp64, monkeypatch, E, k, masked):
    """load_balancing_loss_func casts the one-hot assignments with `.float()`, so their means are fp32 roundings;
    that cast is restated in fp64 for the pin."""
    g = torch.Generator().manual_seed(E + k)
    B, S, L = 2, 13, 3
    logits = [torch.randn(B * S, E, generator=g, dtype=torch.float64) for _ in range(L)]
    mask = (torch.rand(B, S, generator=g) > 0.3).long() if masked else None
    with monkeypatch.context() as mp:
        mp.setattr(torch.Tensor, "float", lambda self: self.double())
        want = mixtral_fp64.load_balancing_loss_func(tuple(logits), E, k, mask)
    got = mo.aux_loss(logits, k, mask)
    assert abs(float(got) - float(want)) <= 1e-10


CASES = [  # (hidden, inter, layers, heads, kv heads, head_dim, vocab, tied, E, k)
    (64, 64, 2, 4, 2, 16, 40, True, 4, 2),    # GQA, tied
    (64, 128, 2, 4, 4, 16, 40, False, 8, 2),  # MHA, untied
    (64, 64, 1, 2, 1, 32, 33, False, 8, 8),   # MQA, k = E
]


def _moe_params(case, seed):
    H, I, L, nh, nkv, hd, V, tied, E, k = case
    d = _dims(H, I, L, nh, nkv, hd, V, tied)
    p = _params(d, seed)
    for i in range(L):
        for n in ("gate_proj", "up_proj", "down_proj"):
            p.pop(f"layers.{i}.mlp.{n}.weight")
        wr, wg, wu, wd = _expert_params(E, I, H, seed + i)
        m = f"layers.{i}.block_sparse_moe."
        p[m + "gate.weight"], p[m + "switch_mlp.gate_proj.weight"] = wr, wg
        p[m + "switch_mlp.up_proj.weight"], p[m + "switch_mlp.down_proj.weight"] = wu, wd
    return d, p


@pytest.mark.parametrize("case", CASES)
def test_oracle_model_matches_mixtral(mixtral_fp64, case):
    from transformers import MixtralForCausalLM
    from mlx_cuda_distributed_pretraining_b200.tools.export import hf_tensors
    H, I, L, nh, nkv, hd, V, tied, E, k = case
    d, params = _moe_params(case, seed=sum(case[:7]))
    model = MixtralForCausalLM(_mixtral_config(H, I, L, nh, nkv, hd, V, tied, E, k)).double().eval()
    sd = {}
    for n, t in params.items():
        sd.update(hf_tensors(n, t))
    for i in range(L):   # the in-memory module keeps Mixtral's fused layout; the checkpoint names are per expert
        pre = f"model.layers.{i}.block_sparse_moe."
        w1 = torch.stack([sd.pop(f"{pre}experts.{j}.w1.weight") for j in range(E)])
        w3 = torch.stack([sd.pop(f"{pre}experts.{j}.w3.weight") for j in range(E)])
        w2 = torch.stack([sd.pop(f"{pre}experts.{j}.w2.weight") for j in range(E)])
        sd[f"model.layers.{i}.mlp.gate.weight"] = sd.pop(pre + "gate.weight")
        sd[f"model.layers.{i}.mlp.experts.gate_up_proj"] = torch.cat([w1, w3], 1)
        sd[f"model.layers.{i}.mlp.experts.down_proj"] = w2
    if tied:
        sd["lm_head.weight"] = params["embed_tokens.weight"]
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and set(missing) <= {"lm_head.weight"}
    tokens = torch.randint(0, V, (2, 23), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = model(tokens).logits
    got, _r, _i = mo.forward(params, tokens, d, E, k)
    assert float((got - want).abs().max()) <= 1e-10


# ---- exporter ------------------------------------------------------------------------------------------------
def _fake_moe_run(tmp_path, case=CASES[0], **misc):
    from safetensors.torch import save_file
    H, I, L, nh, nkv, hd, V, tied, E, k = case
    dd = _moe_dict(E, k, variant="mlx_lm", tie_word_embeddings=tied, **misc)
    dd["name"] = "r"
    dd["model"]["dimensions"].update(hidden_size=H, intermediate_size=I, num_layers=L)
    dd["model"]["attention"].update(num_heads=nh, num_kv_heads=nkv, head_dim=hd)
    run = tmp_path / "runs" / "r"
    (run / "checkpoints").mkdir(parents=True)
    (run / "config.yaml").write_text(yaml.safe_dump(dd))
    V = dd["data"]["tokenizer"]["normal_vocab_size"] + len(dd["data"]["tokenizer"]["special_tokens"])
    d, params = _moe_params((H, I, L, nh, nkv, hd, V, tied, E, k), seed=21)
    if tied:
        params.pop("lm_head.weight", None)
    save_file({n: t.float().contiguous() for n, t in params.items()},
              str(run / "checkpoints" / "step_final_model.safetensors"))
    return tmp_path / "runs", d, {n: t.float().double() for n, t in params.items()}


@pytest.mark.parametrize("case", CASES[:2])
def test_export_loads_as_mixtral(tmp_path, mixtral_fp64, case):
    from transformers import MixtralForCausalLM
    from mlx_cuda_distributed_pretraining_b200.tools.export import main
    runs, d, params = _fake_moe_run(tmp_path, case)
    out = tmp_path / "out"
    main(["--run", "r", "--out-path", str(out), "--runs-dir", str(runs)])
    cfg = json.loads((out / "config.json").read_text())
    assert cfg["architectures"] == ["MixtralForCausalLM"] and cfg["model_type"] == "mixtral"
    assert (cfg["num_local_experts"], cfg["num_experts_per_tok"], cfg["router_aux_loss_coef"]) == (case[8], case[9],
                                                                                                   0.001)
    model = MixtralForCausalLM.from_pretrained(str(out), dtype=torch.float64,
                                               experts_implementation="eager").eval()
    tokens = torch.randint(0, d.vocab_size, (2, 19), generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        got = model(tokens).logits
    ref, _r, _i = mo.forward(params, tokens, d, case[8], case[9])
    assert float((got - ref).abs().max()) <= 1e-10


def test_export_refuses_reference_block_moe(tmp_path):
    from mlx_cuda_distributed_pretraining_b200.tools.export import export_run
    runs, _, _ = _fake_moe_run(tmp_path)
    p = runs / "r" / "config.yaml"
    d = yaml.safe_load(p.read_text())
    d["model"]["misc"]["variant"] = None
    p.write_text(yaml.safe_dump(d))
    with pytest.raises(ValueError, match="Mixtral"):
        export_run("r", str(tmp_path / "out"), str(runs))
    assert not (tmp_path / "out" / "model.safetensors").exists()


# ---- kernel index arithmetic (CPU emulation) and the faults it rejects ----------------------------------------------
def _ids(T, E, k, seed):
    g = torch.Generator().manual_seed(seed)
    return mo.route(torch.randn(T, E, generator=g, dtype=torch.float64) * 2, k)[1]


@pytest.mark.parametrize("T,E,k", [(1, 8, 2), (7, 4, 1), (129, 8, 2), (1000, 64, 8), (300, 2, 2)])
def test_emulation_is_a_valid_routing(T, E, k):
    ids = _ids(T, E, k, T + E)
    counts, off, tiles, dest = mo.emulate_routing(ids, E)
    mo.check_routing(ids, counts, off, tiles, dest, E)
    x = torch.randn(T, 16, dtype=torch.float64)
    xp = mo.emulate_permute(x, dest, off)
    w = torch.rand(T, k, dtype=torch.float64)
    assert torch.allclose(mo.emulate_combine(xp, dest, w), (w[:, :, None] * x[:, None]).sum(1))


def test_emulation_rejects_faults():
    """Each fault is fed through the checker of its stage; the correct emulation passes the same checkers."""
    T, E, k = 300, 8, 2
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(T, E, generator=g, dtype=torch.float64) * 2
    p, ids, w = mo.route(logits, k)
    mo.check_topk(p, ids)
    counts, off, tiles, dest = mo.emulate_routing(ids, E)
    mo.check_routing(ids, counts, off, tiles, dest, E)
    bad_off = off.clone()                                       # an off-by-one segment offset
    bad_off[3:] += 1
    with pytest.raises(AssertionError):
        mo.check_routing(ids, counts, bad_off, tiles, dest, E)
    e = int(ids[0, 0])                                          # a non-stable permutation: two rows of a segment swapped
    rows = (ids == e).nonzero()
    bad = dest.clone()
    (t0, j0), (t1, j1) = rows[0].tolist(), rows[1].tolist()
    bad[t0, j0], bad[t1, j1] = dest[t1, j1], dest[t0, j0]
    with pytest.raises(AssertionError):
        mo.check_routing(ids, counts, off, tiles, bad, E)
    tied = torch.zeros(4, E, dtype=torch.float64)               # a tie broken toward the higher index
    tied[:, 5] = 1.0
    pt, ids_t, _ = mo.route(tied, 3)
    mo.check_topk(pt, ids_t)
    wrong = torch.stack([torch.tensor([5, 7, 6])] * 4)          # what a "last index wins" argmax returns
    with pytest.raises(AssertionError):
        mo.check_topk(pt, wrong)
    x = torch.randn(T, 16, generator=g, dtype=torch.float64)
    xp = mo.emulate_permute(x, dest, off)
    mo.check_permute(x, dest, counts, off, xp)
    pad_row = int(off[0]) + int(counts[0])                      # a pad row left non-zero
    assert pad_row < int(off[1])
    xp_bad = xp.clone()
    xp_bad[pad_row] = 1.0
    with pytest.raises(AssertionError):
        mo.check_permute(x, dest, counts, off, xp_bad)
    good = mo.emulate_combine(xp, dest, w)
    mo.check_combine(xp, dest, p, ids, good)
    unnorm = mo.emulate_combine(xp, dest, p.gather(1, ids))    # a combine that uses the unnormalised p
    with pytest.raises(AssertionError):
        mo.check_combine(xp, dest, p, ids, unnorm)
