"""CPU: the C-ABI library's symbol table, host-side logic (config, schedules, flat store, optimizer
factory, DP helpers) and the rule that the product never imports the oracle."""
import ctypes
import re
from pathlib import Path

import pytest
import torch
import yaml

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "mlx_cuda_distributed_pretraining_b200"


def test_capi_exports_every_declared_symbol(lib_built):
    header = (ROOT / "include" / "b200_hotpath.h").read_text()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 20
    handle = ctypes.CDLL(str(lib_built))
    missing = [s for s in sorted(declared) if not hasattr(handle, s)]
    assert not missing, f"declared in include/b200_hotpath.h but not exported: {missing}"
    from mlx_cuda_distributed_pretraining_b200._lib import SIGNATURES
    assert set(SIGNATURES) == declared, set(SIGNATURES) ^ declared
    # the ctypes rows must agree with the header prototypes kind by kind (the compiler checks the header against the
    # definitions, nothing else checks _lib.py): pointer, int, long long, size_t / unsigned long long (one ctypes type
    # on LP64), float, void
    def c_kind(decl):
        decl = decl.strip()
        if "*" in decl:
            return "pointer"
        words = [w for w in decl.split()[:-1] if w != "const"]  # drop the name
        return {"void": "void", "int": "int", "long long": "long long", "size_t": "u64",
                "unsigned long long": "u64", "float": "float"}[" ".join(words)]

    def ctypes_kind(t):
        if t is None:
            return "void"
        if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
            return "pointer"
        for ct, kind in ((ctypes.c_int, "int"), (ctypes.c_longlong, "long long"), (ctypes.c_size_t, "u64"),
                         (ctypes.c_ulonglong, "u64"), (ctypes.c_float, "float")):
            if t is ct:
                return kind
        raise AssertionError(f"unexpected ctypes type {t}")

    code = re.sub(r"/\*.*?\*/", " ", header, flags=re.S)
    protos = re.findall(r"([A-Za-z_][\w \t*]*?)\b(b200_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", code)
    assert {name for _, name, _ in protos} == declared
    mismatched = []
    for ret, name, params in protos:
        params = [] if params.strip() in ("", "void") else params.split(",")
        want = (c_kind(ret.strip() + " r"), [c_kind(p) for p in params])
        res, args = SIGNATURES[name]
        if want != (ctypes_kind(res), [ctypes_kind(a) for a in args]):
            mismatched.append(name)
    assert not mismatched, f"_lib.SIGNATURES disagrees with include/b200_hotpath.h: {mismatched}"
    handle.b200_version.restype = ctypes.c_int
    assert handle.b200_version() >= 1
    handle.b200_newton_schulz_workspace_bytes.restype = ctypes.c_size_t
    # pure host arithmetic (no GPU): A,B [m,m] bf16 x2 + X_tmp
    n = handle.b200_newton_schulz_workspace_bytes(2, 128, 256, 5)
    assert n == 2 * 2 * 128 * 128 * 2 + 2 * 128 * 256 * 2


def test_product_never_imports_oracle():
    offenders = []
    for p in list(PKG.rglob("*.py")) + [ROOT / "core" / "training.py"] + list((ROOT / "optimizers").glob("*.py")):
        txt = p.read_text()
        if re.search(r"^\s*(from|import)\s+oracle\b", txt, re.M):
            offenders.append(str(p))
    assert not offenders, offenders


def test_no_cpu_fallback_without_device():
    from mlx_cuda_distributed_pretraining_b200 import _lib, ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.B200Error):
        ops.zeropower_via_newtonschulz5(torch.randn(8, 16))
    with pytest.raises(_lib.B200Error):
        ops.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))


def test_configs_parse_and_match_baseline_dims():
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    want = {
        "c1-llama2m-adamw.yaml": (128, 256, 4, 8, 8, 16, "adamw"),
        "c2-llama80m-muon.yaml": (1024, 2816, 12, 16, 8, 64, "muon"),
        "c3-llama400m-muon-dp8.yaml": (1024, 4096, 16, 16, 8, 64, "muon"),
        "c4-llama256m-shampoo-dp4.yaml": (1024, 2816, 16, 16, 16, 64, "shampoo"),
        "c5-llama1b-adamw-dp8.yaml": (2048, 5632, 16, 16, 16, 128, "adamw"),
    }
    for fn, (h, i, L, H, Hk, D, opt) in want.items():
        c = Config.from_yaml(str(ROOT / "configs" / fn))
        m = c.model
        assert (m.dimensions["hidden_size"], m.dimensions["intermediate_size"], m.dimensions["num_layers"],
                m.attention["num_heads"], m.attention["num_kv_heads"], m.attention["head_dim"]) == (h, i, L, H, Hk, D)
        assert c.training.optimization["optimizer"] == opt
    with pytest.raises(ValueError):
        Config.from_dict({"data": {}, "model": {}, "training": {}, "logging": {}, "system": {}})
    bad = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
    bad["system"]["no_such_key"] = 1
    with pytest.raises(TypeError):  # unknown keys raise, as the reference's dataclasses do
        Config.from_dict(bad)


def test_schedules_equal_oracle():
    from oracle import reference_math as R
    from mlx_cuda_distributed_pretraining_b200.core.training import OptimizationManager, TrainingConfig
    tc = TrainingConfig(hyperparameters={"learning_rate": 3e-4, "batch_size": 1},
                        scheduler={"type": "cosine_with_warmup", "warmup_steps": 20, "min_lr_ratio": 0.1},
                        optimization={"optimizer": "muon"})
    s = OptimizationManager(tc, 200).create_scheduler()
    r = R.make_schedule(tc.scheduler, 3e-4, 200)
    for step in (0, 1, 19, 20, 21, 100, 219, 220, 1000):
        assert s(step) == pytest.approx(r(step), rel=1e-12, abs=1e-18)


def test_optimizer_factory_dispatch():
    from mlx_cuda_distributed_pretraining_b200.core.training import OptimizationManager, TrainingConfig
    from mlx_cuda_distributed_pretraining_b200.optimizers import AdamW, HybridOptimizer, Muon, Shampoo
    def mk(opt):
        tc = TrainingConfig(hyperparameters={"learning_rate": 1e-3, "batch_size": 1, "weight_decay": 0.1},
                            scheduler={"type": "cosine", "min_lr_ratio": 0.1}, optimization=opt)
        om = OptimizationManager(tc, 10)
        return om.create_optimizer(om.create_scheduler())
    assert isinstance(mk({"optimizer": "muon"}), Muon)
    a = mk({"optimizer": "adamw", "betas": [0.9, 0.95], "eps": 1e-8})
    assert isinstance(a, AdamW) and a.betas == (0.9, 0.95) and a.weight_decay == 0.1
    s = mk({"optimizer": "shampoo"})
    assert isinstance(s, Shampoo) and s.params.update_period == 100 and s.params.beta2 == 0.95
    h = mk({"optimizer": "hybrid"})
    assert isinstance(h, HybridOptimizer) and h.matrix_optimizer.alternate_optimizer is h.non_matrix_optimizer
    with pytest.raises(ValueError):
        mk({"optimizer": "lbfgs"})


def test_param_store_layout_and_views():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    from mlx_cuda_distributed_pretraining_b200.flat import ParamStore, flatten_tree
    from oracle import reference_math as R
    args = ModelArgs(model_type="llama", hidden_size=64, num_hidden_layers=2, intermediate_size=96,
                     num_attention_heads=4, head_dim=16, vocab_size=67, num_key_value_heads=2,
                     tie_word_embeddings=True)
    model = Model(args)
    names = [n for n, _ in model.named_parameters()]
    assert names == list(R.param_shapes(R.LlamaDims(64, 96, 2, 4, 2, 16, 67)))  # reference's flattened names
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    store = ParamStore(model, torch.bfloat16, torch.device("cpu"))
    # same-shape matrices are contiguous batches; every group is 16-byte aligned
    shapes = {(g.rows, g.cols): g.batch for g in store.mat_groups}
    assert shapes[(64, 64)] == 4 and shapes[(32, 64)] == 4 and shapes[(96, 64)] == 4 and shapes[(64, 96)] == 2
    assert all(g.offset % 128 == 0 for g in store.mat_groups)
    for n, p in model.named_parameters():
        assert p.dtype == torch.bfloat16 and p.grad is not None
        assert torch.equal(store.view(store.master, n), before[n])
        assert p.data_ptr() == store.view(store.shadow, n).data_ptr()
        assert p.grad.data_ptr() == store.view(store.grad, n).data_ptr()
    # explicit (nested) gradient dicts, as the reference trainer passes them
    nested = {"layers": [{"mlp": {"gate_proj": {"weight": torch.ones(96, 64)}}}]}
    flat = flatten_tree(nested)
    assert list(flat) == ["layers.0.mlp.gate_proj.weight"]
    store.load_gradients(nested)
    assert float(store.view(store.grad, "layers.0.mlp.gate_proj.weight").float().sum()) == 96 * 64
    with pytest.raises(KeyError):
        store.load_gradients({"nope": torch.zeros(1)})


def test_dp_helpers():
    from mlx_cuda_distributed_pretraining_b200.distributed import dp
    b = torch.arange(10).reshape(10, 1)
    shards = [dp.shard_batch(b, r, 3) for r in range(3)]
    assert [s.shape[0] for s in shards] == [3, 3, 4]          # last shard takes the remainder
    assert torch.equal(torch.cat(shards), b)
    owner = dp.partition_by_cost([5, 1, 1, 1, 4, 4], 2)
    load = [sum(c for c, o in zip([5, 1, 1, 1, 4, 4], owner) if o == r) for r in range(2)]
    assert abs(load[0] - load[1]) <= 1


def test_synthetic_data_matches_oracle_stream():
    from oracle import reference_math as R
    from mlx_cuda_distributed_pretraining_b200.core.training import SyntheticData
    d = SyntheticData(256, 4, 32, rank=1)
    assert torch.equal(d.generate_batch(7), R.synthetic_batch(7, 1, 4, 32, 256))


def test_tokenizer_byte_level_ids():
    from mlx_cuda_distributed_pretraining_b200.core.training import DataConfig, TokenizerManager
    cfg = DataConfig(input_file="synthetic", preprocessing={"max_context_size": 8},
                     tokenizer={"normal_vocab_size": 256, "special_tokens": {"pad": "<pad>", "bos": "<bos>", "eos": "<eos>"}})
    tk = TokenizerManager(cfg)
    assert (tk.PAD_TOKEN, tk.BOS_TOKEN, tk.EOS_TOKEN, tk.VOCAB_SIZE) == (256, 257, 258, 259)
    ids = tk.tokenize_doc("hello world, long")
    assert ids[0] == 257 and ids[-1] == 258 and len(ids) == 10
    assert tk.detokenize(ids[1:-1]) == "hello wo"


def test_batch_prefetcher_order_reuse_and_errors():
    """Background batch producer (SURVEY 8f row f4): same batches, in step order, as building them inline;
    buffers are recycled only after release; producer exceptions surface in the training thread."""
    import time
    from mlx_cuda_distributed_pretraining_b200.core.training import BatchPrefetcher

    def make(step):
        g = torch.Generator().manual_seed(42 + 1000 * step)
        return torch.randint(0, 100, (4, 9), generator=g, dtype=torch.int64)

    pf = BatchPrefetcher(make, start=3, stop=20, depth=2)
    seen = []
    for step in range(3, 20):
        buf, slot = pf.get(step)
        assert torch.equal(buf, make(step)), step
        seen.append(buf.data_ptr())
        pf.release(slot, None)
        if step == 5:
            time.sleep(0.05)          # let the producer run ahead: it must stall at the queue depth
    assert len(set(seen)) <= 4        # depth + 2 rotating buffers
    with pytest.raises(RuntimeError):
        pf.get(7)                     # sequential by construction
    pf.close()

    def boom(step):
        if step == 2:
            raise ValueError("bad document")
        return make(step)

    pf = BatchPrefetcher(boom, start=0, stop=5)
    pf.get(0), pf.get(1)
    with pytest.raises(ValueError):
        pf.get(2)
    pf.close()


def test_fuse_adjacent_detects_only_true_neighbours():
    """ops._fuse_adjacent (pointer logic, CPU tensors suffice): merges projections whose weights, flat .grad
    views and output gradients are neighbours in memory, and nothing else."""
    from mlx_cuda_distributed_pretraining_b200 import ops
    n, k_in, B, S = 8, 16, 2, 5
    wflat, gflat = torch.randn(3 * n * k_in), torch.zeros(3 * n * k_in)
    ws = []
    for i in range(3):
        w = wflat[i * n * k_in:(i + 1) * n * k_in].view(n, k_in).requires_grad_(True)
        w.grad = gflat[i * n * k_in:(i + 1) * n * k_in].view(n, k_in)
        w._b200_flat_grad = True
        ws.append(w)
    packed = torch.randn(B, S, 2 * n)
    lone = torch.randn(B, S, n)
    fused = ops._fuse_adjacent((lone, packed[..., :n], packed[..., n:]), ws)
    assert fused is not None and [f[0].shape for f in fused] == [(B * S, n), (B * S, 2 * n)]
    assert fused[1][1].data_ptr() == ws[1].data_ptr() and fused[1][1].shape == (2 * n, k_in)
    assert fused[1][2].data_ptr() == ws[1].grad.data_ptr()
    assert torch.equal(fused[1][0], packed.view(B * S, 2 * n))
    # swapped halves, separate buffers, or a weight without a flat gradient: no merge
    assert ops._fuse_adjacent((lone, packed[..., n:], packed[..., :n]), ws) is None
    assert ops._fuse_adjacent((lone, torch.randn(B, S, n), torch.randn(B, S, n)), ws) is None
    ws[2]._b200_flat_grad = False
    assert ops._fuse_adjacent((lone, packed[..., :n], packed[..., n:]), ws) is None


def test_yaml_schema_matches_reference_parse():
    """configs/c*.yaml parsed by the REFERENCE's own Config dataclasses (tests/golden/ref_config_parse.json,
    written by tests/golden/make_golden.py) vs this repo's Config: every section / key / default the reference
    sees must come out identical here, so a YAML written for the reference runs unchanged."""
    import dataclasses
    import json
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    ref = json.loads((ROOT / "tests" / "golden" / "ref_config_parse.json").read_text())
    assert len(ref) == 5

    def subset(a, b, path):
        if isinstance(a, dict):
            assert isinstance(b, dict), path
            for k, v in a.items():
                assert k in b, f"{path}.{k} missing"
                subset(v, b[k], f"{path}.{k}")
        elif isinstance(a, list):
            assert list(b) == a, path
        else:
            assert a == b, (path, a, b)

    for name, want in ref.items():
        got = dataclasses.asdict(Config.from_yaml(str(ROOT / "configs" / name)))
        subset(want, got, name)


def test_markov_synthetic_stream_matches_oracle_generator():
    """`data.input_file: synthetic:markov` (learnable stream for loss-curve parity) draws exactly what the oracle's
    reference_math.synthetic_batch_markov draws, per step and rank."""
    import torch
    from oracle import reference_math as R
    from mlx_cuda_distributed_pretraining_b200.core.training import SyntheticData
    for step, rank in ((0, 0), (7, 1)):
        a = SyntheticData(256, 3, 96, rank, kind="markov").generate_batch(step)
        assert torch.equal(a, R.synthetic_batch_markov(step, rank, 3, 96, 256))
    u = SyntheticData(256, 3, 96, 0).generate_batch(5)
    assert torch.equal(u, R.synthetic_batch(5, 0, 3, 96, 256))


def test_bench_workload_tables_match_baseline():
    """bench.py derives every workload from configs/*.yaml; its algorithmic-work tables must reproduce BASELINE.md
    section 4 (Newton-Schulz flops per update, attention flops and bytes per micro-batch x accumulation)."""
    import bench
    want_ns = {"c2": 4.129, "c3": 6.566, "c4": 5.413, "c5": 43.30}
    want_attn = {"c1": (0.034, 0.069, 0.138), "c2": (0.825, 1.221, 2.441), "c4": (17.59, 17.31, 34.63),
                 "c5": (17.59, 17.25, 34.49)}
    for tag in bench.CONFIG_FILES:
        c = bench.dims_of(bench.load_config(tag, False))
        if tag in want_ns:
            assert abs(bench.ns_flops_per_step(c) / 1e12 - want_ns[tag]) < 5e-3 * want_ns[tag], tag
        if tag in want_attn:
            f, bf, bb = want_attn[tag]
            assert abs(bench.attn_flops_fwd_per_step(c) / 1e12 - f) < 2e-2 * f + 1e-3, tag
            got_f, got_b = bench.attn_bytes_per_step(c)
            assert abs(got_f / 1e9 - bf) < 1e-2 * bf + 1e-3 and abs(got_b / 1e9 - bb) < 1e-2 * bb + 1e-3, tag
    c3 = bench.dims_of(bench.load_config("c3", False))
    assert c3["accum"] == 8 and abs(bench.attn_flops_fwd_per_step(c3) / 1e12 - 8 * 4.398) < 0.05   # per update
    assert "Muon" in bench.workload_name("c2", bench.dims_of(bench.load_config("c2", False)))


def test_early_stopping_matches_reference_decisions():
    """EarlyStoppingMonitor vs the reference's own class run over five validation-loss sequences
    (tests/golden/make_golden.py, core/training.py:621-668): same stop decision, counter and best value after
    every update, for min / max mode, disabled monitors and all-default settings."""
    import ast

    import numpy as np
    from mlx_cuda_distributed_pretraining_b200.core.training import EarlyStoppingMonitor
    g = np.load(ROOT / "tests" / "golden" / "reference_vectors.npz")
    n_cases = sum(1 for k in g.files if k.startswith("es") and k.endswith("_seq"))
    assert n_cases == 5
    for i in range(n_cases):
        cfg = dict(ast.literal_eval(str(g[f"es{i}_cfg"])))
        mon = EarlyStoppingMonitor(cfg)
        for v, stop, counter, best in zip(g[f"es{i}_seq"], g[f"es{i}_stop"], g[f"es{i}_counter"], g[f"es{i}_best"]):
            assert int(mon.update({"val_loss": float(v)})) == int(stop), (i, v)
            assert mon.counter == int(counter) and mon.best_value == float(best), (i, v)
    assert EarlyStoppingMonitor({"enabled": True}).update({"other_metric": 1.0}) is False   # metric absent: never stops


def test_header_is_plain_c_and_links_against_the_library(lib_built, tmp_path):
    """include/b200_hotpath.h is the boundary a non-Python host binds: it must compile as C99 (no C++-isms, no torch
    types) and a C program using it must link against the built library by its exported names alone."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "host.c"
    src.write_text('#include <stddef.h>\n#include "b200_hotpath.h"\n'
                   "int main(void) {\n"
                   "  b200_dw_job j; b200_ns_group g; unsigned long long h = 0, m = 0;\n"
                   "  (void)j; (void)g;\n"
                   "  b200_tensor_map_cache_stats(&h, &m);\n"
                   "  /* no device here: only calls that need none */\n"
                   "  return (b200_version() >= 2 && b200_reduce_workspace_bytes(4) > 0 && h == 0 && m == 0) ? 0 : 1;\n"
                   "}\n")
    lib_dir = ROOT / "mlx_cuda_distributed_pretraining_b200"
    exe = tmp_path / "host"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", f"-I{ROOT / 'include'}", str(src),
                    f"-L{lib_dir}", "-lb200hotpath", f"-Wl,-rpath,{lib_dir}", "-o", str(exe)], check=True)
    assert subprocess.run([str(exe)]).returncode == 0
