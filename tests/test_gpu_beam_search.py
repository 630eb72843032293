"""Beam search on the GPU: b200_attn_decode_beam element by element against fp64 over the materialised rows (prefix
positions >= T0, unused slots and everything past each length NaN, outputs canary-framed), bit-identical on repeat,
in any batch and, with one beam, to b200_attn_decode(_alibi); b200_kv_append_beam against b200_kv_append(_half);
b200_kv_beam_fork against a torch copy; beam_search(n_beams=1) against greedy generate; the cache's memory."""
from __future__ import annotations

import pytest
import torch

from tests.test_gpu_cached_attention import _frame_intact, _framed, _ops

pytestmark = pytest.mark.gpu


def _layout(P, n_live, tail_len, H, Hk, D, dtype, seed, n_beams=None):
    """Groups with prompt lengths P[g] (all rows of group g hold P[g] + tail_len[g] positions) and n_live[g] rows.
    Returns the device inputs and, per row, the materialised keys / values [len, Hk, D]."""
    g = torch.Generator().manual_seed(seed)
    G = len(P)
    n_beams = n_beams or max(n_live)
    s_prefix = max(256, -(-max(P) // 256) * 256)
    tail_cap = -(-(255 + max(tail_len)) // 256) * 256
    S = G * n_beams
    nan = float("nan")
    kp = torch.full((G, s_prefix, Hk, D), nan)
    vp = torch.full((G, s_prefix, Hk, D), nan)
    kt = torch.full((S, tail_cap, Hk, D), nan)
    vt = torch.full((S, tail_cap, Hk, D), nan)
    groups, slots, lens, rows_k, rows_v, t0s, row0, nrows = [], [], [], [], [], [], [], []
    for gi in range(G):
        t0 = 256 * (P[gi] // 256)
        t0s.append(t0)
        kp[gi, :t0] = torch.randn(t0, Hk, D, generator=g)
        vp[gi, :t0] = torch.randn(t0, Hk, D, generator=g)
        perm = torch.randperm(n_beams, generator=g)[:n_live[gi]].tolist()  # ragged, shuffled slots
        row0.append(len(groups))
        nrows.append(n_live[gi])
        L = P[gi] + tail_len[gi]
        for j in range(n_live[gi]):
            s = gi * n_beams + perm[j]
            kt[s, :L - t0] = torch.randn(L - t0, Hk, D, generator=g)
            vt[s, :L - t0] = torch.randn(L - t0, Hk, D, generator=g)
            groups.append(gi)
            slots.append(s)
            lens.append(L)
            rows_k.append(torch.cat([kp[gi, :t0], kt[s, :L - t0]]))
            rows_v.append(torch.cat([vp[gi, :t0], vt[s, :L - t0]]))
    R = len(groups)
    q = torch.randn(R, H, D, generator=g)
    cast = lambda t: t.to(dtype).cuda()
    kp, vp, kt, vt, q = cast(kp), cast(vp), cast(kt), cast(vt), cast(q)
    rows_k = [r.to(dtype).double() for r in rows_k]
    rows_v = [r.to(dtype).double() for r in rows_v]
    lens_t = torch.tensor(lens, dtype=torch.int32).cuda()
    tables = torch.tensor(groups + slots + t0s + row0 + nrows, dtype=torch.int32).cuda()
    return q, kp, vp, kt, vt, lens_t, tables, rows_k, rows_v, lens


def _beam_raw(q, kp, vp, kt, vt, lens, tables, window=-1, slopes=None):
    from mlx_cuda_distributed_pretraining_b200._lib import check, lib
    from mlx_cuda_distributed_pretraining_b200.ops import _ptr, _stream, attention_decode_beam_workspace_bytes
    R, H, D = q.shape
    G, s_prefix, Hk = kp.shape[:3]
    S, tail_cap = kt.shape[:2]
    o, ob = _framed((R, H, D), q.dtype)
    lse, lb = _framed((R, H), torch.float32)
    ws = torch.empty(attention_decode_beam_workspace_bytes(R, H, s_prefix, tail_cap, D), device="cuda",
                     dtype=torch.uint8)
    check(lib().b200_attn_decode_beam(q.data_ptr(), kp.data_ptr(), vp.data_ptr(), kt.data_ptr(), vt.data_ptr(),
                                      lens.data_ptr(), tables.data_ptr(), o.data_ptr(),
                                      lse.data_ptr(), window, _ptr(slopes), R, G, s_prefix, S, tail_cap, H, Hk, D,
                                      float(D ** -0.5), int(q.dtype == torch.bfloat16), ws.data_ptr(), ws.numel(),
                                      _stream()), "b200_attn_decode_beam")
    torch.cuda.synchronize()
    return o.clone(), lse.clone(), _frame_intact(ob) and _frame_intact(lb)


def _check_fp64(o, q, rows_k, rows_v, lens, window, slopes, name):
    """Each row's output against the fp64 reference and element-wise bound of tests/attn_fwd_check.py (the decode
    bound of DESIGN §4.2.1): the row's query as the last of a compact causal problem over its materialised keys."""
    from tests import attn_fwd_check as AF
    R, H, D = q.shape
    for b in range(R):
        L = lens[b]
        dev = "cuda"
        qf = torch.zeros(1, L, H, D, dtype=torch.float64, device=dev)
        qf[0, L - 1] = q[b].double()
        k = rows_k[b][None].to(dev)
        v = rows_v[b][None].to(dev)
        pos = torch.arange(L, device=dev)
        mask = pos[None, :] <= pos[:, None]
        if window >= 0:
            mask &= pos[:, None] - pos[None, :] <= window
        mask |= torch.eye(L, dtype=torch.bool, device=dev)
        r = AF.reference(qf, k, v, D ** -0.5, mask, None, slopes=slopes)
        ro, bo = r["o"]
        AF.check(f"{name} row {b}", o[b:b + 1][:, None].cpu(), ro[:, L - 1:L].cpu(), bo[:, L - 1:L].cpu())


CASES = [  # P per group, rows per group, tail lengths, H, Hk, D, dtype, window, alibi
    ([1], [1], [1], 4, 4, 16, torch.float32, -1, False),
    ([255, 256, 257], [3, 1, 16], [1, 300, 40], 8, 4, 64, torch.bfloat16, -1, False),
    ([1000, 4000], [5, 16], [7, 120], 16, 2, 64, torch.bfloat16, -1, True),
    ([1000], [16], [33], 8, 1, 128, torch.bfloat16, 20, False),
    ([4000, 300], [4, 9], [50, 299], 8, 8, 32, torch.float32, 700, True),
    ([600, 513], [12, 2], [3, 255], 2, 2, 16, torch.float32, -1, True),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_decode_beam_matches_fp64(case):
    _ops()
    P, n_live, tails, H, Hk, D, dt, window, alibi = CASES[case]
    q, kp, vp, kt, vt, lens, tables, rk, rv, hl = _layout(P, n_live, tails, H, Hk, D, dt, 100 + case)
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    slopes = alibi_slopes(H).cuda() if alibi else None
    o, _, intact = _beam_raw(q, kp, vp, kt, vt, lens, tables, window, slopes)
    assert intact, "canary frame overwritten"
    _check_fp64(o, q, rk, rv, hl, window, slopes, f"case {case}")
    o2, _, _ = _beam_raw(q, kp, vp, kt, vt, lens, tables, window, slopes)
    assert torch.equal(o, o2), "not bit-identical on repeat"


def test_decode_beam_group_alone_and_one_beam_equals_decode():
    ops = _ops()
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    H, Hk, D = 8, 2, 64
    slopes = alibi_slopes(H).cuda()
    q, kp, vp, kt, vt, lens, tables, rk, rv, hl = _layout([700, 300], [3, 4], [20, 5], H, Hk, D, torch.bfloat16, 7,
                                                          n_beams=4)
    o, _, _ = _beam_raw(q, kp, vp, kt, vt, lens, tables, -1, slopes)
    # group 1 alone: its rows, renumbered
    R0 = 3
    t = tables.cpu().tolist()
    R = 7
    groups, slots, t0, row0, nrows = t[:R], t[R:2 * R], t[2 * R:2 * R + 2], t[2 * R + 2:2 * R + 4], t[2 * R + 4:]
    alone = torch.tensor([0] * 4 + slots[R0:] + [t0[1]] + [0] + [4], dtype=torch.int32).cuda()
    oa, _, _ = _beam_raw(q[R0:].contiguous(), kp[1:].contiguous(), vp[1:].contiguous(), kt, vt,
                         lens[R0:].contiguous(), alone, -1, slopes)
    assert torch.equal(oa, o[R0:]), "a group differs alone and in the batch"
    # one beam per group: bit-equal to b200_attn_decode_alibi over the materialised rows
    for b in (0, R0):
        one = torch.tensor([0, slots[b], t0[groups[b]], 0, 1], dtype=torch.int32).cuda()
        g = groups[b]
        ob, _, _ = _beam_raw(q[b:b + 1].contiguous(), kp[g:g + 1].contiguous(), vp[g:g + 1].contiguous(), kt, vt,
                             lens[b:b + 1].contiguous(), one, -1, slopes)
        s_max = kp.shape[1] + kt.shape[1]
        kc = torch.zeros(1, s_max, Hk, D, dtype=torch.bfloat16, device="cuda")
        vc = torch.zeros_like(kc)
        kc[0, :hl[b]] = rk[b].to(torch.bfloat16).cuda()
        vc[0, :hl[b]] = rv[b].to(torch.bfloat16).cuda()
        od = ops.attention_decode(q[b:b + 1].contiguous(), kc, vc, lens[b:b + 1].contiguous(), alibi=slopes)
        assert torch.equal(ob, od), f"row {b}: one beam differs from b200_attn_decode_alibi"


@pytest.mark.parametrize("layout", ["interleaved", "half"])
def test_kv_append_beam_bit_equal(layout):
    ops = _ops()
    H, Hk, D, R = 8, 4, 64, 3
    g = torch.Generator().manual_seed(3)
    cos_t, sin_t = ops.rope_tables(2048, D, 10000.0, "cuda")
    q = torch.randn(R, H, D, generator=g).to(torch.bfloat16).cuda()
    k = torch.randn(R, Hk, D, generator=g).to(torch.bfloat16).cuda()
    v = torch.randn(R, Hk, D, generator=g).to(torch.bfloat16).cuda()
    lens = [600, 600, 1300]
    t0 = [512, 1280]
    tables = torch.tensor([0, 0, 1] + [2, 0, 5] + t0 + [0, 2] + [2, 1], dtype=torch.int32).cuda()
    kt = torch.zeros(6, 256, Hk, D, dtype=torch.bfloat16, device="cuda")
    vt = torch.zeros_like(kt)
    q1 = q.clone()
    ops.kv_append_beam(q1, k, v, kt, vt, torch.tensor(lens, dtype=torch.int32).cuda(), tables, 2, (cos_t, sin_t),
                       layout)
    kc = torch.zeros(R, 1536, Hk, D, dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros_like(kc)
    q2 = q.clone()
    ops.kv_append(q2, k, v, kc, vc, torch.tensor(lens, dtype=torch.int32).cuda(), (cos_t, sin_t), layout)
    assert torch.equal(q1, q2)
    for b, (s, grp) in enumerate(zip([2, 0, 5], [0, 0, 1])):
        assert torch.equal(kt[s, lens[b] - 1 - t0[grp]], kc[b, lens[b] - 1])
        assert torch.equal(vt[s, lens[b] - 1 - t0[grp]], vc[b, lens[b] - 1])


def test_kv_beam_fork_matches_torch_copy():
    ops = _ops()
    tails = [torch.randn(8, 512, 2, 32, device="cuda").to(torch.bfloat16) for _ in range(6)]
    ref = [t.clone() for t in tails]
    copies = [(0, 3, 300), (0, 5, 300), (6, 1, 17)]
    ptrs = torch.tensor([t.data_ptr() for t in tails], dtype=torch.int64).cuda()
    ops.kv_beam_fork(ptrs, torch.tensor(copies, dtype=torch.int32).cuda(), 300, tails)
    for r in ref:
        for s, d, n in copies:
            r[d, :n] = r[s, :n]
    for t, r in zip(tails, ref):
        assert torch.equal(t, r)


def _model(kind):
    from tests.test_gpu_cached_attention import _trainer
    if kind != "prefix_lm":
        return _trainer(kind).model
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.test_gpu_generation import _cfg
    import tempfile
    c = _cfg("bf16_gqa")
    c["model"]["attention"]["prefix_lm"] = True
    return Trainer(Config.from_dict(c), for_training=False, synthetic=True, quiet=True,
                   run_root=tempfile.mkdtemp(prefix="beam_runs_")).model


def _full_logits(model, seq, prompt_len):
    """fp32 logits after `seq` from Model.forward over the whole sequence (the reference's way)."""
    prefix = None
    if model.args.prefix_lm:
        prefix = torch.tensor([prompt_len], dtype=torch.int32, device="cuda")
    with torch.no_grad():
        return model(torch.tensor([seq], device="cuda"), prefix_lens=prefix).float()[0, -1]


KINDS = ["bf16_gqa", "moe", "mlx_lm", "mlx_lm_interleaved", "window", "alibi", "prefix_lm", "bf16_rope"]


@pytest.mark.parametrize("kind", KINDS)
def test_beams_match_full_forward(kind):
    """The cached path's per-step logits of every live beam against Model.forward over the beam's whole sequence (the
    reference's way): within the logits tolerance for every row, and, where the top n + 1 log-probabilities are
    separated by more than the tolerance, the same candidate tokens in the same order (near-tie rows are counted)."""
    from mlx_cuda_distributed_pretraining_b200.core.generation import beam_search
    from tests.test_gpu_cached_attention import _tol
    model = _model(kind)
    tol = _tol("bf16_gqa" if kind == "prefix_lm" else kind)
    g = torch.Generator().manual_seed(11)
    prompts = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (300, 257, 40)]
    n_beams = 4
    rows_seen = ordered = 0

    def on_step(rows, logits):
        nonlocal rows_seen, ordered
        for r, seq in enumerate(rows):
            P = next(len(p) for p in prompts if seq[:len(p)] == p)
            full = _full_logits(model, seq, P)
            err = float((logits[r] - full).abs().max()) / float(full.abs().max())
            assert err < tol, f"{kind}: row {r} ({len(seq) - P} generated) logits differ by {err:.2e}"
            rows_seen += 1
            ref = torch.log_softmax(full, -1)
            top = torch.sort(ref, descending=True, stable=True)
            gaps = top.values[:n_beams] - top.values[1:n_beams + 1]
            if float(gaps.min()) > tol * float(full.abs().max()):
                ordered += 1
                mine = torch.sort(torch.log_softmax(logits[r], -1), descending=True, stable=True).indices[:n_beams]
                assert torch.equal(mine, top.indices[:n_beams]), f"{kind}: candidates differ from the full forward"

    out = beam_search(model, prompts, n_beams=n_beams, max_tokens=10, stop_tokens=[3], on_step=on_step)
    print(f"{kind}: {rows_seen} beam rows within tolerance, {ordered} with clear margins compared in order")
    assert rows_seen > 3 * n_beams and len(out) == 3


@pytest.mark.parametrize("kind", ["bf16_rope", "mlx_lm", "alibi", "window"])
def test_one_beam_equals_greedy(kind):
    """beam_search(n_beams=1) follows greedy generate token for token, except where the top two logits are closer
    than the logits tolerance (greedy takes the argmax of the logits, beam search a stable sort of log_softmax, and
    the subtraction of the log-sum-exp can merge two logits an ulp apart): the runs are compared up to the first
    such step."""
    from mlx_cuda_distributed_pretraining_b200.core.generation import beam_search, generate
    from tests.test_gpu_cached_attention import _tol
    model = _model(kind)
    g = torch.Generator().manual_seed(5)
    prompts = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (300, 40)]
    greedy = generate(model, prompts, max_tokens=24, temperature=0, repetition_penalty=1.0, eos_token=None)
    beams = beam_search(model, prompts, n_beams=1, max_tokens=24)
    for p, gr, bs in zip(prompts, greedy, beams):
        assert len(bs) == 1
        for i, (a, b) in enumerate(zip(gr, bs[0][0])):
            if a != b:
                lg = _full_logits(model, p + gr[:i], len(p))
                top2 = torch.topk(lg, 2).values
                assert float(top2[0] - top2[1]) <= _tol(kind) * float(lg.abs().max()), f"{kind}: step {i}"
                break


def test_cli_num_beams_end_to_end():
    """`--num-beams 4` on a small bf16 run and on a C1-shaped fp32 run prints ranked `Beam Output` lines."""
    import os
    import re
    import subprocess
    import sys
    import tempfile
    from pathlib import Path

    import yaml
    root = Path(__file__).resolve().parents[1]
    env = dict(os.environ, PYTHONPATH=str(root) + os.pathsep + os.environ.get("PYTHONPATH", ""))
    for name, bf16 in (("beam-bf16", True), ("beam-c1", False)):
        with tempfile.TemporaryDirectory(prefix="beam_e2e_") as tmp:
            cfg = yaml.safe_load((root / "configs" / "c1-llama2m-adamw.yaml").read_text())
            cfg["name"] = name
            cfg["data"]["input_file"] = "synthetic:markov"
            cfg["data"]["preprocessing"]["max_context_size"] = 128
            cfg["training"]["hyperparameters"]["iters"] = 3
            if bf16:
                cfg["model"]["attention"].update(num_heads=4, num_kv_heads=2, head_dim=64)
                cfg["system"]["mixed_precision"] = True
            cfg_path = Path(tmp) / "cfg.yaml"
            cfg_path.write_text(yaml.safe_dump(cfg))
            subprocess.run([sys.executable, "-m", "core.training", "--config", str(cfg_path)], cwd=tmp, env=env,
                           check=True, timeout=600)
            out = subprocess.run([sys.executable, "-m", "core.generation", "--run", name, "--runs-dir",
                                  str(Path(tmp) / "runs"), "--prompt", "hello there", "--max-tokens", "12",
                                  "--num-beams", "4"],
                                 cwd=root, env=env, check=True, capture_output=True, text=True, timeout=600).stdout
            lines = [l for l in out.splitlines() if l.startswith("Beam Output (Score: ")]
            scores = [float(re.match(r"Beam Output \(Score: (\S+)\): ", l).group(1)) for l in lines]
            assert 1 <= len(lines) <= 4 and scores == sorted(scores, reverse=True), out


def test_beam_search_runs_and_memory():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import BeamKVCache, KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import beam_search
    from tests.test_gpu_cached_attention import _trainer
    model = _trainer("bf16_gqa").model
    g = torch.Generator().manual_seed(9)
    prompts = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (100, 257, 30)]
    out = beam_search(model, prompts, n_beams=4, max_tokens=12, stop_tokens=[3])
    for res in out:
        assert 1 <= len(res) <= 4
        assert [s for _, s in res] == sorted([s for _, s in res], reverse=True)
    P = 2048
    prefix = KVCache(model, 1, P)
    model.prefill(torch.randint(0, 256, (1, P)).cuda(), [P], prefix)
    bc = BeamKVCache(model, prefix, 8, 64)
    per_pos = prefix.nbytes() // prefix.s_max
    assert bc.nbytes() <= per_pos * (prefix.s_max + 8 * bc.tail_cap)
    assert bc.nbytes() < 8 * per_pos * (P + 64) / 2
