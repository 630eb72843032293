"""Text generation from a trained run (core/generation.py of the reference) on the KV-cached decode path.

    python -m core.generation --run <name> --prompt "..." [--max-tokens 256 --temperature 1.0 --min-p 0.05
                              --repetition-penalty 1.1 --repetition-context-size 20]
                              [--top-p P --seed N --num-samples N --checkpoint step_N --runs-dir runs]
                              [--kv-bits {4,8} --kv-group-size {32,64,128} --quantized-kv-start N]
                              [--prefill-step-size N] [--num-beams N]
                              [--draft-run NAME --draft-checkpoint step_N --num-draft-tokens K]

The run's config.yaml (written by the trainer) rebuilds the model through Trainer(cfg, for_training=False), the
checkpoint's weights are loaded into it, and `generate` prefills [BOS] + tokenize(prompt) once and then decodes one
token per step against the cache (arch/llama.py: Model.prefill / Model.decode_step).

Sampling follows the reference's mlx_lm_utils.make_sampler / make_logits_processors (DESIGN.md §2 records each
decision): repetition penalty over the literal window tokens[max(0, idx - R):idx] with idx = len(tokens) - 1, then
min-p when min_p is truthy, else top-p when top_p is truthy, else plain temperature sampling; temperature 0 is
argmax.  The filters below are device-agnostic torch over [..., V] fp32 logits.
"""
from __future__ import annotations

import argparse
import math
import random
import sys
import time
from pathlib import Path
from typing import Callable, List, Optional, Sequence, Tuple

import torch


# ------------------------------------------------------------------------------------------------
# logits processing and sampling distributions (mlx_lm_utils.py:57-142)
# ------------------------------------------------------------------------------------------------
def repetition_window(tokens: Sequence[int], context_size: int) -> List[int]:
    """tokens[max(0, idx - R):idx] with idx = len(tokens) - 1: the window the reference's processor divides over
    (it leaves out the token just fed)."""
    idx = len(tokens) - 1
    return list(tokens[max(0, idx - context_size):idx])


def apply_repetition_penalty(logits: torch.Tensor, windows: Sequence[Sequence[int]], penalty: float) -> torch.Tensor:
    """logits [B, V]: logits[b, t] / penalty once per occurrence of t in windows[b] (sign ignored, as written)."""
    if penalty == 1.0 or not any(len(w) for w in windows):
        return logits
    B, V = logits.shape
    width = max(len(w) for w in windows)
    ids = torch.zeros((B, width), dtype=torch.int64)
    ones = torch.zeros((B, width), dtype=logits.dtype)
    for b, w in enumerate(windows):
        ids[b, :len(w)] = torch.tensor(list(w), dtype=torch.int64)
        ones[b, :len(w)] = 1.0
    counts = torch.zeros_like(logits).scatter_add_(1, ids.to(logits.device), ones.to(logits.device))
    return logits / torch.pow(torch.full_like(logits, float(penalty)), counts)


def _sorted_desc(x: torch.Tensor) -> torch.Tensor:
    """argsort(-x) along the last axis, ties in index order (stable)."""
    return torch.sort(x, dim=-1, descending=True, stable=True).indices


def _unsort(sorted_vals: torch.Tensor, order: torch.Tensor) -> torch.Tensor:
    return torch.zeros_like(sorted_vals).scatter_(-1, order, sorted_vals)


def min_p_distribution(logits: torch.Tensor, temp: float, min_p: float) -> torch.Tensor:
    """make_sampler's min-p branch (mlx_lm_utils.py:69-84) as a distribution over the vocabulary: softmax(l / temp),
    keep the sorted probabilities p >= min_p * p_max (always the top one), renormalise."""
    probs = torch.softmax(logits * (1 / temp), dim=-1)
    order = _sorted_desc(logits)
    sp = torch.gather(probs, -1, order)
    remove = sp < min_p * sp[..., :1]
    remove[..., 0] = False
    sel = torch.where(remove, torch.zeros_like(sp), sp)
    sel = sel / sel.sum(dim=-1, keepdim=True)
    return _unsort(sel, order)


def top_p_distribution(logits: torch.Tensor, temp: float, top_p: float) -> torch.Tensor:
    """make_sampler's top-p branch (mlx_lm_utils.py:85-103): keep the sorted prefix with cumsum <= top_p (the token
    crossing the threshold is dropped), or the top token alone when that prefix is empty; renormalise."""
    probs = torch.softmax(logits * (1 / temp), dim=-1)
    order = _sorted_desc(probs)
    sp = torch.gather(probs, -1, order)
    mask = torch.cumsum(sp, dim=-1) <= top_p
    mask[..., 0] |= ~mask.any(dim=-1)
    sel = torch.where(mask, sp, torch.zeros_like(sp))
    sel = sel / sel.sum(dim=-1, keepdim=True)
    return _unsort(sel, order)


def temperature_distribution(logits: torch.Tensor, temp: float) -> torch.Tensor:
    """make_sampler's plain branch (mlx_lm_utils.py:104-107): categorical(l / temp)."""
    return torch.softmax(logits * (1 / temp), dim=-1)


def sampling_distribution(logits: torch.Tensor, temp: float, min_p: Optional[float] = None,
                          top_p: Optional[float] = None) -> torch.Tensor:
    if min_p:
        return min_p_distribution(logits, temp, min_p)
    if top_p:
        return top_p_distribution(logits, temp, top_p)
    return temperature_distribution(logits, temp)


def token_probs(logits: torch.Tensor, temp: float, min_p: Optional[float], top_p: Optional[float]) -> torch.Tensor:
    """The distribution sample() draws from (temp > 0): the sampler over log-probabilities (logits - logsumexp)."""
    logprobs = logits - torch.logsumexp(logits, dim=-1, keepdim=True)
    return sampling_distribution(logprobs, temp, min_p, top_p)


def sample(logits: torch.Tensor, temp: float, min_p: Optional[float], top_p: Optional[float],
           generator: Optional[torch.Generator]) -> torch.Tensor:
    """Next tokens [B] from fp32 logits [B, V], on the logits' device.  Like the reference, the sampler sees
    log-probabilities (logits - logsumexp); temperature 0 is argmax."""
    if temp == 0:
        return torch.argmax(logits - torch.logsumexp(logits, dim=-1, keepdim=True), dim=-1)
    return torch.multinomial(token_probs(logits, temp, min_p, top_p), 1, generator=generator).squeeze(-1)


# ------------------------------------------------------------------------------------------------
# generation
# ------------------------------------------------------------------------------------------------
def position_limit(args) -> Optional[int]:
    """The longest sequence a model may generate: max_position_embeddings, or None (no limit) for an ALiBi model
    without RoPE, whose attention depends on key distances alone and so runs past its training length (the KV cache
    is sized to prompt + max_tokens)."""
    rope = getattr(args, "apply_rope", False) or getattr(args, "variant", None) == "mlx_lm"
    if getattr(args, "alibi", False) and not rope:
        return None
    return args.max_position_embeddings


def prefill_chunks(prompts: Sequence[Sequence[int]], step: int) -> List[List[List[int]]]:
    """The chunks of prefill_step_size = step: chunk c holds tokens [c step, (c + 1) step) of every prompt (empty for
    a prompt already done), until the longest prompt is used up."""
    longest = max(len(p) for p in prompts)
    return [[list(p[c0:c0 + step]) for p in prompts] for c0 in range(0, longest, step)]


def _prefill(model, prompts: List[List[int]], cache, step: Optional[int]) -> torch.Tensor:
    """The fp32 logits [B, V] after each prompt's last token, the prompts appended to what the cache holds: in chunks
    of `step` tokens (None: one chunk), each through Model.extend, except that the first chunk of an empty cache goes
    through Model.prefill unless the cache rotates.  A row's logits come from the chunk that holds its last token."""
    device = model.embed_tokens.weight.device
    empty = all(n == 0 for n in cache.host_lens)
    logits = None
    for c, chunk in enumerate(prefill_chunks(prompts, step or max(len(p) for p in prompts))):
        counts = [len(t) for t in chunk]
        tokens = torch.zeros((len(chunk), max(counts)), dtype=torch.int64)
        for b, t in enumerate(chunk):
            tokens[b, :len(t)] = torch.tensor(t, dtype=torch.int64)
        run = model.prefill if empty and c == 0 and not cache.rotating else model.extend
        lg = run(tokens.to(device), counts, cache)
        if logits is None:
            logits = lg
        else:
            fresh = torch.tensor([n > 0 for n in counts], device=device)
            logits = torch.where(fresh[:, None], lg, logits)
    return logits


def generate(model, prompts: List[List[int]], max_tokens: int = 256, temperature: float = 1.0,
             min_p: Optional[float] = 0.05, top_p: Optional[float] = None, repetition_penalty: float = 1.1,
             repetition_context_size: int = 20, eos_token: Optional[int] = None, seed: Optional[int] = None,
             on_step: Optional[Callable[[List[int]], None]] = None, kv_bits: Optional[int] = None,
             kv_group_size: int = 64, quantized_kv_start: int = 0, prefill_step_size: Optional[int] = None,
             prompt_cache=None, max_kv_size: Optional[int] = None, draft_model=None, num_draft_tokens: int = 3,
             on_round: Optional[Callable[[List[List[int]], List[List[int]]], None]] = None) -> List[List[int]]:
    """Generates up to max_tokens tokens for each of the ragged prompts in one batch.  A row stops at EOS, which is
    included in its output.  Returns the generated tokens per row (prompt excluded).  Per step, the sampled tokens
    are the one value read back from the device.  kv_bits (4 or 8; None: no quantization), kv_group_size and
    quantized_kv_start select the reference's quantized KV cache (arch.llama.KVCache).

    prefill_step_size (int >= 1): the prompts go through the model in chunks of that many tokens (Model.extend), each
    attending over the cache the earlier chunks filled, so prefill holds B x step activations rather than
    B x prompt.  prompt_cache: a KVCache of batch len(prompts) that the caller built and keeps (its kv settings
    apply; a different kv_bits is an error).  The prompts are appended to what it holds, and it is updated in place
    so that it ends holding prompt + output of every row, ready for the next turn.  Without both, the prompts go
    through Model.prefill in one piece.

    max_kv_size (an int >= 5): a rotating KV cache (arch.llama.KVCache(max_kv_size=...)), as the reference's
    make_prompt_cache(model, max_kv_size) (core/generation_lite.py:103, :120): each query sees the first 4 positions
    of its row and its most recent max_kv_size - 4, and the cache holds a constant number of slots whatever the
    length.  The prompts then always go through Model.extend, in chunks of prefill_step_size (default 512).  A
    rotating prompt_cache brings its own max_kv_size (a different one is an error).  A row that stops at EOS neither
    advances nor writes afterwards, as a ring cannot be truncated.

    draft_model (a Model with the same vocabulary): speculative decoding, as mlx_lm's generate(..., draft_model=...)
    (DESIGN §2).  Each round the draft proposes up to num_draft_tokens (1 to 15, default 3) tokens and the target
    scores them all in one Model.verify call; the output is still a sample of the target, with plain generation's
    distribution.  on_round(emitted, drafted), if given, sees each round's tokens emitted and drafted per row.  It
    does not combine with kv_bits, max_kv_size, prompt_cache or on_step.  With prefill_step_size the draft is
    prefilled in the same chunks when Model.extend serves it, else in one piece (draft_prefill_step)."""
    from ..arch.llama import KVCache, check_cache_options

    if not prompts or any(len(p) == 0 for p in prompts):
        raise ValueError("every prompt needs at least one token")
    if draft_model is not None:
        check_draft(model, draft_model, num_draft_tokens, max(len(p) for p in prompts) + max_tokens, kv_bits=kv_bits,
                    max_kv_size=max_kv_size, prompt_cache=prompt_cache, on_step=on_step)
    if prefill_step_size is not None and (isinstance(prefill_step_size, bool) or not isinstance(prefill_step_size, int)
                                          or prefill_step_size < 1):
        raise ValueError(f"generate: prefill_step_size must be None or an int >= 1, got {prefill_step_size!r}")
    check_cache_options(model, kv_bits, kv_group_size, quantized_kv_start, max_kv_size, "generate")
    if prompt_cache is not None:
        if not isinstance(prompt_cache, KVCache):
            raise ValueError(f"generate: prompt_cache must be an arch.llama.KVCache, got {type(prompt_cache).__name__}")
        if max_kv_size is not None and max_kv_size != prompt_cache.max_kv_size:
            raise ValueError(f"generate: max_kv_size={max_kv_size!r} conflicts with the prompt_cache's max_kv_size "
                             f"{prompt_cache.max_kv_size!r} (the cache's settings apply)")
        if prompt_cache.rotating and prefill_step_size is not None and prefill_step_size > prompt_cache.max_chunk:
            raise ValueError(f"generate: prefill_step_size {prefill_step_size} exceeds the rotating prompt_cache's "
                             f"max_chunk {prompt_cache.max_chunk}")
        if kv_bits is not None and kv_bits != prompt_cache.kv_bits:
            raise ValueError(f"generate: kv_bits={kv_bits!r} conflicts with the prompt_cache's kv_bits "
                             f"{prompt_cache.kv_bits!r} (the cache's settings apply)")
        if prompt_cache._batch != len(prompts):
            raise ValueError(f"generate: prompt_cache holds {prompt_cache._batch} rows, {len(prompts)} prompts given")
    start = [0] * len(prompts) if prompt_cache is None else list(prompt_cache.host_lens)
    limit = position_limit(model.args)
    longest = max(len(p) for p in prompts)
    reach = max(s + len(p) for s, p in zip(start, prompts)) + max_tokens
    if limit is not None and reach > limit:
        raise ValueError(f"cached ({max(start)}) + prompt ({longest} tokens) + max_tokens ({max_tokens}) exceeds "
                         f"max_position_embeddings ({limit}): training truncates there and the RoPE tables end there")
    rotating = max_kv_size is not None or (prompt_cache is not None and prompt_cache.rotating)
    if rotating and prefill_step_size is None:
        prefill_step_size = 512 if prompt_cache is None else min(512, prompt_cache.max_chunk)
    if prompt_cache is not None and not rotating and reach > prompt_cache.s_max:
        raise ValueError(f"generate: prompt_cache holds {prompt_cache.s_max} positions, {reach} needed (cached + prompt "
                         f"+ max_tokens)")
    chunked = prefill_step_size is not None or any(start)
    if chunked:
        if prefill_step_size is not None and model.args.prefix_lm and not any(start) and longest > prefill_step_size:
            raise ValueError("generate: a prefix-LM model's first prompt cannot be split into chunks (its prefix "
                             f"attends to keys of later chunks): prompt of {longest} tokens, prefill_step_size "
                             f"{prefill_step_size}")
        model.check_extend(prompt_cache)
    device = model.embed_tokens.weight.device
    gen = None
    if temperature != 0:
        gen = torch.Generator(device=device)
        gen.manual_seed(seed if seed is not None else time.time_ns() % (1 << 63))
    B = len(prompts)
    tokens = torch.zeros((B, longest), dtype=torch.int64)
    for b, p in enumerate(prompts):
        tokens[b, :len(p)] = torch.tensor(p, dtype=torch.int64)
    cache = prompt_cache
    if cache is None and rotating:
        cache = KVCache(model, B, longest + max_tokens, max_kv_size=max_kv_size, max_chunk=prefill_step_size)
    elif cache is None:
        cache = KVCache(model, B, longest + max_tokens, kv_bits, kv_group_size, quantized_kv_start)
    if chunked:
        logits = _prefill(model, prompts, cache, prefill_step_size)
    else:
        logits = model.prefill(tokens.to(device), [len(p) for p in prompts], cache)
    if draft_model is not None:
        draft_cache = KVCache(draft_model, B, longest + max_tokens)
        draft_step = draft_prefill_step(draft_model, prefill_step_size, longest)
        if draft_step is not None:
            _prefill(draft_model, prompts, draft_cache, draft_step)
        else:
            draft_model.prefill(tokens.to(device), [len(p) for p in prompts], draft_cache)
        sampler = (temperature, min_p, top_p, repetition_penalty, repetition_context_size, gen)
        return _speculative(model, draft_model, prompts, logits, cache, draft_cache, max_tokens, num_draft_tokens,
                            eos_token, sampler, on_round)
    history = [list(p) for p in prompts]
    out: List[List[int]] = [[] for _ in prompts]
    done = [False] * B
    live = None  # rotating: the rows that took a token this step (the others must not write into the ring)
    for step in range(max_tokens):
        if repetition_penalty != 1.0 and repetition_context_size > 0:
            logits = apply_repetition_penalty(logits, [repetition_window(h, repetition_context_size) for h in history],
                                              repetition_penalty)
        nxt = sample(logits, temperature, min_p, top_p, gen)
        picked = nxt.tolist()
        if rotating:
            live = None if not any(done) else [not d for d in done]
        for b, t in enumerate(picked):
            if done[b]:
                continue
            out[b].append(t)
            history[b].append(t)
            if eos_token is not None and t == eos_token:
                done[b] = True
        if on_step is not None:
            on_step(picked)
        if all(done) or step + 1 == max_tokens:
            break
        logits = model.decode_step(nxt, cache, live)
    if prompt_cache is not None and rotating:
        # the last tokens, fed only to the rows that took one: the ring then holds prompt + output of every row
        if max_tokens > 0:
            model.decode_step(nxt, cache, live)
    elif prompt_cache is not None:
        # the reference feeds every token it yields: feed the last ones, then drop what finished rows were fed past EOS
        if max_tokens > 0:
            model.decode_step(nxt, cache)
        cache.truncate([s + len(p) + len(o) for s, p, o in zip(start, prompts, out)])
    return out


# ------------------------------------------------------------------------------------------------
# speculative decoding (mlx_lm's generate with a draft_model; DESIGN §2 records each rule)
# ------------------------------------------------------------------------------------------------
MAX_DRAFT_TOKENS = 15  # the target verifies K + 1 <= 16 positions per row (ops.attention_decode_multi)


def check_draft(model, draft_model, num_draft_tokens, reach: int, kv_bits=None, max_kv_size=None, prompt_cache=None,
                on_step=None, num_beams=None) -> None:
    """Raises ValueError for a draft generate cannot run: a different vocabulary size, K outside 1..15, options a
    draft does not combine with, or a draft whose position limit is below reach = prompt + max_tokens."""
    if draft_model.vocab_size != model.vocab_size:
        raise ValueError(f"draft_model: vocabulary of {draft_model.vocab_size} tokens, the model has "
                         f"{model.vocab_size}: the draft must share the target's tokenizer")
    if isinstance(num_draft_tokens, bool) or not isinstance(num_draft_tokens, int) \
            or not 1 <= num_draft_tokens <= MAX_DRAFT_TOKENS:
        raise ValueError(f"num_draft_tokens must be an int in [1, {MAX_DRAFT_TOKENS}], got {num_draft_tokens!r}")
    for name, given in (("kv_bits", kv_bits is not None), ("max_kv_size (a ring cannot be rewound)",
                                                             max_kv_size is not None),
                        ("prompt_cache", prompt_cache is not None), ("num_beams", num_beams is not None),
                        ("on_step (use on_round)", on_step is not None)):
        if given:
            raise ValueError(f"draft_model does not combine with {name}")
    limit = position_limit(draft_model.args)
    if limit is not None and reach > limit:
        raise ValueError(f"draft_model: prompt + max_tokens ({reach}) exceeds the draft's max_position_embeddings "
                         f"({limit})")


def draft_prefill_step(draft_model, prefill_step_size: Optional[int], longest: int) -> Optional[int]:
    """The draft's prefill chunk: prefill_step_size when Model.extend serves the draft, else None (one piece).
    Model.extend needs a bf16 model with head_dim 64 or 128, and a prefix-LM prompt cannot be split; a draft outside
    that (C1: fp32, head_dim 16) is prefilled whole, as such drafts are small."""
    if prefill_step_size is None:
        return None
    try:
        draft_model.check_extend(None)
    except ValueError:
        return None
    if draft_model.args.prefix_lm and longest > prefill_step_size:
        return None
    return prefill_step_size


def check_draft_tokenizer(tokenizer, draft_tokenizer) -> None:
    """Raises ValueError when two runs' tokenizers differ: the byte-level vocabulary size, or the tokenizer file's
    contents."""
    def ident(t):  # a core.training.TokenizerManager
        path = t.config.tokenizer_path if t.external_tokenizer is not None else None
        data = (Path(path) / "tokenizer.json").read_bytes() if path is not None else None
        byte_level = t.config.tokenizer.get("normal_vocab_size") if path is None else None
        return t.VOCAB_SIZE, t.EOS_TOKEN, byte_level, data

    if ident(tokenizer) != ident(draft_tokenizer):
        raise ValueError("the draft run's tokenizer differs from the target run's (vocabulary or tokenizer file)")


def repetition_windows(history: Sequence[int], drafted: Sequence[int], context_size: int) -> List[List[int]]:
    """The repetition window of each of the k + 1 positions a round samples at, drafted = d_1 .. d_k: position i
    follows history + drafted[:i] (history ends with the round's input token), repetition_window's rule."""
    h = list(history)
    return [repetition_window(h + list(drafted[:i]), context_size) for i in range(len(drafted) + 1)]


def draft_counts(emitted: Sequence[int], done: Sequence[bool], K: int, max_tokens: int) -> List[int]:
    """Tokens each row drafts this round: min(K, max_tokens - emitted[b]) for a live row, 0 for a finished one."""
    return [0 if d else min(K, max_tokens - n) for n, d in zip(emitted, done)]


def accept_drafts(drafted: Sequence[int], sampled: Sequence[int], room: int, eos_token: Optional[int] = None):
    """One row's accept step.  drafted = d_1 .. d_k (k >= 1), sampled = the target's t_0 .. t_k, t_i sampled after
    the round's input token and d_1 .. d_i; room >= 1 tokens the row may still emit.  Drafts are accepted while
    t_i == d_{i+1}; the row emits them and then t_n, the target's token at the first mismatch or its bonus token t_k,
    cut after the first EOS and at room.  Returns (emitted, n accepted, stopped)."""
    n = 0
    while n < len(drafted) and sampled[n] == drafted[n]:
        n += 1
    emitted = list(drafted[:n]) + [int(sampled[n])]
    if eos_token is not None and eos_token in emitted:
        emitted = emitted[:emitted.index(eos_token) + 1]
    emitted = emitted[:room]
    stopped = len(emitted) == room or (eos_token is not None and emitted[-1] == eos_token)
    return emitted, n, stopped


def rewind(base: int, k: int, emitted: Sequence[int], drafted: Sequence[int]):
    """The caches after a round that started with the target holding base positions (its input token unfed at
    position base) and drafted k tokens: the target was fed the input and d_1 .. d_k, the draft the input (after any
    catch-up) and d_1 .. d_{k-1}.  Returns (target length, draft length, the draft's next input): both keep the input
    and the emitted tokens but the last, which is the next round's input; when all k drafts were accepted the draft
    never saw d_k, so its next input is [d_k, last]."""
    keep = base + len(emitted)
    draft_keep = min(keep, base + k)
    nxt = [int(emitted[-1])] if draft_keep == keep else [int(drafted[k - 1]), int(emitted[-1])]
    return keep, draft_keep, nxt


def _padded(rows: Sequence[Sequence[int]], device) -> torch.Tensor:
    t = torch.zeros((len(rows), max(1, max(len(r) for r in rows))), dtype=torch.int64)
    for b, r in enumerate(rows):
        t[b, :len(r)] = torch.tensor(list(r), dtype=torch.int64)
    return t.to(device)


def _feed(model, rows: Sequence[Sequence[int]], cache) -> torch.Tensor:
    """Appends rows[b] (0 to 16 tokens) to row b of the cache; returns the fp32 logits [B, V] after each row's last
    token (unspecified for an empty row).  One token for every row is a decode step, anything else Model.verify."""
    device = model.embed_tokens.weight.device
    counts = [len(r) for r in rows]
    if all(n == 1 for n in counts):
        return model.decode_step(_padded(rows, device)[:, 0], cache)
    logits = model.verify(_padded(rows, device), counts, cache)
    last = torch.tensor([max(n - 1, 0) for n in counts], device=device)
    return logits[torch.arange(len(rows), device=device), last]


def _speculative(model, draft_model, prompts, logits, cache, draft_cache, max_tokens, K, eos_token, sampler,
                 on_round):
    temperature, min_p, top_p, penalty, ctx, gen = sampler
    penalize = penalty != 1.0 and ctx > 0
    B = len(prompts)

    def pick(lg: torch.Tensor, idx: List[int], windows) -> List[int]:
        """Tokens sampled from rows idx of lg only (the others, a finished row's or a padding position's, hold
        unspecified logits), with windows[i] the repetition window of row idx[i]."""
        lg = lg[torch.tensor(idx, dtype=torch.int64, device=lg.device)]
        if penalize:
            lg = apply_repetition_penalty(lg, windows, penalty)
        return sample(lg, temperature, min_p, top_p, gen).tolist()

    device = model.embed_tokens.weight.device
    history = [list(p) for p in prompts]
    out: List[List[int]] = [[] for _ in prompts]
    done = [False] * B
    if max_tokens <= 0:
        return out
    # the first token is the target's sample after the prompt, as in plain generation
    for b, t in enumerate(pick(logits, list(range(B)), [repetition_window(h, ctx) for h in history])):
        out[b].append(t)
        history[b].append(t)
        done[b] = max_tokens == 1 or (eos_token is not None and t == eos_token)
    base = [len(p) for p in prompts]  # target positions held; the input token out[b][-1] sits at base[b]
    pending = [[out[b][-1]] for b in range(B)]  # the draft's next input
    while not all(done):
        k = draft_counts([len(o) for o in out], done, K, max_tokens)
        drafted: List[List[int]] = [[] for _ in prompts]
        dl = _feed(draft_model, [[] if done[b] else pending[b] for b in range(B)], draft_cache)
        for j in range(max(k)):
            need = [b for b in range(B) if j < k[b]]  # rows fed this step: the others' logits are unspecified
            d = dict(zip(need, pick(dl, need, [repetition_window(history[b] + drafted[b], ctx) for b in need])))
            for b in need:
                drafted[b].append(d[b])
            if j + 1 < max(k):
                dl = _feed(draft_model, [[d[b]] if j + 1 < k[b] else [] for b in range(B)], draft_cache)
        rows = [[] if done[b] else [out[b][-1]] + drafted[b] for b in range(B)]
        tl = model.verify(_padded(rows, device), [len(r) for r in rows], cache)  # [B, max k + 1, V]
        L = tl.shape[1]
        idx, windows = [], []  # the valid (row, position) pairs: k[b] + 1 per live row
        for b in range(B):
            if not done[b]:
                idx += [b * L + i for i in range(k[b] + 1)]
                windows += repetition_windows(history[b], drafted[b], ctx)
        flat = pick(tl.reshape(B * L, -1), idx, windows)
        t = {}
        for b in range(B):
            if not done[b]:
                t[b], flat = flat[:k[b] + 1], flat[k[b] + 1:]
        emitted_all: List[List[int]] = [[] for _ in prompts]
        keep, draft_keep = list(cache.host_lens), list(draft_cache.host_lens)
        for b in range(B):
            if done[b]:
                continue
            emitted, _, stopped = accept_drafts(drafted[b], t[b], max_tokens - len(out[b]), eos_token)
            keep[b], draft_keep[b], pending[b] = rewind(base[b], k[b], emitted, drafted[b])
            base[b] = keep[b]
            out[b] += emitted
            history[b] += emitted
            emitted_all[b] = emitted
            done[b] = stopped
        cache.truncate(keep)
        draft_cache.truncate(draft_keep)
        if on_round is not None:
            on_round(emitted_all, drafted)
    return out


# ------------------------------------------------------------------------------------------------
# beam search (generate_lite.py:400-484 of the reference; DESIGN §2 records each rule)
# ------------------------------------------------------------------------------------------------
Beam = Tuple[List[int], float]


def select_beams(beams: Sequence[Beam], top_tokens, top_logprobs, n: int, stop_tokens=None):
    """One step of the reference's selection for one group.  beams: the live beams (generated tokens, score) in order;
    top_tokens / top_logprobs: per beam, its top candidates in rank order (at least n).  Candidates are scored
    parent + log-probability (Python floats), ordered beam-major then by rank, stably sorted by score descending and
    popped until n are chosen; one ending in a stop token is finished instead (its token stripped, score -inf when it
    is the first generated token) and n drops by one.  Returns (chosen (parent index, token, score) in order, finished
    beams, the new n)."""
    stops = set(stop_tokens) if stop_tokens is not None else None
    cands = [(i, int(top_tokens[i][k]), score + float(top_logprobs[i][k]))
             for i, (_, score) in enumerate(beams) for k in range(n)]
    cands.sort(key=lambda c: c[2], reverse=True)
    chosen, finished = [], []
    for i, t, score in cands:
        if len(chosen) >= n:
            break
        if stops is not None and t in stops:
            finished.append((list(beams[i][0]), -math.inf if not beams[i][0] else score))
            n -= 1
        else:
            chosen.append((i, t, score))
    return chosen, finished, n


def plan_slots(slots: Sequence[int], free: Sequence[int], parents: Sequence[int]):
    """Copy-on-fork for one group.  slots[i]: the tail slot of live beam i; free: the group's unused slots; parents:
    the parent of each chosen child, in row order.  A parent's first child keeps its slot; each further child takes a
    free slot (those unused, then those of beams without children) that receives a copy of the parent's tail.
    Returns (the children's slots, (src, dst) copies, the slots left free)."""
    has_child = set(parents)
    pool = list(free) + [s for i, s in enumerate(slots) if i not in has_child]
    kept, out, copies = set(), [], []
    for p in parents:
        if p not in kept:
            kept.add(p)
            out.append(slots[p])
        else:
            d = pool.pop(0)
            copies.append((slots[p], d))
            out.append(d)
    return out, copies, pool


def beam_result(live: Sequence[Beam], finished: Sequence[Beam]) -> List[Beam]:
    """The reference's result: the live beams when nothing finished, else the finished beams and the live beams that
    generated a token; sorted by score descending (stable)."""
    res = list(live) if not finished else list(finished) + [b for b in live if len(b[0]) > 0]
    res.sort(key=lambda b: b[1], reverse=True)
    return [(list(t), s) for t, s in res]


def beam_search(model, prompts: List[List[int]], n_beams: int = 4, max_tokens: int = 512,
                stop_tokens: Optional[Sequence[int]] = None, *, kv_bits: Optional[int] = None,
                max_kv_size: Optional[int] = None, prompt_cache=None,
                on_step: Optional[Callable[[List[List[int]], torch.Tensor], None]] = None) -> List[List[Beam]]:
    """The reference's beam_search for each prompt, the prompts searched independently in one batch.  Returns per
    prompt the list of (generated tokens, score), best first (beam_result).  The model's logits go through
    log_softmax; there is no temperature, sampler or repetition penalty.  Each prompt is prefilled once and its cache
    shared by its beams (arch.llama.BeamKVCache); a beam step reads back the [rows, n] candidates once, selects on the
    host (select_beams), forks the tails (plan_slots) and runs Model.decode_step over the live beams.  A quantized or
    rotating cache and continuing from a prompt_cache are not supported.  on_step(rows, logits), if given, sees each
    step's decode rows (prompt + generated tokens, in row order) and their fp32 logits [rows, V] before selection."""
    from ..arch.llama import BeamKVCache, KVCache

    if isinstance(n_beams, bool) or not isinstance(n_beams, int) or n_beams < 1:
        raise ValueError(f"beam_search: n_beams must be an int >= 1, got {n_beams!r}")
    if kv_bits is not None or max_kv_size is not None or prompt_cache is not None:
        raise ValueError("beam_search: kv_bits, max_kv_size and prompt_cache are not supported (the beams share one "
                         "unquantized, unbounded prompt cache)")
    if not prompts or any(len(p) == 0 for p in prompts):
        raise ValueError("beam_search: every prompt needs at least one token")
    if isinstance(max_tokens, bool) or not isinstance(max_tokens, int) or max_tokens < 0:
        raise ValueError(f"beam_search: max_tokens must be an int >= 0, got {max_tokens!r}")
    limit = position_limit(model.args)
    longest = max(len(p) for p in prompts)
    if limit is not None and longest + max_tokens > limit:
        raise ValueError(f"prompt ({longest} tokens) + max_tokens ({max_tokens}) exceeds max_position_embeddings "
                         f"({limit}): training truncates there and the RoPE tables end there")
    G = len(prompts)
    if max_tokens == 0:
        return [[([], 0.0) for _ in range(n_beams)] for _ in prompts]
    device = model.embed_tokens.weight.device
    tokens = torch.zeros((G, longest), dtype=torch.int64)
    for g, p in enumerate(prompts):
        tokens[g, :len(p)] = torch.tensor(p, dtype=torch.int64)
    prefix = KVCache(model, G, longest)
    logits = model.prefill(tokens.to(device), [len(p) for p in prompts], prefix)
    cache = BeamKVCache(model, prefix, n_beams, max_tokens)
    # per group: live beams, their slots, the free slots, n, finished beams (step 0 starts from one beam per prompt:
    # the reference's n identical copies give the same candidates once duplicates are dropped)
    beams: List[List[Beam]] = [[([], 0.0)] for _ in prompts]
    slots = [[g * n_beams] for g in range(G)]
    free = [list(range(g * n_beams + 1, (g + 1) * n_beams)) for g in range(G)]
    n = [n_beams] * G
    finished: List[List[Beam]] = [[] for _ in prompts]
    for step in range(max_tokens):
        alive = [g for g in range(G) if beams[g]]
        if on_step is not None:
            on_step([list(prompts[g]) + b[0] for g in alive for b in beams[g]], logits)
        width = max(n[g] for g in alive)
        logprobs = torch.log_softmax(logits, dim=-1)
        top = _sorted_desc(logprobs)[:, :width]
        host = torch.cat([top.double(), torch.gather(logprobs, -1, top).double()], dim=1).cpu().tolist()
        r = 0
        rows_g, rows_slot, rows_len, next_tokens, copies = [], [], [], [], []
        for g in alive:
            rows = host[r:r + len(beams[g])]
            r += len(beams[g])
            chosen, done, n[g] = select_beams(beams[g], [x[:width] for x in rows], [x[width:] for x in rows], n[g],
                                              stop_tokens)
            finished[g] += done
            parents = [c[0] for c in chosen]
            new_slots, pairs, free[g] = plan_slots(slots[g], free[g], parents)
            held = len(prompts[g]) + step - cache.t0[g]  # tail positions each parent holds
            copies += [(s, d, held) for s, d in pairs]
            beams[g] = [(beams[g][i][0] + [t], score) for i, t, score in chosen]
            slots[g] = new_slots
            rows_g += [g] * len(chosen)
            rows_slot += new_slots
            rows_len += [len(prompts[g]) + step] * len(chosen)
            next_tokens += [t for _, t, _ in chosen]
        if step + 1 == max_tokens or not next_tokens:
            break
        cache.set_rows(rows_g, rows_slot, rows_len)
        cache.fork(copies)
        logits = model.decode_step(torch.tensor(next_tokens, dtype=torch.int64).to(device), cache)
    return [beam_result(beams[g], finished[g]) for g in range(G)]


# ------------------------------------------------------------------------------------------------
# CLI (core/generation.py:10-78 of the reference)
# ------------------------------------------------------------------------------------------------
def parse_args(argv: Optional[List[str]] = None) -> argparse.Namespace:
    ap = argparse.ArgumentParser(description="Generate text using a trained model")
    ap.add_argument("--run", type=str, required=True, help="Name of the training run to use")
    ap.add_argument("--prompt", type=str, required=True, help="Text prompt to start generation")
    ap.add_argument("--max-tokens", type=int, default=256, help="Maximum number of tokens to generate")
    ap.add_argument("--temperature", type=float, default=1.0, help="Sampling temperature (0: greedy)")
    ap.add_argument("--min-p", type=float, default=0.05, help="Minimum probability for min-p sampling")
    ap.add_argument("--repetition-penalty", type=float, default=1.1, help="Repetition penalty factor")
    ap.add_argument("--repetition-context-size", type=int, default=20, help="Context size for repetition penalty")
    ap.add_argument("--top-p", type=float, default=None, help="Nucleus threshold (used when --min-p is 0)")
    ap.add_argument("--seed", type=int, default=None, help="Sampling seed (default: from the clock)")
    ap.add_argument("--num-samples", type=int, default=1, help="Rows decoded as one batch")
    ap.add_argument("--checkpoint", type=str, default=None,
                    help="Checkpoint to load, e.g. step_1000 (default: the final checkpoint)")
    ap.add_argument("--runs-dir", type=str, default="runs", help="Directory holding the run directories")
    ap.add_argument("--kv-bits", type=int, choices=(4, 8), default=None,
                    help="Quantize the KV cache to this many bits (default: no quantization)")
    ap.add_argument("--kv-group-size", type=int, choices=(32, 64, 128), default=64,
                    help="Group size of the KV cache quantization")
    ap.add_argument("--quantized-kv-start", type=int, default=0,
                    help="Quantize the KV cache once it holds more than this many tokens")
    ap.add_argument("--prefill-step-size", type=int, default=None,
                    help="Prefill the prompt in chunks of this many tokens (default: the whole prompt at once)")
    ap.add_argument("--max-kv-size", type=int, default=None,
                    help="Keep a rotating KV cache: each token attends to the first 4 and the most recent "
                         "max-kv-size - 4 tokens (default: an unbounded cache)")
    ap.add_argument("--num-beams", type=int, default=None,
                    help="Beam search with this many beams, printing every returned beam with its score (default: "
                         "sampling).  The sampling flags (temperature, min-p, top-p, repetition penalty, seed) do not "
                         "apply to it, as in the reference")
    ap.add_argument("--draft-run", type=str, default=None,
                    help="Speculative decoding: a run with the same tokenizer whose model drafts tokens for this one")
    ap.add_argument("--draft-checkpoint", type=str, default=None,
                    help="Checkpoint of the draft run (default: its final checkpoint)")
    ap.add_argument("--num-draft-tokens", type=int, default=3,
                    help="Tokens the draft proposes per round, 1 to 15 (with --draft-run)")
    a = ap.parse_args(argv)
    if a.draft_run is not None:
        if not 1 <= a.num_draft_tokens <= MAX_DRAFT_TOKENS:
            ap.error(f"--num-draft-tokens must lie in [1, {MAX_DRAFT_TOKENS}]")
        for flag, given in (("--num-beams", a.num_beams is not None), ("--kv-bits", a.kv_bits is not None),
                            ("--max-kv-size", a.max_kv_size is not None)):
            if given:
                ap.error(f"--draft-run does not combine with {flag}")
    elif a.draft_checkpoint is not None:
        ap.error("--draft-checkpoint needs --draft-run")
    if a.num_beams is not None:
        if a.num_beams < 1:
            ap.error("--num-beams must be >= 1")
        for flag, given in (("--num-samples > 1", a.num_samples > 1), ("--kv-bits", a.kv_bits is not None),
                            ("--max-kv-size", a.max_kv_size is not None),
                            ("--prefill-step-size", a.prefill_step_size is not None)):
            if given:
                ap.error(f"--num-beams does not combine with {flag}")
    if a.num_samples < 1:
        ap.error("--num-samples must be >= 1")
    if a.quantized_kv_start < 0:
        ap.error("--quantized-kv-start must be >= 0")
    if a.prefill_step_size is not None and a.prefill_step_size < 1:
        ap.error("--prefill-step-size must be >= 1")
    if a.max_kv_size is not None and a.max_kv_size < 5:
        ap.error("--max-kv-size must be >= 5")
    return a


def resolve_checkpoint(run_dir: Path, checkpoint: Optional[str] = None) -> Path:
    """Model weights of a run: checkpoints/<checkpoint>_model.safetensors (or the exact file name given), else
    step_final_model.safetensors, then step_final.safetensors, as the reference looks them up."""
    ck = Path(run_dir) / "checkpoints"
    if checkpoint is not None:
        for cand in (ck / f"{checkpoint}_model.safetensors", ck / checkpoint, ck / f"{checkpoint}.safetensors"):
            if cand.is_file():
                return cand
        raise ValueError(f"Checkpoint {checkpoint} not found in {ck}")
    for name in ("step_final_model.safetensors", "step_final.safetensors"):
        if (ck / name).is_file():
            return ck / name
    raise ValueError(f"Final checkpoint not found for run: {Path(run_dir).name}")


def load_run(run: str, runs_dir: str = "runs", checkpoint: Optional[str] = None):
    """Trainer(cfg, for_training=False) of a run with the checkpoint's weights in its parameter store."""
    from safetensors.torch import load_file
    from .training import Config, Trainer

    run_dir = Path(runs_dir) / run
    cfg_path = run_dir / "config.yaml"
    if not cfg_path.is_file():
        raise ValueError(f"Config not found for run: {run} ({cfg_path})")
    path = resolve_checkpoint(run_dir, checkpoint)
    cfg = Config.from_yaml(str(cfg_path))
    trainer = Trainer(cfg, for_training=False, run_root=str(Path(runs_dir)), quiet=True)
    weights = load_file(str(path))
    store = trainer.store
    with torch.no_grad():
        for name, (_, shape) in store.index.items():
            if name not in weights:
                raise ValueError(f"{path.name}: parameter {name} missing")
            if tuple(weights[name].shape) != tuple(shape):
                raise ValueError(f"{path.name}: parameter {name} has shape {tuple(weights[name].shape)}, "
                                 f"the model expects {tuple(shape)}")
        for name, t in weights.items():
            if name in store.index:  # non-strict, like Trainer.load_checkpoint
                store.view(store.master, name).copy_(t.to(trainer.device))
        store.refresh_shadow()
    trainer.model.eval()
    return trainer


def main(argv: Optional[List[str]] = None) -> None:
    a = parse_args(argv)
    trainer = load_run(a.run, a.runs_dir, a.checkpoint)
    tok = trainer.tokenizer
    prompt = [tok.BOS_TOKEN] + tok.tokenize(a.prompt)
    if a.num_beams is not None:
        for toks, score in beam_search(trainer.model, [prompt], n_beams=a.num_beams, max_tokens=a.max_tokens,
                                       stop_tokens=[tok.EOS_TOKEN])[0]:
            print(f"Beam Output (Score: {score:.3f}): {tok.detokenize(toks)}")
        sys.stdout.flush()
        return
    seed = a.seed if a.seed is not None else random.SystemRandom().randrange(1 << 62)
    draft, counts = None, [0, 0]
    if a.draft_run is not None:
        draft_trainer = load_run(a.draft_run, a.runs_dir, a.draft_checkpoint)
        check_draft_tokenizer(tok, draft_trainer.tokenizer)
        draft = draft_trainer.model

    def on_round(emitted, drafted):
        for e, d in zip(emitted, drafted):
            n = 0
            while n < min(len(e), len(d)) and e[n] == d[n]:
                n += 1
            counts[0] += n
            counts[1] += len(d)

    outs = generate(trainer.model, [prompt] * a.num_samples, max_tokens=a.max_tokens, temperature=a.temperature,
                    min_p=a.min_p, top_p=a.top_p, repetition_penalty=a.repetition_penalty,
                    repetition_context_size=a.repetition_context_size, eos_token=tok.EOS_TOKEN, seed=seed,
                    kv_bits=a.kv_bits, kv_group_size=a.kv_group_size, quantized_kv_start=a.quantized_kv_start,
                    prefill_step_size=a.prefill_step_size, max_kv_size=a.max_kv_size, draft_model=draft,
                    num_draft_tokens=a.num_draft_tokens, on_round=on_round if draft is not None else None)
    if draft is not None:
        rate = counts[0] / counts[1] if counts[1] else 0.0
        sys.stderr.write(f"[speculative] {counts[0]} of {counts[1]} draft tokens accepted ({rate:.1%})\n")
    for o in outs:
        print(f"Greedy Output: {tok.detokenize(o)}")
    sys.stdout.flush()


if __name__ == "__main__":
    main()
