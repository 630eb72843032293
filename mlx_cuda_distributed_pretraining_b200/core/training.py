"""`python -m core.training --config <yaml>` -- the reference's entry point (core/training.py),
re-hosted on the CUDA hot path (H100).

Kept from the reference: the YAML schema (dataclasses core/training.py:52-138), `Config.from_yaml`
(:141-167), the byte-level / tokenizers-JSON `TokenizerManager` (:324-440), JSONL chunking
`DataManager` (:442-543), schedules (mlx_lm_utils.py:5-56 as joined in :770-785), the optimizer
factory names (:787-896), `compute_loss` (:1195-1234), the hot loop's order of operations
(:1637-1768: fwd/bwd -> fp32 grads -> elementwise clip -> accumulate -> optimizer.update),
the `Step n: k=v | ...` log line (:257-271) and the three-file checkpoint layout (:1347-1394).

Replaced: mlx arrays/autograd -> PyTorch autograd over the sm_90a kernels; the thread-queue
"devices" (distributed/utils.py) -> one process per GPU with an NCCL all-reduce of the flat
gradient buffer, engaged only when `system.distributed: true` and the job runs under torchrun.

Synthetic data: `data.input_file: synthetic` (or Trainer(..., synthetic=True)) draws
randint(0, normal_vocab_size, (B, S+1)) with seed 42 + 1000*step + rank (SURVEY 8d), which is what
bench.py and the parity tests use; there is no network for real corpora here.
"""
from __future__ import annotations

import argparse
import json
import logging
import math
import os
import random
import sys
import time
from dataclasses import asdict, dataclass, field
from datetime import datetime
from pathlib import Path
from typing import Any, Callable, Dict, List, Optional, Tuple

import numpy as np
import torch
import yaml

from .. import ops
from ..arch.llama import Model, ModelArgs
from ..distributed import dp
from ..flat import ParamStore
from ..optimizers import SGD, AdamW, HybridOptimizer, Lion, Muon, SGDEnhanced, Shampoo, ShampooParams


# ------------------------------------------------------------------------------------------------
# configuration (same sections and keys as the reference)
# ------------------------------------------------------------------------------------------------
@dataclass
class DataConfig:
    input_file: str
    preprocessing: Dict[str, int]
    tokenizer: Dict[str, Any]
    tokenizer_path: Optional[str] = None
    validation_file: Optional[str] = None
    weight_path: Optional[str] = None


@dataclass
class ModelConfig:
    architecture: str
    dimensions: Dict[str, int]
    attention: Dict[str, Any]
    normalization: Dict[str, float]
    rope: Dict[str, Any]
    misc: Dict[str, bool]

    def __post_init__(self):
        # extension: attention.sliding_window W (absent / null: full causal); query q sees keys q - W .. q
        w = self.attention.get("sliding_window")
        if w is not None and (isinstance(w, bool) or not isinstance(w, int) or w < 0):
            raise ValueError(f"model.attention.sliding_window must be null or a non-negative integer, got {w!r}")
        # extension: attention.alibi (absent / null / false: off); ALiBi's bias slope_h * (k - q) on every score
        a = self.attention.get("alibi")
        if a is not None and not isinstance(a, bool):
            raise ValueError(f"model.attention.alibi must be null, true or false, got {a!r}")
        # extension: attention.prefix_lm (absent / null / false: off); each row's prefix attends bidirectionally
        pl = self.attention.get("prefix_lm")
        if pl is not None and not isinstance(pl, bool):
            raise ValueError(f"model.attention.prefix_lm must be null, true or false, got {pl!r}")
        if pl:
            if w is not None:
                raise ValueError("model.attention.prefix_lm does not combine with model.attention.sliding_window")
            if a:
                raise ValueError("model.attention.prefix_lm does not combine with model.attention.alibi")
        # extension: attention.dropout p (absent / null / 0: off); drops attention weights after the softmax in
        # training (arch/flash_attention.py:146-148 of the reference)
        d = self.attention.get("dropout")
        if d is not None and (isinstance(d, bool) or not isinstance(d, (int, float)) or not 0.0 <= d < 1.0):
            raise ValueError(f"model.attention.dropout must be null or a number in [0, 1), got {d!r}")
        if d and pl:
            raise ValueError("model.attention.dropout does not combine with model.attention.prefix_lm")
        # extension: misc.variant selects the block (absent / null / "reference": arch/llama.py's; "mlx_lm": the
        # mlx_lm.models.llama block the reference's trainer actually imports, DESIGN D4)
        v = (self.misc or {}).get("variant")
        if v is not None and (not isinstance(v, str) or v not in ("reference", "mlx_lm")):
            raise ValueError(f"model.misc.variant must be null, 'reference' or 'mlx_lm', got {v!r}")
        if v == "mlx_lm":
            if self.rope.get("enabled", True) is False:
                raise ValueError("model.misc.variant: mlx_lm always applies RoPE; rope.enabled: false contradicts it")
            if self.rope.get("scaling") is not None:
                raise ValueError(f"model.misc.variant: mlx_lm does not support rope.scaling "
                                 f"(got {self.rope.get('scaling')!r}); set it to null")
        validate_moe_keys(self.misc or {})


def _int_or_none(misc: Dict[str, Any], key: str) -> int:
    v = misc.get(key)
    if v is None:
        return 0
    if isinstance(v, bool) or not isinstance(v, int):
        raise ValueError(f"model.misc.{key} must be null or an integer, got {v!r}")
    return v


def validate_moe_keys(misc: Dict[str, Any]) -> None:
    """model.misc.num_local_experts E (absent / null / 0: dense MLP; 2..64: every layer's MLP becomes a sparse MLP of E
    experts), num_experts_per_tok k (1..min(E, 8); absent / null / 0 when dense) and router_aux_loss_coef c (finite,
    >= 0; default 0.001 as in MixtralConfig)."""
    E = _int_or_none(misc, "num_local_experts")
    k = _int_or_none(misc, "num_experts_per_tok")
    if E != 0 and not 2 <= E <= 64:
        raise ValueError(f"model.misc.num_local_experts must be null, 0 or 2..64, got {E!r}")
    if E == 0 and k != 0:
        raise ValueError(f"model.misc.num_experts_per_tok={k} needs num_local_experts > 0")
    if E > 0 and not 1 <= k <= min(E, 8):
        raise ValueError(f"model.misc.num_experts_per_tok must lie in 1..{min(E, 8)} with {E} experts, got {k!r}")
    c = misc.get("router_aux_loss_coef", 0.001)
    if isinstance(c, bool) or not isinstance(c, (int, float)) or not math.isfinite(c) or c < 0:
        raise ValueError(f"model.misc.router_aux_loss_coef must be a finite number >= 0, got {c!r}")
    if E > 0 and misc.get("mlp_bias"):
        raise ValueError("model.misc.mlp_bias: true is not supported with num_local_experts > 0 (experts have no bias)")


@dataclass
class TrainingConfig:
    hyperparameters: Dict[str, Any]
    scheduler: Dict[str, Any]
    optimization: Dict[str, Any]
    epochs: Optional[int] = None
    early_stopping: Dict[str, Any] = field(default_factory=lambda: {
        "enabled": False, "patience": 3, "min_delta": 0.001, "metric": "val_loss", "mode": "min"})
    lr_finder: Dict[str, Any] = field(default_factory=lambda: {
        "enabled": False, "min_lr": 1e-7, "max_lr": 1.0, "num_steps": 100})


@dataclass
class LoggingConfig:
    log_dir: str
    checkpoint_dir: str
    steps: Dict[str, int]
    metrics: Dict[str, bool]
    tensorboard: bool = False
    wandb: bool = False
    wandb_project: Optional[str] = None
    wandb_entity: Optional[str] = None
    log_memory_usage: bool = False
    log_gradient_norm: bool = False
    log_parameter_norm: bool = False
    log_samples: bool = False
    log_samples_count: int = 3


@dataclass
class SystemConfig:
    seed: int
    device: str
    distributed: bool = False
    devices: Optional[List[str]] = None
    cuda_devices: Optional[List[int]] = None
    memory_limit: Optional[int] = None
    mixed_precision: bool = False
    precision: str = "float16"
    gradient_checkpointing: bool = False
    gradient_checkpointing_ratio: float = 0.5
    model_parallel: bool = False
    model_parallel_size: int = 1
    zero_optimization_level: int = 0


@dataclass
class ResumeConfig:
    checkpoint: str
    reset_optimizer: bool = False
    reset_training_state: bool = False


@dataclass
class Config:
    name: str
    data: DataConfig
    model: ModelConfig
    training: TrainingConfig
    logging: LoggingConfig
    system: SystemConfig
    resume: Optional[ResumeConfig] = None
    overwrite: bool = False

    def __post_init__(self):
        if self.model.attention.get("prefix_lm") and (self.data.preprocessing or {}).get("pack_sequences"):
            raise ValueError("model.attention.prefix_lm does not combine with data.preprocessing.pack_sequences "
                             "(a prefix per packed document is not supported)")
        E = _int_or_none(self.model.misc or {}, "num_local_experts")
        if E > 0:
            opt = self.training.optimization or {}
            names = {opt.get("optimizer"),
                     opt.get("matrix_optimizer", "muon") if opt.get("optimizer") == "hybrid" else None}
            inter = (self.model.dimensions or {}).get("intermediate_size")
            if not isinstance(inter, int) or inter % 64 != 0:
                raise ValueError(f"model.dimensions.intermediate_size must be a multiple of 64 with num_local_experts "
                                 f"> 0 (the expert GEMMs' k-blocks), got {inter!r}")
            if "shampoo" in names:
                raise ValueError("optimization.optimizer: shampoo is not supported with num_local_experts > 0 "
                                 "(Shampoo on stacked expert weights is out of scope); use muon, adamw, lion or sgd")
            if not self.system.mixed_precision:
                raise ValueError("model.misc.num_local_experts > 0 needs system.mixed_precision: true "
                                 "(the expert kernels take bf16 operands)")

    @classmethod
    def from_dict(cls, d: Dict[str, Any]) -> "Config":
        if "name" not in d:
            raise ValueError("Config must specify a 'name' field at the top level")
        training = dict(d["training"])
        epochs = training.pop("epochs", None)
        resume = ResumeConfig(**d["resume"]) if d.get("resume") else None
        return cls(name=d["name"], overwrite=d.get("overwrite", False), data=DataConfig(**d["data"]),
                   model=ModelConfig(**d["model"]), training=TrainingConfig(**training, epochs=epochs),
                   logging=LoggingConfig(**d["logging"]), system=SystemConfig(**d["system"]), resume=resume)

    @classmethod
    def from_yaml(cls, yaml_path: str) -> "Config":
        with open(yaml_path, "r") as f:
            return cls.from_dict(yaml.safe_load(f))


# ------------------------------------------------------------------------------------------------
# schedules (mlx_lm_utils.py:5-56)
# ------------------------------------------------------------------------------------------------
def linear_schedule(start_value, end_value, steps):
    def schedule(step):
        return end_value if step >= steps else start_value + (end_value - start_value) * (step / steps)
    return schedule


def cosine_decay(start_value, steps, end_value=0.0):
    def schedule(step):
        if step >= steps:
            return end_value
        return end_value + (start_value - end_value) * 0.5 * (1 + math.cos(math.pi * (step / steps)))
    return schedule


def join_schedules(schedules, transition_steps):
    def schedule(step):
        for i, t in enumerate(transition_steps):
            if step < t:
                return schedules[i](step)
        return schedules[-1](step - transition_steps[-1])
    return schedule


# ------------------------------------------------------------------------------------------------
# tokenizer / data
# ------------------------------------------------------------------------------------------------
class TokenizerManager:
    def __init__(self, config: DataConfig, run_dir: Optional[Path] = None, synthetic: bool = False):
        self.config = config
        self.external_tokenizer = None
        if config.tokenizer_path is not None and not synthetic:
            self.use_external_tokenizer(config.tokenizer_path)
        else:
            self.setup_vocabulary()

    def use_external_tokenizer(self, tokenizer_path: str) -> None:
        from tokenizers import Tokenizer
        tokenizer_file = os.path.join(tokenizer_path, "tokenizer.json")
        if not os.path.exists(tokenizer_file):
            raise ValueError(f"Tokenizer file not found at {tokenizer_file}")
        self.external_tokenizer = Tokenizer.from_file(tokenizer_file)
        vocab = self.external_tokenizer.get_vocab()
        sp = self.config.tokenizer["special_tokens"]
        self.PAD_TOKEN, self.BOS_TOKEN, self.EOS_TOKEN = vocab.get(sp["pad"]), vocab.get(sp["bos"]), vocab.get(sp["eos"])
        self.VOCAB_SIZE = len(vocab)
        if None in (self.PAD_TOKEN, self.BOS_TOKEN, self.EOS_TOKEN):
            raise ValueError("One or more special tokens not found in the external tokenizer vocabulary")

    def setup_vocabulary(self) -> None:
        n = self.config.tokenizer["normal_vocab_size"]
        sp = self.config.tokenizer["special_tokens"]
        self.special_token_map = {tok: n + i for i, tok in enumerate(sp.values())}
        self.PAD_TOKEN = self.special_token_map[sp["pad"]]
        self.BOS_TOKEN = self.special_token_map[sp["bos"]]
        self.EOS_TOKEN = self.special_token_map[sp["eos"]]
        self.VOCAB_SIZE = n + len(self.special_token_map)

    def tokenize(self, text: str) -> list:
        if self.external_tokenizer is not None:
            return self.external_tokenizer.encode(text).ids
        return list(text.encode("utf-8"))

    def detokenize(self, tokens) -> str:
        if hasattr(tokens, "tolist"):
            tokens = tokens.tolist()
        if self.external_tokenizer is not None:
            return self.external_tokenizer.decode(tokens)
        return bytes(t for t in tokens if t < 256).decode("utf-8", errors="ignore")

    def tokenize_doc(self, doc: str) -> list:
        max_length = self.config.preprocessing["max_context_size"]
        return [self.BOS_TOKEN] + self.tokenize(doc)[:max_length] + [self.EOS_TOKEN]


class SyntheticData:
    """SURVEY 8d synthetic token stream; same draws for the CUDA path and the CPU oracle.

    `data.input_file: synthetic`         uniform tokens (BASELINE configs), optimum loss = ln(vocab)
    `data.input_file: synthetic:markov`  a fixed first-order Markov chain (4 successors per token, 10 % uniform
                                         noise): LEARNABLE, so a loss curve can tell two optimizers apart; the
                                         oracle's twin is reference_math.synthetic_batch_markov (same draws)."""

    def __init__(self, vocab: int, batch_size: int, seq_len: int, rank: int = 0, num_batches: int = 1 << 30,
                 kind: str = "uniform", prefix_lm: bool = False):
        self.vocab, self.batch_size, self.seq_len, self.rank = vocab, batch_size, seq_len, rank
        self.prefix_lm = prefix_lm
        self.train_docs = range(num_batches * batch_size)
        self.has_validation_data = False
        self.num_validation_batches = 0
        self.val_ptr = 0
        self.kind = kind
        if kind not in ("uniform", "markov"):
            raise ValueError(f"unknown synthetic data kind {kind!r} (uniform | markov)")
        self._succ = (torch.randint(0, vocab, (vocab, 4), generator=torch.Generator().manual_seed(4242), dtype=torch.int64)
                      if kind == "markov" else None)

    def generate_batch(self, step: int) -> torch.Tensor:
        """[B, S + 1] tokens; with prefix_lm, [B, 1 + S + 1] with each row's split point in column 0, drawn uniformly
        from [0, S] by split_points (the tokens are the same draws as without prefix_lm)."""
        toks = self._tokens(step)
        if not self.prefix_lm:
            return toks
        P = split_points([self.seq_len] * self.batch_size, train_split_seed(step, self.rank))
        return torch.cat([P[:, None], toks], dim=1)

    def _tokens(self, step: int) -> torch.Tensor:
        g = torch.Generator().manual_seed(42 + 1000 * step + self.rank)
        B, S = self.batch_size, self.seq_len
        if self.kind == "uniform":
            return torch.randint(0, self.vocab, (B, S + 1), generator=g, dtype=torch.int64)
        out = torch.empty((B, S + 1), dtype=torch.int64)
        out[:, 0] = torch.randint(0, self.vocab, (B,), generator=g, dtype=torch.int64)
        choice = torch.randint(0, 4, (B, S), generator=g, dtype=torch.int64)
        noisy = torch.rand((B, S), generator=g) < 0.1
        rnd = torch.randint(0, self.vocab, (B, S), generator=g, dtype=torch.int64)
        for t in range(S):
            out[:, t + 1] = torch.where(noisy[:, t], rnd[:, t], self._succ[out[:, t], choice[:, t]])
        return out


def train_split_seed(step: int, rank: int) -> int:
    """Seed of the prefix-LM split points of training step `step` on data-parallel rank `rank`."""
    return 0x5EED_0000 + 4096 * step + rank


def val_split_seed(batch_idx: int) -> int:
    """Seed of the prefix-LM split points of validation batch `batch_idx`."""
    return 0x7A1_0000 + batch_idx


def split_points(lengths: List[int], seed: int) -> torch.Tensor:
    """Prefix-LM split points (int64 [len(lengths)]): row b's P is uniform in [0, lengths[b]], drawn from a generator
    of its own seeded with `seed`, so the shuffling and the token stream are untouched by the draws."""
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(len(lengths), generator=g, dtype=torch.float64)
    n = torch.tensor(lengths, dtype=torch.float64)
    return torch.minimum((u * (n + 1)).floor(), n).to(torch.int64)


def prefix_targets(targets: torch.Tensor, prefix: torch.Tensor, pad_token: int) -> torch.Tensor:
    """Targets [B, S] of prefix-LM rows with prefix lengths prefix [B]: a prefix position q <= P_b - 2 sees its own
    target x[q + 1], so those targets become PAD (no loss, no token count); the target at q = P_b - 1, the first token
    after the prefix, is kept.  Runs on the targets' device without a host synchronisation."""
    q = torch.arange(targets.shape[1], device=targets.device)
    return targets.masked_fill(q[None, :] < (prefix.to(targets.device)[:, None] - 1), pad_token)


def pack_first_fit(lengths: List[int], capacity: int) -> List[List[int]]:
    """First-fit bin packing in the given order: item i goes to the lowest-numbered row with at least lengths[i]
    free slots, or opens a new row.  Returns each row's item indices in placement order.  A max-tree over the rows'
    free space finds that row in O(log rows)."""
    size = 1
    while size < max(len(lengths), 1):
        size *= 2
    free = [0] * (2 * size)  # leaves: free slots of rows (0 until opened); inner nodes: max of the children
    rows: List[List[int]] = []
    for i, n in enumerate(lengths):
        if n > capacity:
            raise ValueError(f"item {i} of length {n} exceeds the row capacity {capacity}")
        if free[1] >= n:
            node = 1
            while node < size:
                node = 2 * node if free[2 * node] >= n else 2 * node + 1
            r = node - size
        else:
            r = len(rows)
            rows.append([])
            node = size + r
            free[node] = capacity
        rows[r].append(i)
        free[node] -= n
        node //= 2
        while node:
            free[node] = max(free[2 * node], free[2 * node + 1])
            node //= 2
    return rows


def document_positions(inputs: torch.Tensor, bos_token: int) -> torch.Tensor:
    """pos (int32, inputs' shape [B, S]) of packed token rows: each token's position within its document, where a
    document starts at every BOS token.  Tokens before a row's first BOS count from the row start.  Runs on the
    inputs' device without a host synchronisation."""
    S = inputs.shape[-1]
    idx = torch.arange(S, device=inputs.device, dtype=torch.int64).expand_as(inputs)
    start = torch.where(inputs == bos_token, idx, torch.zeros_like(idx)).cummax(dim=-1).values
    return (idx - start).to(torch.int32)


def _doc_len(doc) -> int:
    """Characters of a text chunk or of a prompt / completion pair (the order the batches are formed in)."""
    return len(doc) if isinstance(doc, str) else len(doc[0]) + len(doc[1])


class DataManager:
    """Unpacked (default): each training row is one chunk, padded to the longest chunk of its batch.

    `data.preprocessing.pack_sequences: true`: training rows of max_context_size + 1 tokens hold whole tokenised
    chunks (tokenize_doc: BOS first), placed first-fit in the shuffled order, tails filled with PAD; a chunk longer
    than a row is cut to the row.  Every chunk appears once per epoch.  The packed batches are walked in a permuted
    order drawn from the same global RNG after the unpacked state, so the validation batches (never packed) are the
    unpacked run's.

    prefix_lm: a `{"prompt": ..., "completion": ...}` line is one document, never chunked, whose row is
    [BOS] + tokenize(prompt) + tokenize(completion) + [EOS] with the prefix P = 1 + len(tokenize(prompt)); a `{"text":
    ...}` chunk's P is drawn uniformly from [0, n_b] (n_b: the row's non-PAD inputs) by split_points.  Rows are
    truncated as without prefix_lm and P is clipped to the row.  Batches are then [B, 1 + S + 1] with P in column 0."""

    def __init__(self, config: DataConfig, tokenizer: TokenizerManager, batch_size: int = 1, rank: int = 0,
                 world: int = 1, prefix_lm: bool = False):
        self.config, self.tokenizer, self.batch_size = config, tokenizer, batch_size
        self.rank, self.world = rank, world
        self.prefix_lm = prefix_lm
        self.train_docs: List[Any] = []
        self.val_docs: List[Any] = []
        self.val_ptr = 0
        self._load_file(config.input_file, self.train_docs)
        idx = sorted(range(len(self.train_docs)), key=lambda i: _doc_len(self.train_docs[i]))
        random.shuffle(idx)
        self.train_batch_idx = [idx[i:i + batch_size] for i in range(0, len(idx) - batch_size + 1, batch_size)]
        self.train_indices = np.random.permutation(len(self.train_batch_idx))
        self.val_batch_idx: List[List[int]] = []
        if config.validation_file:
            self._load_file(config.validation_file, self.val_docs)
            vidx = sorted(range(len(self.val_docs)), key=lambda i: _doc_len(self.val_docs[i]))
            self.val_batch_idx = [vidx[i:min(i + batch_size, len(vidx))] for i in range(0, len(vidx), batch_size)]
            self.val_indices = np.random.permutation(len(self.val_batch_idx))
        self.pack = bool(config.preprocessing.get("pack_sequences", False))
        if self.pack:
            self._setup_packing(idx)

    def _setup_packing(self, order: List[int]) -> None:
        row_len = self.config.preprocessing["max_context_size"] + 1
        bos = self.tokenizer.BOS_TOKEN
        self.packed_tokens: List[List[int]] = []
        for i in order:
            t = self.tokenizer.tokenize_doc(self.train_docs[i])
            if bos in t[1:]:
                raise ValueError(f"document {i} ({self.train_docs[i][:40]!r}...) contains the BOS token id {bos} "
                                 "after its first position: packed rows find document starts at BOS tokens")
            self.packed_tokens.append(t[:row_len])
        self.packed_rows = pack_first_fit([len(t) for t in self.packed_tokens], row_len)
        bs = self.batch_size
        self.packed_batch_idx = [list(range(i, min(i + bs, len(self.packed_rows))))
                                 for i in range(0, len(self.packed_rows), bs)]
        self.packed_indices = np.random.permutation(len(self.packed_batch_idx))

    @property
    def num_train_batches(self) -> int:
        """Training batches per epoch (packed batches when packing is on)."""
        return len(self.packed_batch_idx) if self.pack else len(self.train_batch_idx)

    def _load_file(self, file_path: str, docs: List[Any]) -> None:
        chunk = self.config.preprocessing["max_context_size"]
        stride = chunk - self.config.preprocessing.get("chunk_overlap", 0)
        with open(file_path, "r") as f:
            for line in f:
                rec = json.loads(line)
                if self.prefix_lm and "text" not in rec and "prompt" in rec and "completion" in rec:
                    docs.append((str(rec["prompt"]), str(rec["completion"])))  # a pair is never chunked
                    continue
                if "text" not in rec:
                    keys = '"text", or "prompt" and "completion"' if self.prefix_lm else '"text"'
                    raise ValueError(f"{file_path}: a line has keys {sorted(rec)}; expected {keys}")
                text = rec["text"]
                for i in range(0, len(text), stride):
                    docs.append(text[i:i + chunk])

    def generate_batch(self, step: int) -> torch.Tensor:
        if self.pack:
            return self._packed_batch(step)
        # data-parallel ranks walk disjoint batches of the shared shuffled order
        j = (step * self.world + self.rank) % len(self.train_indices)
        return self._create_batch([self.train_docs[i] for i in self.train_batch_idx[self.train_indices[j]]],
                                  train_split_seed(step, self.rank))

    def _packed_batch(self, step: int) -> torch.Tensor:
        """[batch_size, max_context_size + 1] rows of whole documents; the last batch of an epoch may hold rows
        of PAD only (no loss, no tokens)."""
        j = (step * self.world + self.rank) % len(self.packed_indices)
        row_len = self.config.preprocessing["max_context_size"] + 1
        out = torch.full((self.batch_size, row_len), self.tokenizer.PAD_TOKEN, dtype=torch.int64)
        for r, row in enumerate(self.packed_batch_idx[self.packed_indices[j]]):
            toks = [t for d in self.packed_rows[row] for t in self.packed_tokens[d]]
            out[r, :len(toks)] = torch.tensor(toks, dtype=torch.int64)
        return out

    def generate_validation_batch(self, batch_idx: int) -> torch.Tensor:
        if not self.val_batch_idx:
            raise ValueError("No validation data available")
        ids = self.val_batch_idx[self.val_indices[self.val_ptr % len(self.val_indices)]]
        self.val_ptr += 1
        return self._create_batch([self.val_docs[i] for i in ids], val_split_seed(batch_idx))

    def _tokenize_pair(self, doc) -> Tuple[List[int], int]:
        """A prompt / completion pair -> ([BOS] + prompt + completion + [EOS], its prefix 1 + len(prompt))."""
        t = self.tokenizer
        p = t.tokenize(doc[0])
        return [t.BOS_TOKEN] + p + t.tokenize(doc[1]) + [t.EOS_TOKEN], 1 + len(p)

    def _create_batch(self, docs: List[Any], split_seed: int = 0) -> torch.Tensor:
        pairs = [self._tokenize_pair(d) if isinstance(d, tuple) else (self.tokenizer.tokenize_doc(d), None)
                 for d in docs]
        batch = [x for x, _ in pairs]
        max_len = min(max(len(x) for x in batch), self.config.preprocessing.get("max_context_size", 2048))
        rows = [x[:max_len] + [self.tokenizer.PAD_TOKEN] * (max_len - len(x[:max_len])) for x in batch]
        out = torch.tensor(rows, dtype=torch.int64)
        if not self.prefix_lm:
            return out
        # inputs are row[:-1]: row b has min(len, max_len - 1) non-PAD inputs
        n_in = [min(len(x), max_len - 1) for x in batch]
        drawn = split_points(n_in, split_seed)
        P = torch.tensor([min(p, max_len) if p is not None else int(drawn[b]) for b, (_, p) in enumerate(pairs)],
                         dtype=torch.int64)
        return torch.cat([P[:, None], out], dim=1)

    @property
    def has_validation_data(self) -> bool:
        return self.config.validation_file is not None and len(self.val_docs) > 0

    @property
    def num_validation_batches(self) -> int:
        return len(self.val_batch_idx)


# ------------------------------------------------------------------------------------------------
# optimizer factory (core/training.py:770-896)
# ------------------------------------------------------------------------------------------------
class OptimizationManager:
    def __init__(self, config: TrainingConfig, num_training_steps: int):
        self.config = config
        self.num_training_steps = num_training_steps

    def create_scheduler(self) -> Callable[[int], float]:
        cfg = self.config.scheduler
        lr = self.config.hyperparameters["learning_rate"]
        if cfg["type"] == "cosine_with_warmup":
            warm = linear_schedule(0, lr, steps=cfg["warmup_steps"])
            cos = cosine_decay(lr, self.num_training_steps, lr * cfg["min_lr_ratio"])
            return join_schedules([warm, cos], [cfg["warmup_steps"]])
        if cfg["type"] == "cosine":
            return cosine_decay(lr, self.num_training_steps, lr * cfg["min_lr_ratio"])
        if cfg["type"] == "linear":
            return linear_schedule(lr, 0, steps=self.num_training_steps)
        raise ValueError(f"Unsupported scheduler type: {cfg['type']}")

    def create_optimizer(self, schedule, cfg: Optional[Dict[str, Any]] = None):
        cfg = self.config.optimization if cfg is None else cfg
        hp = self.config.hyperparameters
        kwargs: Dict[str, Any] = {"learning_rate": schedule}
        if "betas" in cfg:
            kwargs["betas"] = tuple(cfg["betas"])
        if "eps" in cfg:
            kwargs["eps"] = cfg["eps"]
        # the reference only forwards weight_decay when optimization.weight_decay exists (SURVEY D14);
        # mlx AdamW's default 0.01 otherwise.  Forward the hyperparameter explicitly when present.
        if "weight_decay" in cfg or "weight_decay" in hp:
            kwargs["weight_decay"] = hp.get("weight_decay", cfg.get("weight_decay", 0.01))
        name = cfg["optimizer"]
        if name in ("adamw", "adamw_enhanced"):
            return AdamW(bias_correction=(name == "adamw_enhanced"), **kwargs)
        if name == "adam":
            kwargs.pop("weight_decay", None)
            return AdamW(weight_decay=0.0, **kwargs)
        if name == "muon":
            # `optimizer: muon` binds to the Newton-Schulz Muon of optimizers/muon.py (SURVEY D3)
            return Muon(learning_rate=schedule, momentum=cfg.get("momentum", 0.95),
                        nesterov=cfg.get("nesterov", True), ns_steps=cfg.get("ns_steps", 5),
                        betas=kwargs.get("betas"), eps=kwargs.get("eps"),
                        weight_decay=kwargs.get("weight_decay"))
        if name == "shampoo":
            params = ShampooParams(
                beta1=cfg.get("beta1", 0.9), beta2=cfg.get("beta2", 0.95), epsilon=cfg.get("epsilon", 1e-8),
                weight_decay=kwargs.get("weight_decay", 0.0) if "weight_decay" in cfg else 0.0,
                update_period=cfg.get("update_period", 100),
                start_preconditioning_step=cfg.get("start_preconditioning_step", 1000),
                preconditioner_epsilon=cfg.get("preconditioner_epsilon", 1e-6),
                exponent_override=cfg.get("exponent_override", 0.75), use_bias_correction=True,
                grafting_optimizer=cfg.get("grafting_optimizer", "adam"), use_decoupled_weight_decay=True,
                inverse_root=cfg.get("inverse_root", "reference"))
            return Shampoo(learning_rate=schedule, params=params)
        # the enhanced optimizers' extras (core/training.py:800-803): forwarded where the optimizer has them
        extras = {k: cfg[k] for k in ("grad_clip_norm", "ema_momentum") if k in cfg}
        if name == "lion":
            kwargs.pop("eps", None)
            return Lion(lion_variant=cfg.get("lion_variant", "reference"), **kwargs, **extras)
        if name == "sgd_enhanced":
            kwargs.pop("betas", None)
            kwargs.pop("eps", None)
            return SGDEnhanced(momentum=cfg.get("momentum", 0.9), nesterov=cfg.get("nesterov", False),
                               **kwargs, **extras)
        if name == "sgd":
            # mlx.optimizers.SGD given the learning rate only (:891-894); the reference would raise TypeError on
            # the extras, and dropping them silently would train without them
            if extras:
                raise ValueError(f"optimizer 'sgd' does not take {sorted(extras)}; use 'sgd_enhanced'")
            return SGD(learning_rate=schedule)
        if name == "hybrid":
            m_cfg = {k: v for k, v in cfg.items() if k not in ("optimizer", "non_matrix_optimizer")}
            n_cfg = {k: v for k, v in cfg.items() if k not in ("optimizer", "matrix_optimizer")}
            m_cfg["optimizer"] = cfg.get("matrix_optimizer", "muon")
            n_cfg["optimizer"] = cfg.get("non_matrix_optimizer", "adamw")
            return HybridOptimizer(learning_rate=schedule, matrix_optimizer=self.create_optimizer(schedule, m_cfg),
                                   non_matrix_optimizer=self.create_optimizer(schedule, n_cfg))
        raise ValueError(f"Unsupported optimizer: {name}")


# ------------------------------------------------------------------------------------------------
# trainer
# ------------------------------------------------------------------------------------------------
def _precision_dtype(system: SystemConfig) -> torch.dtype:
    if not system.mixed_precision:
        return torch.float32
    # the tensor-core kernels take bf16 operands; `precision: float16` is served in bf16 (same
    # width, wider exponent) -- documented in DESIGN.md
    return torch.bfloat16


class BatchPrefetcher:
    """Background producer of token batches (SURVEY 8f row f4; the reference builds every batch on the
    training thread, core/training.py:519-543,1651).  A daemon thread runs `make_batch(step)` for the
    coming steps into a rotating pool of PINNED host buffers; `get(step)` hands the training loop the
    buffer for exactly that step, so tokenisation / padding / the pinned staging copy overlap the GPU
    step and the loop's own work is one asynchronous H2D copy.  A buffer is only rewritten after the
    copy that read it has completed (`release(step, event)`)."""

    def __init__(self, make_batch: Callable[[int], torch.Tensor], start: int, stop: int, depth: int = 2,
                 pin: bool = True):
        import queue
        import threading
        self._make, self._stop_step, self._depth = make_batch, stop, max(1, depth)
        self._pin = pin and torch.cuda.is_available()
        self._q: "queue.Queue" = queue.Queue(maxsize=self._depth)
        self._pool: List[Optional[torch.Tensor]] = [None] * (self._depth + 2)
        self._events: List[Any] = [None] * (self._depth + 2)
        self._halt = threading.Event()
        self._next = start
        self._thread = threading.Thread(target=self._run, args=(start,), daemon=True, name="batch-prefetch")
        self._thread.start()

    def _run(self, start: int) -> None:
        try:
            for step in range(start, self._stop_step):
                if self._halt.is_set():
                    return
                batch = self._make(step)
                slot = (step - start) % len(self._pool)
                ev = self._events[slot]
                if ev is not None:
                    ev.synchronize()          # the H2D copy that last read this buffer has finished
                    self._events[slot] = None
                buf = self._pool[slot]
                if buf is None or buf.shape != batch.shape or buf.dtype != batch.dtype:
                    buf = torch.empty(batch.shape, dtype=batch.dtype, pin_memory=self._pin)
                    self._pool[slot] = buf
                buf.copy_(batch)
                while not self._halt.is_set():
                    try:
                        self._q.put((step, slot, buf), timeout=0.1)
                        break
                    except Exception:
                        continue
        except BaseException as e:  # surfaced to the training thread by get()
            self._q.put((None, None, e))

    def get(self, step: int):
        """-> (pinned batch for `step`, slot token to pass to release())."""
        if step != self._next:
            raise RuntimeError(f"prefetcher is sequential: expected step {self._next}, got {step}")
        got_step, slot, buf = self._q.get()
        if got_step is None:
            raise buf
        assert got_step == step
        self._next += 1
        return buf, slot

    def release(self, slot: int, event=None) -> None:
        """Call once the H2D copy of the buffer has been enqueued; `event` (recorded after it) guards reuse."""
        self._events[slot] = event

    def close(self) -> None:
        self._halt.set()
        try:
            while True:
                self._q.get_nowait()
        except Exception:
            pass
        self._thread.join(timeout=5)


class EarlyStoppingMonitor:
    """core/training.py:621-668: stop after `patience` validations without a `min_delta` improvement."""

    def __init__(self, config: Optional[Dict[str, Any]]):
        config = config or {}
        self.enabled = config.get("enabled", False)
        self.patience = config.get("patience", 3)
        self.min_delta = config.get("min_delta", 0.001)
        self.metric = config.get("metric", "val_loss")
        self.mode = config.get("mode", "min")
        self.best_value = float("inf") if self.mode == "min" else float("-inf")
        self.counter = 0

    def update(self, metrics: Dict[str, float]) -> bool:
        if not self.enabled or self.metric not in metrics:
            return False
        cur = metrics[self.metric]
        improved = (self.best_value - cur > self.min_delta) if self.mode == "min" else (cur - self.best_value > self.min_delta)
        if improved:
            self.best_value, self.counter = cur, 0
            return False
        self.counter += 1
        return self.counter >= self.patience


class Trainer:
    def __init__(self, config, for_training: bool = True, synthetic: Optional[bool] = None,
                 run_root: str = "runs", quiet: bool = False, init_params: Optional[Dict[str, torch.Tensor]] = None):
        self.config = config if isinstance(config, Config) else Config.from_yaml(config)
        self.quiet = quiet
        self.synthetic = (self.config.data.input_file.startswith("synthetic")
                          if synthetic is None else synthetic)
        self.rank, self.world, self.local_rank = dp.env_rank_world()
        self.run_dir = Path(run_root) / self.config.name
        self.checkpoint_dir = self.run_dir / "checkpoints"
        self.log_file = self.run_dir / "log.txt"
        if self.rank == 0:
            self.checkpoint_dir.mkdir(parents=True, exist_ok=True)
        self.logger = logging.getLogger(f"trainer.{self.config.name}")
        self.logger.setLevel(logging.WARNING if quiet else logging.INFO)
        if not self.logger.handlers and not quiet:
            self.logger.addHandler(logging.StreamHandler(sys.stdout))
        self.total_tokens = 0
        self.validation_losses: List[Tuple[int, float]] = []
        self.setup_system()
        self.tokenizer = TokenizerManager(self.config.data, self.run_dir, synthetic=self.synthetic)
        self.setup_model(init_params)
        if for_training:
            self.setup_data()
            self.setup_training()

    # -- setup ---------------------------------------------------------------------------------
    def setup_system(self) -> None:
        seed = self.config.system.seed
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        ops.require_device()  # the hot path has no CPU fallback (system.device: cpu is the oracle's job)
        torch.cuda.set_device(self.local_rank)
        self.device = torch.device("cuda", self.local_rank)
        self.distributed = bool(self.config.system.distributed) and self.world > 1
        if self.config.system.distributed and self.world == 1:
            self.logger.info("system.distributed is set but WORLD_SIZE=1: running single-GPU "
                             "(launch with torchrun --nproc-per-node N for data parallelism)")
        if self.distributed:
            dp.init_process_group(self.device)

    def setup_model(self, init_params: Optional[Dict[str, torch.Tensor]] = None) -> None:
        m = self.config.model
        if m.architecture not in ("llama", "llama_standard"):
            raise ImportError(f"Model architecture '{m.architecture}' not found")
        args = ModelArgs(
            model_type=m.architecture, hidden_size=m.dimensions["hidden_size"],
            num_hidden_layers=m.dimensions.get("num_layers", 8), intermediate_size=m.dimensions["intermediate_size"],
            num_attention_heads=m.attention["num_heads"], rms_norm_eps=m.normalization["rms_norm_eps"],
            vocab_size=self.tokenizer.VOCAB_SIZE,
            head_dim=m.attention.get("head_dim") or m.dimensions["hidden_size"] // m.attention["num_heads"],
            max_position_embeddings=m.attention["max_position_embeddings"],
            num_key_value_heads=m.attention.get("num_kv_heads") or m.attention["num_heads"],
            attention_bias=m.misc["attention_bias"], mlp_bias=m.misc["mlp_bias"], rope_theta=m.rope["theta"],
            rope_traditional=m.rope["traditional"], rope_scaling=m.rope["scaling"],
            tie_word_embeddings=m.misc["tie_word_embeddings"], logit_scale=m.misc.get("logit_scale"),
            use_flash_attention=m.attention.get("use_flash_attention", True),
            use_flex_attention=m.attention.get("use_flex_attention", False),
            flash_block_size=m.attention.get("flash_block_size", 128),
            apply_rope=bool(m.rope.get("enabled", m.architecture == "llama_standard")) or m.misc.get("variant") == "mlx_lm",
            sliding_window=m.attention.get("sliding_window"), alibi=bool(m.attention.get("alibi")),
            prefix_lm=bool(m.attention.get("prefix_lm")), variant=m.misc.get("variant"),
            attention_dropout=float(m.attention.get("dropout") or 0.0),
            num_local_experts=m.misc.get("num_local_experts") or 0,
            num_experts_per_tok=m.misc.get("num_experts_per_tok") or 0,
            router_aux_loss_coef=float(m.misc.get("router_aux_loss_coef", 0.001)))
        self.model_args = args
        model = Model(args)
        init_model_(model, args, self.config.system.seed)
        if init_params is not None:
            model.load_parameters(init_params)
        model.to(self.device)
        self.model = model
        self.store = ParamStore(model, _precision_dtype(self.config.system), self.device)
        if self.distributed:
            dp.broadcast_(self.store.master)
            self.store.refresh_shadow()
        n = sum(p.numel() for p in model.parameters()) / 1e6
        self.logger.info(f"Model has {n:.2f}M parameters (vocab {args.vocab_size})")

    def setup_data(self) -> None:
        hp = self.config.training.hyperparameters
        bs = hp["batch_size"]
        seq = self.config.data.preprocessing["max_context_size"]
        if self.synthetic:
            kind = self.config.data.input_file.split(":", 1)[1] if ":" in self.config.data.input_file else "uniform"
            self.data_manager = SyntheticData(self.config.data.tokenizer["normal_vocab_size"], bs, seq, self.rank,
                                              num_batches=hp.get("iters", 1000), kind=kind,
                                              prefix_lm=self.model_args.prefix_lm)
        else:
            self.data_manager = DataManager(self.config.data, self.tokenizer, bs, self.rank, self.world,
                                            prefix_lm=self.model_args.prefix_lm)

    def setup_training(self) -> None:
        hp = self.config.training.hyperparameters
        if getattr(self.data_manager, "pack", False):
            steps_per_epoch = max(self.data_manager.num_train_batches, 1)
        else:
            steps_per_epoch = max(len(self.data_manager.train_docs) // hp["batch_size"], 1)
        self.steps_per_epoch = steps_per_epoch
        self.total_steps = (steps_per_epoch * self.config.training.epochs if self.config.training.epochs is not None
                            else hp.get("iters", steps_per_epoch))
        om = OptimizationManager(self.config.training, self.total_steps)
        self.lr_schedule = om.create_scheduler()
        self.optimizer = om.create_optimizer(self.lr_schedule)
        self.grad_accum_steps = hp.get("gradient_accumulation_steps", 1)
        self.clip_value = float(hp["gradient_clip"]) if "gradient_clip" in hp else 0.0
        self.use_acc = self.grad_accum_steps > 1 or self.clip_value > 0.0
        if self.use_acc:
            self.store.ensure_acc()
        self.optimizer.use_accumulated = self.use_acc
        self.optimizer.grad_scale = 1.0 / self.world if self.distributed else 1.0
        if hasattr(self.optimizer, "shard_ns"):
            # owner-computes Newton-Schulz across the data-parallel ranks (SURVEY 8e fused mode)
            self.optimizer.shard_ns = bool(self.distributed and self.world > 1 and
                                           os.environ.get("B200_SHARD_NS", "1") != "0")
        self.validation_steps = self.config.logging.steps.get("validation_interval", 0)
        self.early_stopping = EarlyStoppingMonitor(self.config.training.early_stopping)
        self._pin = None

    # -- loss --------------------------------------------------------------------------------------
    def compute_loss(self, model, inputs: torch.Tensor, targets: torch.Tensor, packed: bool = False,
                     aux: bool = True, prefix: Optional[torch.Tensor] = None, dropout_seed: Optional[int] = None):
        """Masked token-mean cross-entropy.  packed: the rows hold several documents (DataManager with
        pack_sequences); the model then attends within documents (position_ids from the BOS tokens), and the one
        target per document boundary that an unpacked row never has -- a document's last token predicting the
        next document's BOS -- becomes PAD, so the loss terms and ntoks are those of the documents run alone.
        prefix (int [B] on the device): prefix-LM rows; the model attends with PrefixCausalMask and the targets a
        prefix position can see become PAD (prefix_targets).  dropout_seed: the attention-dropout base of this
        micro-step (used only when the model drops: attention dropout on, training mode, grad enabled)."""
        max_ctx = self.config.model.attention.get("max_position_embeddings", 2048)
        if inputs.shape[1] > max_ctx:
            inputs, targets = inputs[:, :max_ctx], targets[:, :max_ctx]
        position_ids = None
        kw = {} if dropout_seed is None else {"dropout_seed": dropout_seed}
        if prefix is not None:
            targets = prefix_targets(targets, prefix, self.tokenizer.PAD_TOKEN)
            kw["prefix_lens"] = prefix.to(torch.int32)
        if packed:
            position_ids = document_positions(inputs, self.tokenizer.BOS_TOKEN)
            targets = targets.masked_fill(targets == self.tokenizer.BOS_TOKEN, self.tokenizer.PAD_TOKEN)
        pad_mask = targets != self.tokenizer.PAD_TOKEN
        ntoks = pad_mask.sum()
        # prefix-LM rows can keep no target (a prompt that fills the row, or a split point at the row's end), so a
        # micro-batch may have none: its loss is then 0 with no gradient, and ntoks reports the true count 0
        denom = ntoks if prefix is None else ntoks.clamp_min(1)
        # MoE models: the load-balancing loss counts the non-PAD inputs; it is kept in self.last_aux_loss for
        # micro_step, and skipped entirely when its coefficient is 0 or aux is off (validation reports CE only)
        args = getattr(self, "model_args", None)
        self.last_aux_loss = None
        moe_kw = {}
        if aux and args is not None and args.num_local_experts and args.router_aux_loss_coef > 0:
            moe_kw = {"token_mask": inputs != self.tokenizer.PAD_TOKEN}
        if not hasattr(model, "padded_logits"):
            logits2d, V = None, None
        elif position_ids is None:
            logits2d, V = model.padded_logits(inputs, **moe_kw, **kw)
        else:
            logits2d, V = model.padded_logits(inputs, position_ids, **moe_kw, **kw)
        if moe_kw and logits2d is not None:
            self.last_aux_loss = model.moe_aux_loss()
        if logits2d is not None:
            # fused path: fp32 log-sum-exp over bf16 logits, pad mask applied per row, no fp32 [B,S,V] copy
            rows = ops.cross_entropy_rows(logits2d, targets.reshape(-1).contiguous(), V, self.tokenizer.PAD_TOKEN)
            return rows.sum() / denom, ntoks
        logits = (model(inputs, **moe_kw, **kw) if position_ids is None
                  else model(inputs, position_ids, **moe_kw, **kw)).float()
        if moe_kw:
            self.last_aux_loss = model.moe_aux_loss()
        ce = torch.nn.functional.cross_entropy(logits.view(-1, logits.shape[-1]), targets.reshape(-1),
                                               reduction="none").view(targets.shape)
        return (ce * pad_mask).sum() / denom, ntoks

    def _to_device(self, batch: torch.Tensor) -> torch.Tensor:
        """Per-step host->device copy of the token batch from pinned memory.  The CPU can run a whole step
        ahead of the GPU, so a staging buffer is only rewritten after the asynchronous copy that last read it
        has completed (event recorded right after that copy): two rotating buffers, the same guard as
        BatchPrefetcher.release."""
        if self._pin is None:
            self._pin = [[None, None], [None, None]]   # [buffer, event of the last H2D copy that read it]
            self._pin_next = 0
        slot = self._pin[self._pin_next]
        self._pin_next ^= 1
        if slot[1] is not None:
            slot[1].synchronize()
        if slot[0] is None or slot[0].shape != batch.shape or slot[0].dtype != batch.dtype:
            slot[0] = torch.empty(batch.shape, dtype=batch.dtype, pin_memory=True)
        slot[0].copy_(batch)
        dev_batch = slot[0].to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        slot[1] = ev
        return dev_batch

    # -- one micro-step + (maybe) update; the unit bench.py times ----------------------------------
    def train_step(self, step: int, batch: Optional[torch.Tensor] = None):
        pf = getattr(self, "_prefetcher", None)
        if batch is None and pf is not None:
            pinned, slot = pf.get(step)       # built and staged by the background thread
            dev_batch = pinned.to(self.device, non_blocking=True)
            ev = None
            if self.device.type == "cuda":
                ev = torch.cuda.Event()
                ev.record()
            pf.release(slot, ev)
        else:
            if batch is None:
                batch = self.data_manager.generate_batch(step)
            dev_batch = self._to_device(batch)
        return self.micro_step(step, dev_batch)

    def micro_step(self, step: int, dev_batch: torch.Tensor):
        """Forward + backward of one micro-batch already resident on the device, gradient clamp / 1/k
        accumulation (core/training.py:1664-1696), and -- on the k-th micro-step -- the data-parallel
        exchange and the optimizer update.  Returns (loss, ntoks, did_update)."""
        prefix = None
        if self.model_args.prefix_lm:  # column 0 holds each row's prefix length
            prefix, dev_batch = dev_batch[:, 0], dev_batch[:, 1:]
        # attention dropout's per-micro-step base: a function of (system.seed, rank, step) only, so a resumed run
        # draws the masks of the uninterrupted one and the ranks draw different masks
        seed = None
        if self.model_args.attention_dropout > 0:
            seed = ops.dropout_seed(self.config.system.seed, self.rank, step)
        loss, ntoks = self.compute_loss(self.model, dev_batch[:, :-1], dev_batch[:, 1:],
                                        packed=getattr(self.data_manager, "pack", False), prefix=prefix,
                                        dropout_seed=seed)
        aux = getattr(self, "last_aux_loss", None)
        if aux is None:
            loss.backward()
        else:   # MoE: the training loss is CE + c * aux; `loss` stays the CE that is logged
            (loss + self.model_args.router_aux_loss_coef * aux).backward()
            self.step_aux_loss = aux.detach()
        k = self.grad_accum_steps
        store = self.store
        if self.use_acc:
            first = (self._accum_step == 0)
            ops.clip_accum(store.grad, store.acc, self.clip_value, 1.0 / k, init=first)
            store.zero_grad()
        self._accum_step += 1
        self._accum_tokens = self._accum_tokens + ntoks
        did_update = False
        if self._accum_step == k or step == self.total_steps - 1:
            if self.distributed:
                dp.all_reduce_sum_(store.acc if self.use_acc else store.grad)
            self.optimizer.update(self.model)
            if not self.use_acc:
                store.zero_grad()
            self._accum_step = 0
            did_update = True
        return loss.detach(), ntoks.detach(), did_update

    def validate(self) -> Optional[float]:
        if not self.data_manager.has_validation_data:
            return None
        tot_loss = torch.zeros((), device=self.device)
        tot_tok = torch.zeros((), device=self.device)
        with torch.no_grad():
            for i in range(min(self.data_manager.num_validation_batches, 50)):
                b = self._to_device(self.data_manager.generate_validation_batch(i))
                prefix = None
                if self.model_args.prefix_lm:
                    prefix, b = b[:, 0], b[:, 1:]
                loss, ntoks = self.compute_loss(self.model, b[:, :-1], b[:, 1:], aux=False, prefix=prefix)
                tot_loss += loss * ntoks
                tot_tok += ntoks
        if self.distributed:
            v = torch.stack([tot_loss, tot_tok])
            dp.all_reduce_sum_(v)
            tot_loss, tot_tok = v[0], v[1]
        if self.model_args.prefix_lm and float(tot_tok.item()) == 0:
            raise ValueError("prefix_lm: no validation target is left after the prefix masking (every prompt fills "
                             "its row); shorten the prompts or raise data.preprocessing.max_context_size")
        return float((tot_loss / tot_tok).item())

    def save_config(self) -> Path:
        """Writes the effective config (CLI overrides applied) to <run_dir>/config.yaml, where the reference writes it
        (core/training.py:1173-1176) and where `python -m core.generation --run` finds it.  A run forced onto
        synthetic tokens records `data.input_file: synthetic` (a `synthetic:<kind>` value is kept), so that
        Trainer(cfg, for_training=False) rebuilds the same vocabulary."""
        d = asdict(self.config)
        if self.synthetic and not str(d["data"]["input_file"]).startswith("synthetic"):
            d["data"]["input_file"] = "synthetic"
        path = self.run_dir / "config.yaml"
        path.write_text(yaml.safe_dump(d, sort_keys=False))
        return path

    # -- main loop (core/training.py:1637-1768) ---------------------------------------------------
    def train(self) -> Dict[str, Any]:
        if self.rank == 0:
            self.save_config()
        start_step = 0
        if self.config.resume and self.config.resume.checkpoint:
            start_step = self.load_checkpoint(self.config.resume.checkpoint, self.config.resume.reset_optimizer)
            if self.config.resume.reset_training_state:
                start_step, self.total_tokens, self.validation_losses = 0, 0, []
        self._accum_step, self._accum_tokens = 0, 0
        total_tokens = torch.zeros((), dtype=torch.int64, device=self.device) + int(self.total_tokens)
        log_every = self.config.logging.steps["logging_interval"]
        ckpt_every = self.config.logging.steps.get("checkpoint_interval", 0)
        logf = open(self.log_file, "a" if start_step > 0 else "w") if self.rank == 0 else None
        if logf and start_step == 0:
            logf.write(f"Training started at {datetime.now()}\nTotal steps: {self.total_steps}\n")
            if self.grad_accum_steps > 1:
                logf.write(f"Using gradient accumulation with {self.grad_accum_steps} steps\n")
            logf.write("=" * 50 + "\n\n")
        start_time = time.time()
        val_loss = None
        last: Dict[str, Any] = {}
        if os.environ.get("B200_PREFETCH", "1") != "0":
            self._prefetcher = BatchPrefetcher(self.data_manager.generate_batch, start_step, self.total_steps)
        try:
            last = self._train_loop(start_step, total_tokens, log_every, ckpt_every, logf, start_time, val_loss, last)
        finally:
            if getattr(self, "_prefetcher", None) is not None:
                self._prefetcher.close()
                self._prefetcher = None
        return last

    def _train_loop(self, start_step, total_tokens, log_every, ckpt_every, logf, start_time, val_loss, last):
        pending: Dict[str, Any] = {}   # metrics_to_log of the reference: kept until the next logging step
        for step in range(start_step, self.total_steps):
            loss, ntoks, did_update = self.train_step(step)
            if did_update:
                total_tokens += self._accum_tokens
                self._accum_tokens = 0
            if self.validation_steps > 0 and self.data_manager.has_validation_data and (step + 1) % self.validation_steps == 0:
                val_loss = self.validate()
                self.validation_losses.append((step + 1, val_loss))
                pending.update(val_loss=val_loss, val_ppl=float(np.exp(val_loss)))
                if self.early_stopping.update({"val_loss": val_loss}):   # core/training.py:1726
                    self.logger.info("Early stopping triggered, ending training")
                    if logf:
                        logf.write(f"Step {step}: val_loss={val_loss} | early_stopping=1\n")
                    break
            metrics: Dict[str, Any] = {}
            if step % log_every == 0:
                if self.distributed:  # token-weighted loss across ranks (hybrid_distributed.py:504,519-520)
                    v = torch.stack([loss.float() * ntoks, ntoks.float()])
                    dp.all_reduce_sum_(v)
                    loss_val, ntok_val = float((v[0] / v[1]).item()), int(v[1].item())
                else:
                    loss_val, ntok_val = float(loss.item()), int(ntoks.item())
                tt = int(total_tokens.item()) * (self.world if self.distributed else 1)
                metrics = {**pending, "loss": loss_val, "ppl": float(np.exp(min(loss_val, 80.0))),
                           "lr": float(self.lr_schedule(step)), "tokens": ntok_val, "total_tokens": tt,
                           "tokens_per_sec": float(tt / max(time.time() - start_time, 1e-9))}
                if getattr(self, "step_aux_loss", None) is not None:
                    metrics["aux_loss"] = float(self.step_aux_loss.item())
                pending = {}
                last = metrics
                if logf:
                    line = f"Step {step}: " + " | ".join(f"{k}={v}" for k, v in metrics.items())
                    logf.write(line + "\n")
                    logf.flush()
                    self.logger.info(line)
            if ckpt_every and (step + 1) % ckpt_every == 0 and self.rank == 0:
                self.total_tokens = int(total_tokens.item())
                self.save_checkpoint(step + 1, val_loss)
        self.total_tokens = int(total_tokens.item())
        if self.rank == 0:
            self.save_checkpoint("final", val_loss)
        if logf:
            logf.write("\n" + "=" * 50 + f"\nTraining completed at {datetime.now()}\n")
            logf.close()
        return last

    # -- checkpoints (core/training.py:1347-1394,1437-1478) ---------------------------------------
    def save_checkpoint(self, step, val_loss: Optional[float] = None) -> None:
        from safetensors.torch import save_file
        torch.cuda.synchronize()
        weights = {n: t.detach().cpu().contiguous() for n, t in self.store.named_master().items()}
        save_file(weights, str(self.checkpoint_dir / f"step_{step}_model.safetensors"))
        opt_state = {n: t.detach().cpu().contiguous().clone() for n, t in self.optimizer.state_dict().items()}
        opt_state["count"] = torch.tensor([self.optimizer.count], dtype=torch.int64)
        save_file(opt_state, str(self.checkpoint_dir / f"step_{step}_optimizer.safetensors"))
        state = {"step": step if isinstance(step, int) else self.total_steps, "val_ptr": self.data_manager.val_ptr,
                 "total_tokens": int(self.total_tokens), "validation_losses": self.validation_losses}
        (self.checkpoint_dir / f"step_{step}_state.json").write_text(json.dumps(state))
        meta_path = self.run_dir / "metadata.json"
        meta = json.loads(meta_path.read_text()) if meta_path.exists() else {"name": self.config.name, "checkpoints": []}
        info = {"step": step, "timestamp": datetime.now().isoformat(),
                "paths": {"model": f"checkpoints/step_{step}_model.safetensors",
                          "optimizer": f"checkpoints/step_{step}_optimizer.safetensors",
                          "state": f"checkpoints/step_{step}_state.json"}}
        if val_loss is not None:
            info["validation_loss"] = val_loss
        meta.setdefault("checkpoints", []).append(info)
        meta_path.write_text(json.dumps(meta, indent=2))

    def load_checkpoint(self, checkpoint_path: str, reset_optimizer: bool = False) -> int:
        from safetensors.torch import load_file
        weights = load_file(f"{checkpoint_path}_model.safetensors")
        with torch.no_grad():
            for n, t in weights.items():
                if n in self.store.index:  # non-strict, like models/llama.py:440-475
                    self.store.view(self.store.master, n).copy_(t.to(self.device))
            self.store.refresh_shadow()
        if not reset_optimizer and os.path.exists(f"{checkpoint_path}_optimizer.safetensors"):
            self.optimizer.init(self.model)   # allocate state so the saved tensors have somewhere to go
            st = load_file(f"{checkpoint_path}_optimizer.safetensors")
            own = self.optimizer.state_dict()
            with torch.no_grad():
                for n, t in st.items():
                    if n == "count":
                        self.optimizer.count = int(t.item())
                    elif n in own and own[n].is_cuda:
                        own[n].copy_(t.to(self.device))
            if hasattr(self.optimizer, "load_extra_state"):   # e.g. the hybrid optimizer's AdamW step counter
                self.optimizer.load_extra_state(st)
            if hasattr(self.optimizer, "after_load"):         # e.g. Shampoo: rebuild bf16 preconditioner operands
                self.optimizer.after_load()
        state = json.loads(Path(f"{checkpoint_path}_state.json").read_text())
        self.total_tokens = state.get("total_tokens", 0)
        self.validation_losses = [tuple(x) for x in state.get("validation_losses", [])]
        if getattr(self, "data_manager", None) is not None:
            self.data_manager.val_ptr = state.get("val_ptr", 0)   # core/training.py:1469
        return int(state["step"])


def init_model_(model: Model, args: ModelArgs, seed: int) -> None:
    """Harness-owned init shared with the oracle (oracle.reference_math.init_params draws the same
    values in the same parameter order): linears U(+-1/sqrt(in)), embedding N(0, 1/hidden), gains 1."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() == 1:
                p.fill_(1.0)
            elif name == "embed_tokens.weight":
                p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float32) * args.hidden_size ** -0.5)
            else:
                bound = 1.0 / math.sqrt(p.shape[-1])   # [E, out, in] experts: each slice as its nn.Linear
                p.copy_((torch.rand(p.shape, generator=g, dtype=torch.float32) * 2 - 1) * bound)


# ------------------------------------------------------------------------------------------------
# CLI (core/training.py:1907-2013) and train() wrapper (:2039-2082)
# ------------------------------------------------------------------------------------------------
def train(config, **trainer_kwargs) -> Dict[str, Any]:
    """Accepts a YAML path or a config dict, like the reference's train(config)."""
    cfg = Config.from_dict(config) if isinstance(config, dict) else Config.from_yaml(config)
    trainer = Trainer(cfg, **trainer_kwargs)
    try:
        return trainer.train()
    finally:
        if trainer.distributed:
            dp.destroy()


def main(argv: Optional[List[str]] = None) -> None:
    ap = argparse.ArgumentParser(description="Train a language model on the CUDA hot path")
    ap.add_argument("--config", type=str, required=True, help="Path to YAML config file")
    ap.add_argument("--mixed-precision", action="store_true")
    ap.add_argument("--precision", type=str, default=None, choices=["float16", "bfloat16"])
    ap.add_argument("--gradient-checkpointing", action="store_true")
    ap.add_argument("--find-lr", action="store_true")
    ap.add_argument("--tensorboard", action="store_true")
    ap.add_argument("--wandb", action="store_true")
    ap.add_argument("--log-interval", type=int, default=None)
    ap.add_argument("--run-id", type=str, default=None)
    ap.add_argument("--synthetic", action="store_true", help="use synthetic tokens instead of data.input_file")
    ap.add_argument("--iters", type=int, default=None, help="override training.hyperparameters.iters")
    a = ap.parse_args(argv)
    with open(a.config) as f:
        d = yaml.safe_load(f)
    if a.mixed_precision:
        d["system"]["mixed_precision"] = True
    if a.precision:
        d["system"]["precision"] = a.precision
    if a.log_interval:
        d["logging"]["steps"]["logging_interval"] = a.log_interval
    if a.run_id:
        d["name"] = f"{d['name']}-{a.run_id}"
    if a.iters:
        d["training"]["hyperparameters"]["iters"] = a.iters
    if a.gradient_checkpointing or a.find_lr or a.tensorboard or a.wandb:
        print("note: --gradient-checkpointing/--find-lr/--tensorboard/--wandb are accepted for CLI "
              "compatibility and ignored (outside the hot path)")
    train(d, synthetic=True if a.synthetic else None)


if __name__ == "__main__":
    main()
