"""Packed training batches (`data.preprocessing.pack_sequences`) on the host: placement, positions, boundary targets,
determinism and data-parallel disjointness, and the unpacked default left as it was."""
import json
import random
from pathlib import Path

import numpy as np
import pytest
import torch

from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import DocumentCausalMask
from mlx_cuda_distributed_pretraining_b200.core.training import (DataConfig, DataManager, TokenizerManager,
                                                                  document_positions, pack_first_fit)

HERE = Path(__file__).resolve().parent / "golden"
CTX = 96


def _cfg(pack=True, corpus=HERE / "tiny_corpus.jsonl", ctx=CTX):
    pre = {"max_context_size": ctx, "chunk_overlap": 16}
    if pack is not None:
        pre["pack_sequences"] = pack
    return DataConfig(input_file=str(corpus), validation_file=str(HERE / "tiny_val.jsonl"), preprocessing=pre,
                      tokenizer={"normal_vocab_size": 256,
                                 "special_tokens": {"pad": "<pad>", "bos": "<bos>", "eos": "<eos>"}})


def _dm(pack=True, seed=42, rank=0, world=1, batch_size=3, **kw):
    random.seed(seed)
    np.random.seed(seed)
    cfg = _cfg(pack, **kw)
    tok = TokenizerManager(cfg)
    return DataManager(cfg, tok, batch_size=batch_size, rank=rank, world=world), tok


def _split(row, tok):
    """Documents of one packed row (BOS-started runs) and the PAD tail length."""
    row = row.tolist()
    n_pad = 0
    while row and row[-1] == tok.PAD_TOKEN:
        row.pop()
        n_pad += 1
    if not row:  # a PAD-only row (the last batch of an epoch is filled up with them)
        return [], n_pad
    starts = [i for i, t in enumerate(row) if t == tok.BOS_TOKEN]
    assert starts and starts[0] == 0
    return [row[a:b] for a, b in zip(starts, starts[1:] + [len(row)])], n_pad


def test_pack_first_fit():
    assert pack_first_fit([5, 3, 4, 2, 6, 1], 8) == [[0, 1], [2, 3, 5], [4]]
    assert pack_first_fit([], 8) == []
    with pytest.raises(ValueError):
        pack_first_fit([9], 8)
    rng = np.random.default_rng(0)
    lens = rng.integers(1, 50, 500).tolist()
    rows = pack_first_fit(lens, 64)
    assert sorted(i for r in rows for i in r) == list(range(500))
    assert all(sum(lens[i] for i in r) <= 64 for r in rows)
    # first fit: no item fits an earlier row as it was when the item was placed
    fill = []
    where = {i: r for r, row in enumerate(rows) for i in row}
    for i, n in enumerate(lens):
        r = where[i]
        assert all(f + n > 64 for f in fill[:r])
        if r == len(fill):
            fill.append(0)
        fill[r] += n


def test_every_document_once_whole_in_full_rows():
    dm, tok = _dm()
    epoch = dm.num_train_batches
    seen = []
    for step in range(epoch):
        b = dm.generate_batch(step)
        assert b.shape == (3, CTX + 1) and b.dtype == torch.int64
        for row in b:
            docs, _ = _split(row, tok)
            seen += [tuple(d) for d in docs]
    want = sorted(tuple(tok.tokenize_doc(d)[:CTX + 1]) for d in dm.train_docs)
    assert sorted(seen) == want
    # BOS only at document starts
    for d in seen:
        assert tok.BOS_TOKEN not in d[1:]


def test_positions_are_each_documents_arange():
    dm, tok = _dm()
    b = dm.generate_batch(0)
    pos = document_positions(b, tok.BOS_TOKEN)
    assert pos.dtype == torch.int32 and pos.shape == b.shape
    for r in range(b.shape[0]):
        docs, n_pad = _split(b[r], tok)
        if not docs:
            assert torch.equal(pos[r].long(), torch.arange(b.shape[1]))
            continue
        want = torch.cat([torch.arange(len(d)) for d in docs] +
                         [torch.arange(len(docs[-1]), len(docs[-1]) + n_pad)])  # the PAD tail continues the last one
        assert torch.equal(pos[r].long(), want)
    # the mask marker's dense form: q sees k iff q - pos[q] <= k <= q
    m = DocumentCausalMask(pos[:1, :40]).dense()
    ok = m[0, 0] == 0
    for q in range(40):
        for k in range(40):
            assert bool(ok[q, k]) == (q - int(pos[0, q]) <= k <= q)


class _FakeTrainer:
    """compute_loss's host-side inputs, with a model that records what it was called with."""

    def __init__(self, tok):
        from mlx_cuda_distributed_pretraining_b200.core.training import Trainer
        self.tokenizer = tok
        self.config = type("C", (), {"model": type("M", (), {"attention": {"max_position_embeddings": 4096}})()})()
        self.compute_loss = Trainer.compute_loss.__get__(self)


class _Recorder(torch.nn.Module):
    def __init__(self, V):
        super().__init__()
        self.V, self.calls = V, []

    def forward(self, inputs, position_ids=None):
        self.calls.append((inputs, position_ids))
        return torch.zeros(*inputs.shape, self.V)


def test_boundary_targets_are_pad_and_ntoks_counts_real_targets():
    dm, tok = _dm()
    tr = _FakeTrainer(tok)
    model = _Recorder(tok.VOCAB_SIZE)
    b = dm.generate_batch(1)
    loss, ntoks = tr.compute_loss(model, b[:, :-1], b[:, 1:], packed=True)
    inputs, position_ids = model.calls[-1]
    assert torch.equal(position_ids, document_positions(b[:, :-1], tok.BOS_TOKEN))
    # host count: every target inside a document that is not PAD; a document's last token predicting the next
    # document's BOS is not a target
    real = 0
    for r in range(b.shape[0]):
        docs, _ = _split(b[r], tok)
        real += sum(len(d) - 1 for d in docs)   # each document's tokens after its BOS
    assert int(ntoks) == real
    assert abs(float(loss) - np.log(tok.VOCAB_SIZE)) < 1e-5   # uniform logits: every counted target costs ln V
    # unpacked call: no position_ids, targets untouched
    tr.compute_loss(model, b[:, :-1], b[:, 1:])
    assert model.calls[-1][1] is None


def test_deterministic_and_disjoint_across_ranks():
    a, _ = _dm()
    b, _ = _dm()
    for step in range(6):
        assert torch.equal(a.generate_batch(step), b.generate_batch(step))
    c, _ = _dm(seed=7)
    assert any(not torch.equal(a.generate_batch(s), c.generate_batch(s)) for s in range(4))
    r0, _ = _dm(rank=0, world=2, batch_size=1)
    r1, _ = _dm(rank=1, world=2, batch_size=1)
    n = r0.num_train_batches
    rows0 = [tuple(r0.generate_batch(s)[0].tolist()) for s in range(n // 2)]
    rows1 = [tuple(r1.generate_batch(s)[0].tolist()) for s in range(n // 2)]
    assert not set(rows0) & set(rows1)
    assert len(set(rows0) | set(rows1)) == 2 * (n // 2)


def test_unpacked_default_unchanged_and_validation_not_packed():
    plain, _ = _dm(pack=None)
    off, _ = _dm(pack=False)
    on, _ = _dm(pack=True)
    assert not plain.pack and not off.pack and on.pack
    for step in range(5):
        assert torch.equal(plain.generate_batch(step), off.generate_batch(step))
    assert plain.num_train_batches == len(plain.train_batch_idx)
    for i in range(3):
        assert torch.equal(plain.generate_validation_batch(i), on.generate_validation_batch(i))


def test_bos_inside_a_document_raises(tmp_path):
    corpus = tmp_path / "c.jsonl"
    corpus.write_text(json.dumps({"text": "plain text"}) + "\n" + json.dumps({"text": "x"}) + "\n")
    dm, tok = _dm(corpus=corpus)          # byte tokens never reach the BOS id
    assert dm.num_train_batches == 1

    class BosTok(TokenizerManager):
        def tokenize(self, text):
            return [self.BOS_TOKEN if c == "!" else ord(c) for c in text]

    random.seed(1)
    np.random.seed(1)
    corpus.write_text(json.dumps({"text": "fine"}) + "\n" + json.dumps({"text": "bad!doc"}) + "\n")
    cfg = _cfg(True, corpus=corpus)
    with pytest.raises(ValueError, match="bad!doc"):
        DataManager(cfg, BosTok(cfg), batch_size=1)


def test_long_document_is_cut_to_the_row(tmp_path):
    corpus = tmp_path / "c.jsonl"
    corpus.write_text(json.dumps({"text": "é" * 60}) + "\n")   # first chunk: 60 characters, 120 UTF-8 bytes
    dm, tok = _dm(corpus=corpus, ctx=64, batch_size=1)
    rows = [dm.generate_batch(s)[0] for s in range(dm.num_train_batches)]
    want = torch.tensor(tok.tokenize_doc("é" * 60)[:65])
    assert len(want) == 65 and any(torch.equal(r, want) for r in rows)
