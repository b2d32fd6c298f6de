"""Data pipeline: token chunks of ``seq_length`` as ``{input_ids, attention_mask, labels}``.

Mirrors the behaviour of the reference's ``_load_and_preprocess_data`` (tokenise ->
concatenate -> chunk to ``seq_length`` dropping the remainder -> ``labels = input_ids``;
``01-single-gpu/train_llm.py:192-245``) and its DataLoader blocks (``01:62-71``,
``02:76-85``, dp-aware sampler ``06-tensor-parallel/train_llm.py:141-147``), with three
sources because the GPU boxes have no network:

  * ``-d synthetic``      random tokens, deterministic in ``--seed`` (the benchmark source);
  * ``-d <path>``         a ``.bin`` token file (uint16/uint32 memmap, served by the native
                          C++ prefetching loader when built), or ``.txt`` / ``.jsonl`` text
                          tokenised with the model's tokenizer if one is on disk, else bytes;
  * ``-d <hf dataset id>`` the reference's path through ``datasets`` + ``AutoTokenizer``.

``--document-masking`` adds ``position_ids`` to every sample: they count up from 0 inside each document, and a
chunk's first token always has position 0 (a document cut by a chunk boundary continues as a new document in the
next chunk).  Without the flag the samples keep exactly the three keys above.  Where documents come from: each
text of a ``.txt`` / ``.jsonl`` file, each example of a hub dataset, the tokens after each ``--eos-token-id`` in a
``.bin`` file, and seeded random cut points for ``synthetic``.

Differences kept deliberately: pinned host memory + non-blocking H2D (the reference copies
from pageable memory, SURVEY.md §8 #24), and ``set_epoch`` is called in every chapter
(the reference forgets it in chapters 06/07, §8 #6).
"""
from __future__ import annotations

import json
import logging
import os
import random
from itertools import chain

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset
from torch.utils.data.distributed import DistributedSampler

LOGGER = logging.getLogger("dtg_b200")


def positions_from_starts(starts):
    """Position ids (int64, same shape) from boolean document-start flags [..., S]: each token's distance from the
    last start at or before it.  The first token of every row is a start whatever its flag says."""
    starts = torch.as_tensor(starts, dtype=torch.bool).clone()
    starts[..., 0] = True
    idx = torch.arange(starts.shape[-1], device=starts.device).expand(starts.shape)
    return idx - torch.where(starts, idx, torch.zeros_like(idx)).cummax(dim=-1).values


def positions_after_eos(ids, eos_token_id: int):
    """Position ids of a [..., S] id tensor in which a document starts after each ``eos_token_id``; runs on the
    tensor's device without a host synchronisation."""
    starts = torch.zeros(ids.shape, dtype=torch.bool, device=ids.device)
    starts[..., 1:] = ids[..., :-1] == eos_token_id
    return positions_from_starts(starts)


class SyntheticTokens(Dataset):
    """``num_samples`` chunks of uniformly random token ids (generated once, up front).

    ``document_masking=True`` keeps the same tokens and adds ``position_ids`` from seeded random document cut
    points (a generator of its own, so the tokens do not change): inside each chunk, document lengths are drawn
    independently and uniformly from 1 .. max(1, seq_length // 2) starting at token 0, and the last document is cut
    at the chunk end.  Documents therefore average about seq_length / 4 tokens."""

    def __init__(self, num_samples: int, seq_length: int, vocab_size: int, seed: int = 0, document_masking=False):
        g = torch.Generator().manual_seed(seed)
        self.tokens = torch.randint(0, vocab_size, (num_samples, seq_length), generator=g, dtype=torch.int64)
        self.starts = None
        if document_masking:
            gd = torch.Generator().manual_seed(seed + 0x5EED)
            max_len = max(1, seq_length // 2)
            self.starts = torch.zeros(num_samples, seq_length, dtype=torch.bool)
            for i in range(num_samples):
                pos = 0
                while pos < seq_length:
                    self.starts[i, pos] = True
                    pos += int(torch.randint(1, max_len + 1, (1,), generator=gd))

    def __len__(self):
        return self.tokens.shape[0]

    def __getitem__(self, i):
        t = self.tokens[i]
        out = {"input_ids": t, "attention_mask": torch.ones_like(t), "labels": t.clone()}
        if self.starts is not None:
            out["position_ids"] = positions_from_starts(self.starts[i])
        return out


class TokenChunks(Dataset):
    """A flat token stream cut into ``seq_length`` chunks (remainder dropped).  For document masking, either
    ``starts`` (a boolean array over the stream: the token begins a document) or ``eos_token_id`` (a document starts
    after each occurrence) gives every chunk its ``position_ids``."""

    def __init__(self, tokens, seq_length: int, starts=None, eos_token_id=None):
        n = (len(tokens) // seq_length) * seq_length
        self.tokens = tokens
        self.seq_length = seq_length
        self.n_chunks = n // seq_length
        self.starts = starts
        self.eos_token_id = eos_token_id

    def __len__(self):
        return self.n_chunks

    def __getitem__(self, i):
        s = self.seq_length
        t = torch.from_numpy(np.asarray(self.tokens[i * s:(i + 1) * s]).astype(np.int64))
        out = {"input_ids": t, "attention_mask": torch.ones_like(t), "labels": t.clone()}
        if self.starts is not None:
            out["position_ids"] = positions_from_starts(torch.from_numpy(np.asarray(self.starts[i * s:(i + 1) * s])))
        elif self.eos_token_id is not None:
            out["position_ids"] = positions_after_eos(t, self.eos_token_id)
        return out


class ByteTokenizer:
    """UTF-8 byte fallback tokenizer (ids 0..255, 256 = end of document)."""

    vocab_size = 257
    model_max_length = 1 << 30

    def encode(self, text: str):
        return list(text.encode("utf-8")) + [256]


def _load_tokenizer(model_name: str):
    if os.path.isdir(model_name):
        try:
            from transformers import AutoTokenizer

            return AutoTokenizer.from_pretrained(model_name)
        except Exception as e:  # pragma: no cover
            LOGGER.warning(f"no usable tokenizer in {model_name} ({e}); falling back to bytes")
    return None


def _read_texts(path: str):
    if path.endswith(".jsonl"):
        with open(path) as fp:
            for line in fp:
                if line.strip():
                    row = json.loads(line)
                    yield row.get("text") or next(iter(row.values()))
    else:
        with open(path, encoding="utf-8", errors="replace") as fp:
            for line in fp:
                if line.strip():
                    yield line


def clamp_seq_length(seq_length, config):
    """Reference rule (``01:216-218``): too-long requests fall back to min(1024, max_pos)."""
    if seq_length > config.max_position_embeddings:
        return min(1024, config.max_position_embeddings)
    return seq_length


def check_document_masking_args(args):
    """Refuse, before anything is built, a ``--document-masking`` run whose documents cannot be found."""
    if not getattr(args, "document_masking", False):
        return
    name = getattr(args, "dataset_name", None) or ""
    if name.endswith(".bin") and getattr(args, "eos_token_id", None) is None:
        raise ValueError("--document-masking with a .bin dataset needs --eos-token-id: documents start after it")


def load_and_preprocess_data(args, config, dp_size: int = 1):
    """Returns the training ``Dataset``.  ``args`` needs dataset_name, dataset_subset,
    model_name, seq_length, seed, batch_size (+ optional num_samples, document_masking, eos_token_id)."""
    check_document_masking_args(args)
    docs = bool(getattr(args, "document_masking", False))
    seq_length = clamp_seq_length(args.seq_length, config)
    name = args.dataset_name
    if name == "synthetic":
        n = getattr(args, "num_samples", None) or 64 * args.batch_size * dp_size
        return SyntheticTokens(n, seq_length, config.vocab_size, seed=args.seed, document_masking=docs)
    if os.path.isfile(name) and name.endswith(".bin"):
        dtype = np.uint16 if config.vocab_size <= 65536 else np.uint32
        ds = TokenChunks(np.memmap(name, dtype=dtype, mode="r"), seq_length,
                         eos_token_id=args.eos_token_id if docs else None)
        ds.path, ds.vocab_size = name, config.vocab_size  # lets build_dataloader pick the native C++ loader
        return ds
    if os.path.isfile(name):
        tok = _load_tokenizer(args.model_name)
        if tok is None:
            bt = ByteTokenizer()
            texts = [bt.encode(t) for t in _read_texts(name)]
        else:
            texts = [tok(t)["input_ids"] for t in _read_texts(name)]
        ids = np.asarray(list(chain.from_iterable(texts)), dtype=np.int64) % config.vocab_size
        starts = None
        if docs:  # each text is one document
            offsets = np.cumsum([0] + [len(t) for t in texts[:-1]])
            starts = np.zeros(len(ids), dtype=bool)
            starts[offsets[offsets < len(ids)]] = True
        return TokenChunks(ids, seq_length, starts=starts)
    return _load_hf(args, config, seq_length, docs)


def _load_hf(args, config, seq_length, document_masking=False):
    """The reference's path (HF hub or ``$HF_HOME`` cache)."""
    import multiprocessing

    import datasets
    from transformers import AutoTokenizer

    tokenizer = AutoTokenizer.from_pretrained(args.model_name)
    data = datasets.load_dataset(args.dataset_name, args.dataset_subset)
    cols = data["train"].column_names
    text_col = "text" if "text" in cols else cols[0]
    nproc = max(1, multiprocessing.cpu_count() // 2)
    tokenized = data.map(lambda ex: tokenizer(ex[text_col]), batched=True, remove_columns=cols,
                         num_proc=nproc, desc="tokenizing")

    def group(examples):
        if document_masking:  # each example is one document: its positions count up from 0
            examples = dict(examples, position_ids=[list(range(len(x))) for x in examples["input_ids"]])
        cat = {k: list(chain(*examples[k])) for k in examples.keys()}
        total = (len(cat["input_ids"]) // seq_length) * seq_length
        out = {k: [v[i:i + seq_length] for i in range(0, total, seq_length)] for k, v in cat.items()}
        out["labels"] = [list(x) for x in out["input_ids"]]
        if document_masking:  # a document cut by the chunk boundary continues as a new one
            out["position_ids"] = [positions_from_starts(torch.tensor(p) == 0).tolist() for p in out["position_ids"]]
        return out

    lm = tokenized.map(group, batched=True, num_proc=nproc, desc=f"chunking to {seq_length}")
    lm.set_format("torch")
    return lm["train"]


class NativeTokenLoader:
    """Iterable over a ``.bin`` token file served by the C++ loader (``csrc/dataloader.cpp``): mmap + a
    producer thread filling a ring of pinned [batch, seq] buffers.  Quacks like a DataLoader as far as
    ``trainer.train`` is concerned (``len``, ``iter``, ``.sampler.set_epoch``)."""

    def __init__(self, path, seq_length, vocab_size, batch_size, dp_size=1, dp_rank=0, seed=0, depth=4,
                 eos_token_id=None):
        from .. import _ext

        C = _ext.load(required=True)
        token_bytes = 2 if vocab_size <= 65536 else 4
        pin = torch.cuda.is_available()
        self._loader = C.TokenLoader(path, token_bytes, seq_length, batch_size, dp_rank, dp_size, seed, depth, pin)
        self.sampler = self
        self._epoch = 0
        self._started = True  # the constructor already started epoch 0
        self.eos_token_id = eos_token_id  # document masking: to_device derives position_ids on the device

    def set_epoch(self, epoch):
        self._epoch = epoch
        self._loader.set_epoch(epoch)
        self._started = True

    def __len__(self):
        return int(self._loader.num_batches())

    def __iter__(self):
        if not self._started:
            self._loader.set_epoch(self._epoch)
        self._started = False
        for _ in range(len(self)):
            ids = self._loader.next()
            yield RingBatch({"input_ids": ids, "attention_mask": torch.ones_like(ids), "labels": ids}, self._loader,
                            self.eos_token_id)


class RingBatch(dict):
    """A batch whose tensors alias a pinned ring slot of the native loader.  ``to_device`` reports its asynchronous
    H2D copies back (``copied()``) so the producer thread never overwrites a slot whose DMA has not executed yet."""

    def __init__(self, tensors, loader, eos_token_id=None):
        super().__init__(tensors)
        self._loader = loader
        self.eos_token_id = eos_token_id

    def copied(self):
        if torch.cuda.is_available():
            self._loader.mark_copied()


def collate(samples):
    keys = samples[0].keys()
    return {k: torch.stack([torch.as_tensor(s[k]) for s in samples]) for k in keys}


def _seed_worker(worker_id):
    seed = torch.initial_seed() % 2**32
    np.random.seed(seed)
    random.seed(seed)


def build_dataloader(dataset, batch_size, dp_size=1, dp_rank=0, seed=0, distributed=False,
                     num_workers=1, prefetch_factor=2, pin_memory=None, deterministic=False):
    """Single-process: shuffle + drop_last (``01:62-70``).  Distributed: a
    ``DistributedSampler`` keyed on *data-parallel* coordinates so tensor-parallel peers see
    identical batches (``06:141-147``)."""
    if isinstance(dataset, TokenChunks) and getattr(dataset, "path", None) is not None:
        from .. import _ext

        if _ext.available():
            return NativeTokenLoader(dataset.path, dataset.seq_length, dataset.vocab_size, batch_size, dp_size, dp_rank,
                                     seed, eos_token_id=dataset.eos_token_id)
    if pin_memory is None:
        pin_memory = torch.cuda.is_available()
    gen = torch.Generator().manual_seed(seed)
    kwargs = dict(batch_size=batch_size, collate_fn=collate, num_workers=num_workers, pin_memory=pin_memory,
                  generator=gen)
    if num_workers > 0:
        kwargs.update(prefetch_factor=prefetch_factor, persistent_workers=False)
        if deterministic:
            kwargs.update(worker_init_fn=_seed_worker)
    if distributed:
        sampler = DistributedSampler(dataset, num_replicas=dp_size, rank=dp_rank, shuffle=True,
                                     drop_last=True, seed=seed)
        return DataLoader(dataset, sampler=sampler, drop_last=True, **kwargs)
    return DataLoader(dataset, shuffle=True, drop_last=True, **kwargs)


def to_device(batch, device):
    nb = torch.device(device).type == "cuda"
    out = {k: v.to(device=device, non_blocking=nb) for k, v in batch.items()}
    if nb and isinstance(batch, RingBatch):
        batch.copied()
    if getattr(batch, "eos_token_id", None) is not None:
        # native .bin loader with document masking: positions from the ids already on the device
        out["position_ids"] = positions_after_eos(out["input_ids"], batch.eos_token_id)
    return out
