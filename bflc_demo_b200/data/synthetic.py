"""Synthetic datasets of the shapes BASELINE.json names (there is no network for the real
ones): FEMNIST 28x28/62 classes, non-IID CIFAR-10 shards, seq-128 token classification, a
topic-mixture bigram corpus for next-token prediction, and
an Occupancy-like 5-feature binary table matching the reference's CSV schema
(python-sdk/data/datatraining.txt: Temperature, Humidity, Light, CO2, HumidityRatio ->
Occupancy; 8143 rows, 21% positive -- SURVEY.md A3).

Every generator is class-conditional (a fixed random prototype per class plus noise) so the
models genuinely learn and committee scores separate honest from Byzantine updates.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import torch


@dataclass
class Shard:
    x: torch.Tensor          # features (uint8 images / float tables / int64 tokens)
    y: torch.Tensor          # int64 labels ([n], or [n, S] next tokens)
    n_classes: int

    def __len__(self) -> int:
        return int(self.x.shape[0])


def _label_split(n: int, n_classes: int, clients: int, alpha: float, rng: np.random.Generator):
    """Per-client label histograms: alpha == 0 -> IID, else Dirichlet(alpha) skew."""
    if alpha <= 0:
        return [np.full(n_classes, 1.0 / n_classes) for _ in range(clients)]
    return [rng.dirichlet(np.full(n_classes, alpha)) for _ in range(clients)]


def femnist_like(clients: int, samples_per_client: int, *, seed: int = 0, alpha: float = 0.0,
                 n_classes: int = 62, hw: int = 28, noise: float = 48.0,
                 only: Optional[int] = None) -> List[Shard]:
    """uint8 [n, hw*hw] images: class prototype (0..255) + Gaussian pixel noise.  The class
    prototypes depend only on ``seed``; client ``i``'s samples only on ``(seed, i)``, so a
    rank can generate just its own shard with ``only=i`` (returns a 1-element list)."""
    protos = np.random.default_rng(seed).integers(0, 256, size=(n_classes, hw * hw)).astype(np.float32)
    out = []
    for i in range(clients):
        if only is not None and i != only:
            continue
        rng = np.random.default_rng([seed, 1000 + i])
        p = _label_split(samples_per_client, n_classes, 1, alpha, rng)[0]
        y = rng.choice(n_classes, size=samples_per_client, p=p)
        x = protos[y] + rng.normal(0, noise, size=(samples_per_client, hw * hw)).astype(np.float32)
        x = np.clip(x, 0, 255).astype(np.uint8)
        out.append(Shard(torch.from_numpy(x), torch.from_numpy(y.astype(np.int64)), n_classes))
    return out


def cifar_like(clients: int, samples_per_client: int, *, seed: int = 0, alpha: float = 0.5,
               n_classes: int = 10) -> List[Shard]:
    """uint8 [n, 3, 32, 32]; non-IID (Dirichlet) by default, as in config #3/#4."""
    rng = np.random.default_rng(seed)
    protos = rng.integers(0, 256, size=(n_classes, 3, 8, 8)).astype(np.float32)
    protos = np.repeat(np.repeat(protos, 4, axis=2), 4, axis=3)  # blocky 32x32 prototypes
    out = []
    for p in _label_split(samples_per_client, n_classes, clients, alpha, rng):
        y = rng.choice(n_classes, size=samples_per_client, p=p)
        x = protos[y] + rng.normal(0, 40.0, size=(samples_per_client, 3, 32, 32)).astype(np.float32)
        out.append(Shard(torch.from_numpy(np.clip(x, 0, 255).astype(np.uint8)),
                         torch.from_numpy(y.astype(np.int64)), n_classes))
    return out


def tokens_like(clients: int, samples_per_client: int, *, seed: int = 0, seq_len: int = 128,
                vocab: int = 30522, n_classes: int = 2, min_len: Optional[int] = None,
                pad_id: int = 0) -> List[Shard]:
    """int64 [n, seq_len] token ids; the label decides which half of the vocabulary the
    sequence is mostly drawn from (sequence classification, BERT config #5).

    ``min_len``: variable-length, right-padded sequences.  Each sample's length is uniform in
    [min_len, seq_len]; its real tokens avoid ``pad_id`` and every position at or past its
    length holds ``pad_id``.  None: every sample fills all seq_len positions."""
    if min_len is not None and not 1 <= min_len <= seq_len:
        raise ValueError(f"tokens_like: min_len {min_len} outside [1, {seq_len}]")
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(clients):
        y = rng.integers(0, n_classes, size=samples_per_client)
        lo = (y[:, None] * (vocab // n_classes)).astype(np.int64)
        biased = lo + rng.integers(0, vocab // n_classes, size=(samples_per_client, seq_len))
        unif = rng.integers(0, vocab, size=(samples_per_client, seq_len))
        pick = rng.random((samples_per_client, seq_len)) < 0.7
        x = np.where(pick, biased, unif).astype(np.int64)
        if min_len is not None:
            x[x == pad_id] = (pad_id + 1) % vocab
            lengths = rng.integers(min_len, seq_len + 1, size=samples_per_client)
            x[np.arange(seq_len)[None, :] >= lengths[:, None]] = pad_id
        out.append(Shard(torch.from_numpy(x), torch.from_numpy(y.astype(np.int64)), n_classes))
    return out


def lm_corpus_like(clients: int, samples_per_client: int, *, seed: int, seq_len: int, vocab: int = 8192,
                   topics: int = 8, alpha: float = 0.0, only: Optional[int] = None,
                   successors: int = 4, smoothing: float = 0.1) -> List[Shard]:
    """Next-token corpus: x = tokens[:, :seq_len], y = tokens[:, 1:] (int64 [n, seq_len], n_classes =
    vocab).  Each topic is a sparse bigram chain: every token has ``successors`` fixed next tokens
    with fixed probabilities (halving from the first), mixed with ``smoothing`` of uniform noise.
    A sample draws one topic from its client's mixture -- uniform, or Dirichlet(``alpha``) per client
    when alpha > 0 -- starts at a uniform token and walks seq_len + 1 tokens.

    The topic tables depend only on ``seed``; client ``i``'s samples only on ``(seed, i)``, so a
    rank can generate just its own shard with ``only=i`` (returns a 1-element list)."""
    trng = np.random.default_rng([seed, 77])
    succ = trng.integers(0, vocab, size=(topics, vocab, successors))
    w = 0.5 ** np.arange(successors)
    cum = np.cumsum(w / w.sum())
    out = []
    for i in range(clients):
        if only is not None and i != only:
            continue
        rng = np.random.default_rng([seed, 1000 + i])
        mix = _label_split(samples_per_client, topics, 1, alpha, rng)[0]
        topic = rng.choice(topics, size=samples_per_client, p=mix)
        toks = np.empty((samples_per_client, seq_len + 1), dtype=np.int64)
        toks[:, 0] = rng.integers(0, vocab, size=samples_per_client)
        for t in range(1, seq_len + 1):
            pick = np.minimum(np.searchsorted(cum, rng.random(samples_per_client), side="right"), successors - 1)
            nxt = succ[topic, toks[:, t - 1], pick]
            noise = rng.random(samples_per_client) < smoothing
            toks[:, t] = np.where(noise, rng.integers(0, vocab, size=samples_per_client), nxt)
        out.append(Shard(torch.from_numpy(toks[:, :seq_len].copy()), torch.from_numpy(toks[:, 1:].copy()), vocab))
    return out


def occupancy_like(n_rows: int = 8143, *, seed: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """Unnormalised 5-feature table with the reference CSV's ranges (CO2 up to ~2000, Light up
    to ~1500) and ~21% positives; Light and CO2 carry the signal, as in the real data."""
    rng = np.random.default_rng(seed)
    y = (rng.random(n_rows) < 0.2123).astype(np.int64)
    temp = rng.normal(20.6, 1.0, n_rows) + 1.2 * y
    hum = rng.normal(25.7, 5.5, n_rows)
    light = np.where(y == 1, rng.normal(460, 60, n_rows), np.abs(rng.normal(20, 60, n_rows)))
    co2 = np.where(y == 1, rng.normal(1040, 250, n_rows), rng.normal(490, 90, n_rows))
    ratio = rng.normal(0.0039, 0.0008, n_rows)
    x = np.stack([temp, hum, light, co2, ratio], 1).astype(np.float32)
    return x, y
