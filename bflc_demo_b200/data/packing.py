"""Packed variable-length token batches: the real tokens of every sequence concatenated, with a
``cu_seqlens`` prefix sum marking where each sequence starts (the layout of FlashAttention's varlen
API and of the MLPerf BERT recipes).  Every row-wise layer then runs on the T real tokens only, and
only attention needs the sequence bounds (``ops.nn.attention_packed``).

    pt = PackedTokens.from_padded(ids, pad_id=0)     # ids: right-padded [N, S] on the GPU
    pt[j:j + B]                                       # samples j .. j+B-1, no host sync

Slicing by samples is what the generic engine does to take mini-batches; it returns views of the
ids and positions, a rebased ``cu_seqlens`` and ``seq_ids`` (device subtractions, so they can be
captured in a CUDA graph) and the host ints ``T`` and ``max_len`` the attention kernels size their
grid with.
"""
from __future__ import annotations

from typing import List

import torch

MAX_SEQ = 512   # the packed attention kernels' longest sequence


class PackedTokens:
    """``ids`` int32 [T], ``pos_ids`` int32 [T] (position inside the sequence), ``seq_ids`` int32 [T]
    (index of the token's sequence in the batch), ``cu_seqlens`` int32 [N+1] on the device with
    ``cu_seqlens[0] == 0``; ``offsets`` the same prefix sum on the host.  ``(seq_ids, pos_ids)`` is
    what a padded batch's row r is as ``(r // S, r % S)``: dropout keys its masks by it."""

    def __init__(self, ids: torch.Tensor, pos_ids: torch.Tensor, cu_seqlens: torch.Tensor, offsets: List[int],
                 seq_ids: torch.Tensor):
        self.ids, self.pos_ids, self.cu_seqlens, self.offsets = ids, pos_ids, cu_seqlens, offsets
        self.seq_ids = seq_ids
        self.T = offsets[-1] - offsets[0]
        self.max_len = max(b - a for a, b in zip(offsets[:-1], offsets[1:])) if len(offsets) > 1 else 0

    @classmethod
    def from_padded(cls, ids: torch.Tensor, pad_id: int) -> "PackedTokens":
        """Pack right-padded ids [N, S]: sample i's tokens are the ones before its first ``pad_id``.
        Raises ValueError for S > 512, for a sample of length 0, and for a ``pad_id`` that is not a
        pure suffix (packing would silently drop the real tokens after it).  One host sync."""
        if ids.dim() != 2:
            raise ValueError(f"PackedTokens: ids must be [N, S], got shape {tuple(ids.shape)}")
        N, S = ids.shape
        if S > MAX_SEQ:
            raise ValueError(f"PackedTokens: sequence length {S} exceeds {MAX_SEQ}")
        ids = ids.to(torch.int32)
        real = ids != pad_id
        lengths = real.sum(1, dtype=torch.int32)
        suffix = real == (torch.arange(S, device=ids.device)[None, :] < lengths[:, None])
        bad = (~suffix.all(1)).sum(dtype=torch.int32).view(1)
        host = torch.cat([lengths, bad]).tolist()                 # the one host sync
        lens, n_bad = host[:N], host[N]
        if N and min(lens) == 0:
            raise ValueError(f"PackedTokens: sample {lens.index(0)} has no token other than pad id {pad_id}")
        if n_bad:
            raise ValueError(f"PackedTokens: pad id {pad_id} appears before a real token in {n_bad} sample(s); "
                             "only right padding can be packed")
        offsets = [0]
        for n in lens:
            offsets.append(offsets[-1] + n)
        T = offsets[-1]
        cu = torch.tensor(offsets, dtype=torch.int32).to(ids.device)
        seq = torch.repeat_interleave(torch.arange(N, device=ids.device), lengths.long(), output_size=T)
        pos = torch.arange(T, device=ids.device, dtype=torch.int32) - cu[seq]
        packed = ids[seq, pos.long()].contiguous()
        return cls(packed, pos.contiguous(), cu, offsets, seq.to(torch.int32))

    def __len__(self) -> int:
        return len(self.offsets) - 1

    def __getitem__(self, idx) -> "PackedTokens":
        if not isinstance(idx, slice):
            raise TypeError("PackedTokens: only slicing by samples is supported")
        lo, hi, step = idx.indices(len(self))
        if step != 1:
            raise ValueError("PackedTokens: slices must be contiguous")
        hi = max(hi, lo)
        a, b = self.offsets[lo], self.offsets[hi]
        base = self.offsets[0]
        cu = self.cu_seqlens[lo:hi + 1] - (a - base)
        seq = self.seq_ids[a - base:b - base] - lo
        return PackedTokens(self.ids[a - base:b - base], self.pos_ids[a - base:b - base], cu,
                            self.offsets[lo:hi + 1], seq)

    @property
    def device(self) -> torch.device:
        return self.ids.device
