"""Fine-tuning optimizer recipe over a flat parameter buffer (DESIGN §3.7): decoupled weight decay
that skips every 1-D parameter, a learning-rate warmup followed by a decay, and global-norm gradient
clipping -- all decided on the device, so a captured training graph replays it with no host sync.

Per step (t = the Adam step, ``*step_dev + step``; s = t - 1):

* ``lr_t = lr * f(s)``, with f the HF ``get_{constant,linear,cosine}_schedule_with_warmup`` lambda
  (``lr_factor`` is its host mirror);
* clipping (``clip_grad_norm = c > 0``): ``grad_norm`` writes n = ||g||_2 and coef = min(1, c / (n + 1e-6)),
  the update uses coef * g; a non-finite n skips the step (weights and moments bit-unchanged, the
  gradient still cleared, the skip counter + 1);
* decay: ``w -= lr_t * wd * w`` ahead of the update, on the 8-float blocks whose bit in the
  no-decay mask (``no_decay_mask``) is clear.

With the defaults (wd = 0, constant, no warmup, no clipping) the engine keeps the plain
``optim_step``; the recipe kernel with a constant schedule, wd = 0 and an untriggered clip computes
bit-identical results to it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .._native import C
from ..config import LR_SCHEDULES


def no_decay_mask(spec, n: Optional[int] = None) -> torch.Tensor:
    """One bit per 8-float block of the flat buffer, set where the block belongs to a 1-D entry of
    ``spec`` (biases, norm scales / shifts, running statistics): bit (j & 31) of int32 word j >> 5.
    ``ParamSpec`` offsets are multiples of 8, so no block is shared by two entries.  CPU int32
    [ceil(n / 256)], n = spec.total by default."""
    n = spec.total if n is None else int(n)
    blocks = np.zeros((n + 255) // 256 * 32, dtype=bool)
    for e in spec.entries:
        if len(e.shape) == 1:
            assert e.offset % 8 == 0
            blocks[e.offset // 8:(e.offset + e.numel + 7) // 8] = True
    words = np.packbits(blocks, bitorder="little").view("<u4").view(np.int32)
    return torch.from_numpy(words.copy())


def lr_factor(schedule: str, s: int, warmup: int, total: int) -> float:
    """Host mirror of the kernel's f(s) (s 0-based)."""
    if s < warmup:
        return s / warmup
    if schedule == "constant":
        return 1.0
    span = max(1, total - warmup)
    if schedule == "linear":
        return max(0.0, (total - s) / span)
    if schedule == "cosine":
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * (s - warmup) / span)))
    raise ValueError(f"unknown lr schedule {schedule!r}")


@dataclass(frozen=True)
class OptimRecipe:
    weight_decay: float = 0.0
    lr_schedule: str = "constant"
    warmup_steps: int = 0
    total_steps: int = 0
    clip_grad_norm: float = 0.0

    @classmethod
    def from_config(cls, cfg) -> "OptimRecipe":
        return cls(float(cfg.weight_decay), cfg.lr_schedule, int(cfg.warmup_steps), int(cfg.total_steps),
                   float(cfg.clip_grad_norm))

    @property
    def is_default(self) -> bool:
        return self == OptimRecipe()

    @property
    def schedule_id(self) -> int:
        return LR_SCHEDULES.index(self.lr_schedule)


class RecipeStep:
    """The recipe's device state for one flat buffer -- no-decay mask, norm workspace, ``norms``
    (fp32, the pre-clip norm of each step index of a round) and ``skipped`` (int32, non-finite steps
    so far) -- all allocated here, so that a call allocates and reads back nothing.

    FedProx: with ``prox_mu > 0`` every step adds ``mu * (w - anchor)`` to the (clipped) gradient,
    ``anchor`` an fp32 tensor like ``master`` that holds the round's global model."""

    def __init__(self, recipe: OptimRecipe, spec, steps: int, device, *, n: Optional[int] = None,
                 anchor: Optional[torch.Tensor] = None, prox_mu: float = 0.0):
        self.recipe = recipe
        self.anchor, self.prox_mu = (anchor, float(prox_mu)) if prox_mu > 0 else (None, 0.0)
        self.mod = C()
        self.mask = no_decay_mask(spec, n).to(device)
        self.workspace = torch.zeros(self.mod.grad_norm_workspace_bytes(), dtype=torch.uint8, device=device)
        self.norms = torch.zeros(max(1, steps), dtype=torch.float32, device=device)
        self.skipped = torch.zeros(1, dtype=torch.int32, device=device)

    def __call__(self, adam: bool, master, grad, shadow, m, v, lr: float, step: int, step_dev_ptr: int,
                 index: int, beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-8, zero_grad: bool = True):
        """One step: the norm kernel (clipping on), then the update, its PDL successor.  ``index``
        selects the ``norms`` slot."""
        r = self.recipe
        clip = r.clip_grad_norm > 0
        if clip:
            self.mod.grad_norm(grad, self.workspace, self.norms, index, r.clip_grad_norm, self.skipped)
        self.mod.optim_recipe_step(adam, master, grad, shadow, m, v, lr, beta1, beta2, eps, step, step_dev_ptr,
                                   r.weight_decay, self.mask if r.weight_decay > 0 else None, r.schedule_id,
                                   r.warmup_steps, r.total_steps, self.workspace if clip else None,
                                   zero_grad=zero_grad, anchor=self.anchor, prox_mu=self.prox_mu)
