"""DP-SGD local steps (Abadi et al., 2016) with book-keeping clipping: one backward pass.

One local step on B examples releases

    g = (1 / B) * (sum_n clip_C(grad l_n) + z * C * xi),   clip_C(v) = c_n v,

l_n the example's mean loss over its targets, xi_i = dp_gauss4(seed, step, i / 4)[i % 4] at the
DP-SGD site word (``oracle.DPSGD_SITE``), step the plan's optimizer-step word plus the step index.

While a ``DPSGDStep`` is collecting (``begin`` .. ``finish``), the backward of ``ops.nn.linear``,
``lora_linear`` and ``linear_xent`` computes its input gradient as always but, instead of the
weight-gradient GEMM and the bias column sums, launches the site's per-example norm kernel
(csrc/kernels/dpsgd_kernels.cu) and records (output gradient, operand, gradient views).  ``finish``
forms the clip factors c_n against a certified bound of each example's realised contribution, scales
the recorded output-gradient rows by c_n (rounded to bf16, the GEMMs' operand type; an example dropped for
a non-finite bound gets exact zeros in both its output-gradient and its operand rows), runs the same
weight-gradient GEMMs on them with one writer per output element, forms the bias gradients as
fixed-order column sums, and adds the noise.  A DP-SGD step is therefore bit-reproducible run to run
and under CUDA-graph replay.  With no step collecting, every layer runs exactly as without DP-SGD.

The certified bound (DESIGN.md, "DP-SGD"): for site rows t of example n with output-gradient row
dz_t and operand row x_t (x_t extended by a 1 where the site has a bias),

    bound_n = (B ||v_n||) (1 + gamma) + (B sum_t ||dz_t|| ||x_t||) (u + gamma),

||v_n|| the computed norm over every site, u = 2^-8 (bf16 rounding of the scaled rows) and
gamma = 2^-10 (fp32 accumulation of the GEMMs and the norms).  ``clip_factors`` is the fp32 host
mirror of the kernel, operation for operation.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

from .._native import C
from . import gemm as G

_F = np.float32
ONE_PLUS_GAMMA = _F(1.0 + 2.0 ** -10)
U_PLUS_GAMMA = _F(2.0 ** -8 + 2.0 ** -10)

_ACTIVE: Optional["DPSGDStep"] = None


def active() -> Optional["DPSGDStep"]:
    """The step collecting per-example sites, or None (ops.nn's layers then run as always)."""
    return _ACTIVE


def clip_factors(sq: np.ndarray, ab: np.ndarray, batch: int, clip: float) -> np.ndarray:
    """fp32 mirror of ``k_dpsgd_clip``: sq [n_sq, B] and ab [n_ab, B] summed over their rows in order,
    bound = (B sqrt(sq)) (1 + gamma) + (B ab) (u + gamma); c = 0 for a non-finite bound, 1 for
    bound <= clip (bit-pattern compare), else clip / bound."""
    sq, ab = np.asarray(sq, _F), np.asarray(ab, _F)
    with np.errstate(all="ignore"):
        s = np.zeros(sq.shape[1], _F)
        for row in sq:
            s = (s + row).astype(_F)
        a = np.zeros(ab.shape[1] if ab.size else sq.shape[1], _F)
        for row in ab:
            a = (a + row).astype(_F)
        bsz, cl = _F(batch), _F(clip)
        bound = ((np.sqrt(s) * bsz).astype(_F) * ONE_PLUS_GAMMA).astype(_F) + \
            ((a * bsz).astype(_F) * U_PLUS_GAMMA).astype(_F)
        bound = bound.astype(_F)
        c = np.where(bound.view(np.uint32) <= np.array(cl).view(np.uint32), _F(1), (cl / bound).astype(_F))
        return np.where(np.isfinite(bound), c, _F(0)).astype(_F)


def noise_sigma(noise: float, clip: float, batch: int) -> np.float32:
    """The fp32 noise scale z * C / B of one step's averaged gradient."""
    return _F(_F(_F(noise) * _F(clip)) / _F(batch))


def _rows_like(t: torch.Tensor) -> torch.Tensor:
    """An uninitialised bf16 matrix shaped like ``t`` with a 16-byte row pitch, as the GEMMs need."""
    rows, cols = t.shape
    return torch.empty(rows, (cols + 7) // 8 * 8, device=t.device, dtype=t.dtype)[:, :cols]


def _wide_narrow(a: torch.Tensor, b: torch.Tensor):
    return (b, a) if a.shape[1] <= 64 and b.shape[1] > a.shape[1] else (a, b)


class DPSGDStep:
    """Per-step DP-SGD context over a model's flat gradient buffer.  Graph-capturable: every buffer is
    allocated here, sized from ``spec`` (each 2-D parameter is at most one site, whose wide side spans
    ceil(max(shape) / 64) norm tiles), and the noise reads the step word on the device.

    ``batch`` B: examples per step (a site's rows per example is its row count / B); ``clip`` C > 0;
    ``noise`` z >= 0 (0: clipping only, no noise kernel); ``seed`` the client's secret noise key;
    ``step_word`` the int32 [1] device word the noise is keyed by (plus ``finish``'s ``step_add``)."""

    def __init__(self, spec, batch: int, clip: float, noise: float, seed: int, step_word: torch.Tensor,
                 device):
        clip32, noise32 = _F(clip), _F(noise)
        if not (batch >= 1 and math.isfinite(clip32) and clip32 > 0 and math.isfinite(noise32) and noise32 >= 0):
            raise ValueError(f"DP-SGD needs batch >= 1, a finite clip > 0 and a finite noise >= 0 (fp32); got "
                             f"batch {batch}, clip {clip}, noise {noise}")
        self.B, self.clip, self.noise = int(batch), float(clip32), float(noise32)
        self.sigma = float(noise_sigma(noise32, clip32, batch))
        self.seed, self.step_word = int(seed) % (1 << 64), step_word
        mats = [e.shape for e in spec.entries if len(e.shape) == 2]
        rows = sum((max(s) + 63) // 64 for s in mats) or 1
        self.sq = torch.zeros(rows, self.B, device=device, dtype=torch.float32)
        self.ab = torch.zeros(max(2 * len(mats), 1), self.B, device=device, dtype=torch.float32)
        self.c = torch.ones(self.B, device=device, dtype=torch.float32)
        self.dropped = torch.zeros(1, device=device, dtype=torch.int32)   # examples with a non-finite bound
        self._records: List[tuple] = []
        self._n_sq = self._n_ab = 0

    # ---------------------------------------------------------------- collection
    def begin(self):
        global _ACTIVE
        if _ACTIVE is not None:
            raise RuntimeError("a DP-SGD step is already collecting")
        self._records, self._n_sq, self._n_ab = [], 0, 0
        _ACTIVE = self

    def record(self, dz: torch.Tensor, op: torch.Tensor, gw: Optional[torch.Tensor], gb: Optional[torch.Tensor]):
        """A weight-gradient site gw += dz^T op (and gb += column sums of dz): launch its per-example
        norm kernels now, run the GEMM in ``finish`` on the clipped rows."""
        if gw is None and gb is None:
            return
        M = dz.shape[0]
        if M % self.B != 0:
            raise ValueError(f"DP-SGD: a site has {M} rows, not a multiple of the batch {self.B}")
        R = M // self.B
        if gb is not None and R != 1:
            raise ValueError("DP-SGD: a bias gradient needs one row per example (sequence-level biases are not "
                             "supported)")
        if self._n_ab + 1 > self.ab.shape[0]:
            raise RuntimeError("DP-SGD: more sites than the model's parameter spec allows")
        ab = self.ab[self._n_ab]
        self._n_ab += 1
        if R == 1:
            sq = self.sq[self._n_sq]
            self._n_sq += 1
            C().dpsgd_pe_rows(dz, op, 1, 1.0 if gb is not None else 0.0, sq, ab)
        else:
            wide, narrow = _wide_narrow(dz, op)
            if narrow.shape[1] > 64:
                raise ValueError(f"DP-SGD: a sequence site needs one operand at most 64 wide (a LoRA rank); "
                                 f"got {dz.shape[1]} and {op.shape[1]}")
            tiles = (wide.shape[1] + 63) // 64
            if self._n_sq + tiles > self.sq.shape[0]:
                raise RuntimeError("DP-SGD: more norm tiles than the model's parameter spec allows")
            C().dpsgd_pe_norm(wide, narrow, R, self.sq[self._n_sq:self._n_sq + tiles])
            self._n_sq += tiles
            C().dpsgd_pe_rows(wide, narrow, R, 0.0, None, ab)
        self._records.append((dz, op, gw, gb, R))

    # ---------------------------------------------------------------- release
    def finish(self, grad: torch.Tensor, step_add: int):
        """Clip factors, clipped weight and bias gradients, then the noise over all of ``grad``."""
        global _ACTIVE
        if _ACTIVE is not self:
            raise RuntimeError("DPSGDStep.finish without begin")
        _ACTIVE = None
        m = C()
        m.dpsgd_clip(self.sq[:self._n_sq], self._n_sq, self.ab[:self._n_ab], self._n_ab, self.B, float(self.B),
                     self.clip, self.c, self.dropped)
        for dz, op, gw, gb, R in self._records:
            s = _rows_like(dz)
            m.dpsgd_scale_rows(dz, self.c, R, s)
            if gw is not None:
                # a dropped example's operand rows are zeroed too: they may be what is not finite
                x = _rows_like(op)
                m.dpsgd_scale_rows(op, self.c, R, x, mask_only=True)
                # one writer per output element (no split-K atomics): the same bits on every run
                G.gemm(s, x, out=gw, a_mn=True, b_mn=True, accumulate=True)
            if gb is not None:
                m.dpsgd_colsum(s, gb)
        self._records = []
        if self.sigma > 0.0:
            m.dpsgd_noise(grad, self.seed, self.step_word, int(step_add), self.sigma)

    def abandon(self):
        """Stop collecting without releasing anything (a failed backward)."""
        global _ACTIVE
        if _ACTIVE is self:
            _ACTIVE = None
        self._records = []
