"""Python face of the wgmma GEMM (csrc/kernels/gemm_sm100.cu).

``D[b] = alpha * A[b] @ B[b]^T`` with A given as ``[M, K]`` (K-major) or ``[K, M]``
(``a_mn=True``) and B as ``[N, K]`` or ``[K, N]`` (``b_mn=True``); the transposed forms are
consumed directly through MN-major wgmma descriptors, never materialised.

Reference parity: K1 ``tf.matmul(x, W) + b`` (python-sdk/main.py:120,180,293).
"""
from __future__ import annotations

import os
from typing import Optional

import torch

from .._native import C

EPI_GENERIC, EPI_XENT, EPI_ARGMAX = 0, 1, 2
_GEMM2 = os.environ.get("BFLC_GEMM2", "1") != "0"   # route big K-major GEMMs to the CTA-pair kernel
ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2
_DT = {torch.float32: 0, torch.bfloat16: 1, torch.float8_e4m3fn: 2}


def _mat_dims(t: torch.Tensor, mn: bool):
    """rows(M|N), K, ld, batch, batch_stride of an operand (2-D or 3-D, last dim contiguous)."""
    assert t.stride(-1) == 1, "operand rows must be contiguous"
    if t.dim() == 2:
        r, c = t.shape
        batch, bs = 1, 0
    else:
        batch, r, c = t.shape
        bs = t.stride(0) if batch > 1 else 0
    ld = t.stride(-2)
    if mn:
        return c, r, ld, batch, bs  # memory is [K][MN]
    return r, c, ld, batch, bs


def gemm(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, *,
         a_mn: bool = False, b_mn: bool = False, out_dtype: torch.dtype = torch.bfloat16,
         alpha: float = 1.0, bias: Optional[torch.Tensor] = None, act: int = ACT_NONE,
         aux_out: Optional[torch.Tensor] = None, aux_in: Optional[torch.Tensor] = None,
         act_bwd: int = 0, colsum: Optional[torch.Tensor] = None, split_k: int = 1,
         accumulate: bool = False, n_valid: Optional[int] = None,
         b_maps: Optional[torch.Tensor] = None, dyn_ptr: int = 0, batch: Optional[int] = None,
         dbg=(0, 0, 0, 0), tail: Optional[tuple] = None) -> torch.Tensor:
    """``out = act(alpha * a @ b^T + bias)`` (see the module docstring for the operand forms).

    ``split_k > 1`` splits the reduction over CTAs whose fp32 partial sums are added into
    ``out`` with atomics, so ``out`` must be fp32 and the result is *added* to what ``out``
    holds, whatever ``accumulate`` says: pass a zeroed ``out`` for a plain product, or a
    gradient buffer to accumulate into it.  When ``out`` is None a zeroed one is allocated.
    Split-K takes no ``act``, ``aux_out`` or ``act_bwd`` (they are not linear in a partial
    sum); ``bias`` and ``colsum`` are fine.  ``accumulate=True`` needs an fp32 ``out``.  The
    native code refuses the other combinations with a RuntimeError before any launch.

    ``tail=(a2, b2)`` adds a low-rank K tail: ``out = act(alpha * (a @ b^T + a2 @ b2^T) + bias)``
    with ``a2`` [M, r] and ``b2`` [N, r] (or [r, N] when ``b_mn``), bf16 and contiguous, r a
    multiple of 8 in [8, 64].  The tail runs as one more K block of the same wgmma mainloop (a
    LoRA linear's adapter term), always on the single-CTA kernel; it takes batch 1 and the
    generic epilogue without split-K or ``accumulate``."""
    is_fp8 = a.dtype == torch.float8_e4m3fn
    M, K, lda, ba, a_bs = _mat_dims(a, a_mn)
    N, Kb, ldb, bb, b_bs = _mat_dims(b, b_mn)
    assert K == Kb, f"K mismatch {K} vs {Kb}"
    if n_valid is not None:
        N = n_valid
    nb = batch if batch is not None else max(ba, bb)
    if out is None:
        shape = (M, N) if nb == 1 and a.dim() == 2 else (nb, M, N)
        if split_k > 1:
            out = torch.zeros(shape, device=a.device, dtype=torch.float32)
        else:
            out = torch.empty(shape, device=a.device, dtype=out_dtype)
    ldd = out.stride(-2)
    d_bs = out.stride(0) if out.dim() == 3 else 0
    if tail is not None:
        a2, b2 = tail
        if a2.dim() != 2 or b2.dim() != 2:
            raise ValueError("gemm: tail operands must be 2-D")
        k2 = a2.shape[1]
        if (b2.shape[0] if b_mn else b2.shape[1]) != k2:
            raise ValueError(f"gemm: tail ranks differ: a2 {tuple(a2.shape)}, b2 {tuple(b2.shape)}"
                             f"{' (MN-major)' if b_mn else ''}")
        C().gemm(a, b, out, M, N, K, nb, lda, ldb, a_bs, b_bs, a_mn, b_mn, is_fp8, EPI_GENERIC,
                 _DT[out.dtype], ldd, d_bs, alpha, bias, act, aux_out, aux_in, act_bwd, colsum,
                 split_k, accumulate, None, 0, 1.0, None, None, b_maps, None, *dbg, dyn_ptr, 0,
                 a2, b2, k2)
        return out
    # Large plain K-major problems go to the CTA-pair kernel (2-CTA cluster, 256x256 tiles, B
    # multicast to both CTAs): per SM and K-block it moves 32 KB out of L2 instead of 48 KB.
    if (_GEMM2 and not is_fp8 and not a_mn and not b_mn and nb == 1 and a.dim() == 2 and split_k == 1
            and not accumulate and aux_out is None and aux_in is None and colsum is None
            and b_maps is None and dyn_ptr == 0 and out.dtype in (torch.float32, torch.bfloat16)
            and ldd % 4 == 0 and M >= 512 and N >= 512 and M * N >= (1 << 22)
            and C().current_predicate_is_null()):
        C().gemm2(a, b, out, M, N, K, lda, ldb, alpha, bias, act)
        return out
    C().gemm(a, b, out, M, N, K, nb, lda, ldb, a_bs, b_bs, a_mn, b_mn, is_fp8, EPI_GENERIC,
             _DT[out.dtype], ldd, d_bs, alpha, bias, act, aux_out, aux_in, act_bwd, colsum,
             split_k, accumulate, None, 0, 1.0, None, None, b_maps, None, *dbg, dyn_ptr)
    return out


def gemm_xent(a: torch.Tensor, b: torch.Tensor, labels: torch.Tensor, *, n_classes: int,
              bias: Optional[torch.Tensor], dlogits: Optional[torch.Tensor], grad_scale: float,
              loss_sum: torch.Tensor, correct: Optional[torch.Tensor] = None,
              colsum: Optional[torch.Tensor] = None, b_mn: bool = False, alpha: float = 1.0):
    """logits = A @ B^T + bias fused with softmax-cross-entropy: writes dlogits (bf16, padded
    to its row stride), accumulates the loss sum and #correct.  K2 + K6 of the reference
    (python-sdk/main.py:123, 182-183)."""
    is_fp8 = a.dtype == torch.float8_e4m3fn
    M, K, lda, ba, a_bs = _mat_dims(a, False)
    N, Kb, ldb, bb, b_bs = _mat_dims(b, b_mn)
    assert K == Kb
    ldd = dlogits.stride(-2) if dlogits is not None else 0
    C().gemm(a, b, dlogits, M, n_classes, K, 1, lda, ldb, 0, 0, False, b_mn, is_fp8, EPI_XENT, 1,
             ldd, 0, alpha, bias, 0, None, None, 0, colsum, 1, False, labels, 0, grad_scale,
             loss_sum, correct, None, None, 0, 0, 0, 0)


def gemm_argmax_acc(a: torch.Tensor, b: torch.Tensor, labels: torch.Tensor, correct: torch.Tensor,
                    *, n_classes: int, bias: Optional[torch.Tensor] = None, batch: int = 1,
                    a_bs: int = 0, b_bs: int = 0, labels_bs: int = 0,
                    b_maps: Optional[torch.Tensor] = None, dyn_ptr: int = 0, alpha: float = 1.0):
    """#(argmax(A @ B^T + bias) == label) per batch entry -> correct[b]  (committee score)."""
    is_fp8 = a.dtype == torch.float8_e4m3fn
    M, K = a.shape[-2], a.shape[-1]
    C().gemm(a, b, None, M, n_classes, K, batch, a.stride(-2), b.stride(-2), a_bs, b_bs, False,
             False, is_fp8, EPI_ARGMAX, 1, 0, 0, alpha, bias, 0, None, None, 0, None, 1, False,
             labels, labels_bs, 1.0, None, correct, b_maps, None, 0, 0, 0, 0, dyn_ptr)


def gemm_2cta(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, *,
              out_dtype: torch.dtype = torch.bfloat16, alpha: float = 1.0,
              bias: Optional[torch.Tensor] = None, act: int = ACT_NONE) -> torch.Tensor:
    """Large-problem path: 2-CTA clusters computing 256 x 256 tiles with the B tile multicast to
    both CTAs; ``a`` [M, K] and ``b`` [N, K] bf16, K-major (csrc/kernels/gemm2_sm100.cu)."""
    M, K = a.shape
    N = b.shape[0]
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=out_dtype)
    C().gemm2(a, b, out, M, N, K, a.stride(0), b.stride(0), alpha, bias, act)
    return out


FIXED_SPLIT_CTAS = 132   # deterministic split-K: aim for one wave of this many CTAs (a constant, so shapes alone decide)


def fixed_splits(rows: int, n_out: int, k_out: int, groups: int, align: int = 1) -> int:
    """Split count of a deterministic split-K weight gradient [n_out, k_out] reduced over ``rows`` rows made of
    ``groups`` equal groups (a batch's examples): the largest divisor of ``groups`` that keeps the splits x
    128 x 128 output tiles within one wave, every split at least 8 K blocks of 64 rows and its rows a multiple
    of ``align`` (64 for the implicit-GEMM convolution's pixel boxes); 0 if no split count is aligned.  A
    function of the shapes only, so eager runs and graph replay split alike."""
    tiles = ((n_out + 127) // 128) * ((k_out + 127) // 128)
    cap = min(FIXED_SPLIT_CTAS // tiles, rows // (64 * 8))
    ok = [s for s in range(1, groups + 1) if groups % s == 0 and (rows // s) % align == 0]
    return max((s for s in ok if s <= cap), default=ok[0] if ok else 0)


def gemm_dw_fixed_split(dz: torch.Tensor, x: torch.Tensor, gw: torch.Tensor, splits: int) -> torch.Tensor:
    """``gw += dz^T x`` (dz [M, N], x [M, K] bf16 with unit column stride, gw fp32 [N, K] contiguous) with the
    reduction split into ``splits`` equal row ranges: each split is one batch entry of the wgmma GEMM and stores
    its fp32 partial tiles into its own workspace slice with plain stores, then ``dpsgd_sum_slices`` adds the
    slices into gw in slice order.  One writer per element and a fixed order: the same bits on every run, unlike
    ``split_k``'s atomics.  splits == 1 is the single-writer GEMM accumulating into gw."""
    M = dz.shape[0]
    if dz.dim() != 2 or x.dim() != 2 or x.shape[0] != M or dz.dtype != torch.bfloat16 or x.dtype != torch.bfloat16:
        raise ValueError("gemm_dw_fixed_split: dz and x must be bf16 [M, *] matrices with the same rows")
    if gw.dtype != torch.float32 or not gw.is_contiguous() or tuple(gw.shape) != (dz.shape[1], x.shape[1]):
        raise ValueError(f"gemm_dw_fixed_split: gw must be a contiguous fp32 [{dz.shape[1]}, {x.shape[1]}] tensor")
    if splits < 1 or M % splits != 0:
        raise ValueError(f"gemm_dw_fixed_split: {splits} splits do not divide the {M} rows")
    if splits == 1:
        return gemm(dz, x, out=gw, a_mn=True, b_mn=True, accumulate=True)
    ks = M // splits
    a = dz.as_strided((splits, ks, dz.shape[1]), (ks * dz.stride(0), dz.stride(0), 1))
    b = x.as_strided((splits, ks, x.shape[1]), (ks * x.stride(0), x.stride(0), 1))
    ws = torch.empty((splits,) + tuple(gw.shape), device=gw.device, dtype=torch.float32)
    gemm(a, b, out=ws, a_mn=True, b_mn=True)
    C().dpsgd_sum_slices(ws, gw)
    return gw


def conv_dw_fixed_split(x: torch.Tensor, dz: torch.Tensor, gw: torch.Tensor, geom: tuple, groups: int) -> torch.Tensor:
    """``gw += dW`` of an implicit-GEMM convolution (x [N, H, W, C], dz [N*OH*OW, Cout] bf16, gw fp32 [Cout,
    kh*kw*C] contiguous; ``geom`` = (N, C, H, W, kh, kw, stride, pad, OH, OW)) with a deterministic split-K:
    ``fixed_splits`` runs of whole examples (``groups`` of them in all) each store their dW into their own fp32
    workspace slice with plain stores (``conv_dw_groups``), and ``dpsgd_sum_slices`` adds the slices in order."""
    N, Cin, H, W, kh, kw, stride, pad, OH, OW = geom
    K = kh * kw * Cin
    if gw.dtype != torch.float32 or not gw.is_contiguous() or tuple(gw.shape) != (dz.shape[1], K):
        raise ValueError(f"conv_dw_fixed_split: gw must be a contiguous fp32 [{dz.shape[1]}, {K}] tensor")
    splits = fixed_splits(dz.shape[0], dz.shape[1], K, groups, align=64)
    if splits == 0:
        raise ValueError(f"conv_dw_fixed_split: no split of {groups} examples has a multiple of 64 pixels")
    ws = torch.empty(splits, dz.shape[1], K, device=gw.device, dtype=torch.float32)
    C().conv_dw_groups(x, dz, ws, N, H, W, Cin, OH, OW, kh, kw, stride, pad, splits, False)
    C().dpsgd_sum_slices(ws, gw)
    return gw
