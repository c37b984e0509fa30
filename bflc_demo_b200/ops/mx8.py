"""Block-scaled fp8 (OCP MXFP8) operands and GEMM (csrc/kernels/gemm_mx8_sm100.cu).

An :class:`MX8` holds e4m3 elements ``q [R, ld]`` plus one UE8M0 scale per 32 K-elements in
the chunk layout the GEMM kernels read straight out of shared memory.
``gemm_mx8(a, b)`` = ``(a.q * a.scale) @ (b.q * b.scale)^T`` on
e4m3 wgmma per 32-element K-group with the UE8M0 scales applied in registers.

Reference parity: the reference's dense layers (python-sdk/main.py:120-123) in the precision
BASELINE.json names for the MLP / LeNet-5 configs.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from .._native import C

SF_CHUNK = 512


@dataclass
class MX8:
    q: torch.Tensor          # float8_e4m3fn [R, ld]  (ld = K rounded up to 16)
    sf: torch.Tensor         # uint8 scale chunks [row_block][k_block][512]
    rows: int
    K: int

    def dequantize(self) -> torch.Tensor:
        """fp32 [rows, K] (test / debug path, plain PyTorch)."""
        kb = (self.K + 127) // 128
        rb = self.sf.numel() // (kb * SF_CHUNK)
        s = self.sf.view(rb, kb, 32, 4, 4).permute(0, 3, 2, 1, 4)      # [rb, r1, r0, kb, kk]
        s = s.reshape(rb * 128, kb * 4)[: self.rows]
        scale = torch.exp2(s.float() - 127.0).repeat_interleave(32, dim=1)[:, : self.K]
        return self.q[:, : self.K].float() * scale


FP32_MIN_NORMAL = 2.0 ** -126


def _ftz(t: torch.Tensor) -> torch.Tensor:
    """fp32 values below 2^-126 in magnitude -> signed zero (what ``mul.ftz`` / ``max.ftz`` do)."""
    return torch.where(t.abs() < FP32_MIN_NORMAL, t * 0.0, t)


def mx8_scale_bytes(amax: torch.Tensor) -> torch.Tensor:
    """Exact UE8M0 byte of groups whose largest magnitude is ``amax`` (fp32, >= 0): the smallest
    e with 448 * 2^(e-127) >= amax, clamped to [3, 254]; 127 for an all-zero group.  No
    floating-point log2: frexp gives amax = m * 2^x, m in [0.5, 1), and one exact fp64 comparison
    with 448 * 2^(x-9) = 0.875 * 2^x settles the boundary."""
    a = amax.double()
    m, x = torch.frexp(a)
    k = x.long() - 9 + (m > 0.875).long()          # smallest k with 448 * 2^k >= amax
    e = (k + 127).clamp(3, 254)
    return torch.where(a > 0, e, torch.full_like(e, 127)).to(torch.uint8)


def quantize_mx8_reference(x: torch.Tensor, *, in_scale: float = 1.0) -> MX8:
    """Plain-PyTorch (CPU or GPU) specification of ``k_quantize_mx8`` (and of every other MXFP8
    quantiser, ``epi::mx8_quant32``): per (row, 32-element K group) the UE8M0 byte is the smallest
    e with ``448 * 2^(e-127) >= amax``, computed exactly (:func:`mx8_scale_bytes`), clamped to
    [3, 254] (from 3 up every dequantised value is exactly a bf16 value); elements
    ``e4m3(x * 2^(127-e))`` saturating to +-448.  Like the fast-math kernels, values below 2^-126 in
    magnitude are flushed to signed zero twice: the input ``x`` and the fp32 product
    ``x * in_scale`` (``mul.ftz`` zeroes a subnormal input before ``in_scale`` could make it
    normal).  Scales are stored in the tensor-core chunk layout -- per (128-row block, 128-K block)
    512 bytes, byte ``[r % 32][r // 32][k // 32]``.  Rows are padded to 256, K groups to a multiple
    of 4; padding carries scale 1.0 (0x7F)."""
    assert x.dim() == 2
    R, K = x.shape
    xf = _ftz(_ftz(x.float()) * in_scale)
    kb = (K + 127) // 128
    G = kb * 4
    pad = torch.zeros(R, G * 32, dtype=torch.float32, device=x.device)
    pad[:, :K] = xf
    g = pad.view(R, G, 32)
    e = mx8_scale_bytes(g.abs().amax(-1)).long()
    n_real = (K + 31) // 32
    e[:, n_real:] = 127                                    # groups entirely beyond K
    inv = torch.exp2((127 - e).double())                   # 2^(127-e): exact, as in the kernels
    q = (g.double() * inv.unsqueeze(-1)).clamp(-448.0, 448.0).float().view(R, G * 32)
    ld = (K + 15) // 16 * 16
    qq = torch.zeros(R, ld, dtype=torch.float8_e4m3fn, device=x.device)
    qq[:, :K] = q[:, :K].to(torch.float8_e4m3fn)
    return encode_mx8(qq, e.to(torch.uint8), R, K)


def encode_mx8(q: torch.Tensor, scale_bytes: torch.Tensor, rows: int, K: int) -> MX8:
    """Byte-level encoder: e4m3 codes ``q [rows, ld]`` (float8_e4m3fn or uint8) and UE8M0 bytes
    ``scale_bytes [rows, ceil(K / 32)]`` (or wider) -> an :class:`MX8` with the scales in the chunk
    layout; padding rows / groups carry 0x7F.  :meth:`MX8.dequantize` is its decoder."""
    kb = (K + 127) // 128
    G = kb * 4
    n_real = (K + 31) // 32
    rb = (rows + 255) // 256 * 2
    sf_rows = torch.full((rb * 128, G), 127, dtype=torch.uint8, device=q.device)
    sf_rows[:rows, :n_real] = scale_bytes[:rows, :n_real].to(torch.uint8)
    # [rb, r1, r0, kb, kk] -> chunk bytes [rb, kb, r0, r1, kk]
    sf = sf_rows.view(rb, 4, 32, kb, 4).permute(0, 3, 2, 1, 4).contiguous().view(-1)
    if q.dtype == torch.uint8:
        q = q.view(torch.float8_e4m3fn)
    return MX8(q, sf, rows, K)


def quantize_mx8(x: torch.Tensor, *, in_scale: float = 1.0, out: Optional[MX8] = None) -> MX8:
    """x [R, K] (f32 / bf16 / u8) * in_scale -> MX8 (scales along K)."""
    assert x.dim() == 2 and x.stride(1) == 1
    R, K = x.shape
    if out is None:
        ld = (K + 15) // 16 * 16
        q = torch.zeros(R, ld, device=x.device, dtype=torch.float8_e4m3fn)
        sf = torch.empty(C().mx8_sf_bytes(R, K), device=x.device, dtype=torch.uint8)
        out = MX8(q, sf, R, K)
    C().quantize_mx8(x, out.q, out.sf, R, K, in_scale)
    return out


def gemm_mx8(a: MX8, b: MX8, out: Optional[torch.Tensor] = None, *,
             out_dtype: torch.dtype = torch.bfloat16, alpha: float = 1.0,
             bias: Optional[torch.Tensor] = None, act: int = 0) -> torch.Tensor:
    assert a.K == b.K, f"K mismatch {a.K} vs {b.K}"
    M, N = a.rows, b.rows
    if out is None:
        ldd = (N + 3) // 4 * 4
        buf = torch.empty(M, ldd, device=a.q.device, dtype=out_dtype)
        out = buf[:, :N] if ldd != N else buf
    C().gemm_mx8(a.q, a.sf, b.q, b.sf, out, M, N, a.K, alpha, bias, act)
    return out
