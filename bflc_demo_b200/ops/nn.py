"""Autograd layer functions over the hand-written kernels.

Activations are bf16 autograd tensors; parameters are NOT autograd leaves: every function takes
the bf16 shadow weight it computes with, the fp32 master bias, and the fp32 gradient views
(``gw``/``gb``, slices of the model's flat gradient buffer) that its backward accumulates into
directly.  Passing ``gw=None`` gives an inference-only call, and because a weight is just a
pointer, the same functions run a model whose parameters live in a *peer GPU's* HBM (committee
validation: the GEMMs' TMA loads pull the candidate's weights over NVLink).

Every GEMM here is ``ops.gemm`` (wgmma).  Reference ops covered: K1 matmul+bias, K2
softmax-xent, K3 backward (SURVEY.md 2.7a); the rest exists for the LeNet/ResNet/BERT configs.
"""
from __future__ import annotations

import os
from typing import NamedTuple, Optional

import torch
from torch.autograd import Function

from .._native import C
from . import dpsgd
from . import gemm as G

BF = torch.bfloat16

# Forward-GEMM precision of Linear / Conv2d: "bf16" or "mx8" (block-scaled fp8,
# e4m3 with per-32-element scales: activations and weights are quantised to e4m3 with one UE8M0
# scale per 32 K-elements right before the GEMM).  Backward GEMMs stay bf16 on the saved bf16
# operands (forward-fp8 / backward-bf16 recipe); master weights, gradients and optimizer fp32.


def _sms() -> int:
    """Streaming multiprocessors of the current device (split-K sizing)."""
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


_PRECISION = "bf16"
_MX_BUF: dict = {}


def set_precision(p: str) -> str:
    """-> the previous setting."""
    global _PRECISION
    if p not in ("bf16", "mx8"):
        raise ValueError("precision must be 'bf16' or 'mx8'")
    prev, _PRECISION = _PRECISION, p
    return prev


def get_precision() -> str:
    return _PRECISION


def _mx_quant(tag: str, t: torch.Tensor):
    from .mx8 import MX8, quantize_mx8
    R, K = t.shape
    key = (tag, R, K, t.device.index)
    buf = _MX_BUF.get(key)
    if buf is None:
        ld = (K + 15) // 16 * 16
        buf = MX8(torch.zeros(R, ld, device=t.device, dtype=torch.float8_e4m3fn),
                  torch.empty(C().mx8_sf_bytes(R, K), device=t.device, dtype=torch.uint8), R, K)
        _MX_BUF[key] = buf
    return quantize_mx8(t, out=buf)


def _fwd_gemm(x, w, y, bias, act, pre):
    """y = act(x @ w^T + bias) in the configured forward precision."""
    if _PRECISION == "mx8" and act != G.ACT_GELU and y.stride(0) % 4 == 0:
        from .mx8 import gemm_mx8
        gemm_mx8(_mx_quant("x", x), _mx_quant("w", w), out=y, bias=bias, act=act)
    else:
        G.gemm(x, w, out=y, bias=bias, act=act, aux_out=pre)


def _split_k(out_rows: int, out_cols: int, k: int) -> int:
    """Split the reduction when a weight-gradient GEMM has few output tiles but a long K."""
    tiles = ((out_rows + 127) // 128) * ((out_cols + 127) // 128)   # widest tile: 128 x 128
    kb = (k + 63) // 64
    sms = _sms()
    if 2 * tiles >= sms or kb < 8:
        return 1
    return max(1, min(kb // 2, sms // tiles, 32))


def _dw(dz: torch.Tensor, x: torch.Tensor, gw: torch.Tensor):
    """gw[N, K] += dz[M, N]^T @ x[M, K]   (both operands consumed MN-major, no transposes)."""
    sk = _split_k(gw.shape[0], gw.shape[1], dz.shape[0])
    if sk > 1:
        G.gemm(dz, x, out=gw, a_mn=True, b_mn=True, split_k=sk)
    else:
        G.gemm(dz, x, out=gw, a_mn=True, b_mn=True, accumulate=True)


def _no_dpsgd(who: str, *grads):
    """A layer without per-example gradient norms refuses to accumulate a gradient while a DP-SGD step
    collects: its contribution would escape the clip."""
    if dpsgd.active() is not None and any(g is not None for g in grads):
        raise RuntimeError(f"DP-SGD: {who} has trainable parameters but no per-example gradient norms")


class LinearFn(Function):
    @staticmethod
    def forward(ctx, x, w, b, gw, gb, act, need_dx=True):
        ctx.need_dx = need_dx
        x = x.contiguous()
        M, N = x.shape[0], w.shape[0]
        y = torch.empty(M, N, device=x.device, dtype=BF)
        pre = torch.empty_like(y) if act == G.ACT_GELU else None
        _fwd_gemm(x, w, y, b, act, pre)
        ctx.save_for_backward(x, w, y if act == G.ACT_RELU else pre)
        ctx.gw, ctx.gb, ctx.act = gw, gb, act
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, aux = ctx.saved_tensors
        dy = dy.contiguous()
        M, N = dy.shape
        dp = dpsgd.active()          # DP-SGD: the weight and bias gradients wait for the clip factors
        gb = ctx.gb if dp is None else None
        if ctx.act != G.ACT_NONE:
            dz = torch.empty_like(dy)
            C().act_bwd_colsum(dy, aux, dz, gb, M, N, ctx.act)
        else:
            dz = dy
            if gb is not None:
                C().act_bwd_colsum(dy, None, None, gb, M, N, 0)
        if dp is not None:
            dp.record(dz, x, ctx.gw, ctx.gb)
        elif ctx.gw is not None:
            _dw(dz, x, ctx.gw)
        dx = G.gemm(dz, w, b_mn=True) if (ctx.needs_input_grad[0] and ctx.need_dx) else None
        return dx, None, None, None, None, None, None


def linear(x, w, b=None, gw=None, gb=None, act=G.ACT_NONE, need_dx=True):
    """``need_dx=False`` on a model's first layer: its input only carries ``requires_grad`` so
    that autograd runs the backward functions (parameters are not autograd leaves)."""
    return LinearFn.apply(x, w, b, gw, gb, act, need_dx)


class LoRALinearFn(Function):
    """``y = act(x w^T + scale * (x a^T) bl^T + b)`` with ``w``/``b`` frozen and the adapters
    ``a`` [r, K], ``bl`` [N, r] trained: two GEMMs forward (``u = scale * x a^T`` in bf16, then the
    main GEMM with ``u bl^T`` as its low-rank K tail, so bias and activation see the sum) and four
    backward (``v = scale * dz bl``, ``gbl += dz^T u``, ``ga += v^T x``, ``dx = dz w + v a`` with
    the tail again)."""

    @staticmethod
    def forward(ctx, anchor, x, w, b, a, bl, ga, gbl, scale, act, need_dx=True):
        ctx.need_dx = need_dx
        x = x.contiguous()
        M, N = x.shape[0], w.shape[0]
        u = G.gemm(x, a, alpha=scale)                                  # [M, r] bf16
        y = torch.empty(M, N, device=x.device, dtype=BF)
        pre = torch.empty_like(y) if act == G.ACT_GELU else None
        G.gemm(x, w, out=y, bias=b, act=act, aux_out=pre, tail=(u, bl))
        ctx.save_for_backward(x, w, a, bl, u, y if act == G.ACT_RELU else pre)
        ctx.ga, ctx.gbl, ctx.scale, ctx.act = ga, gbl, scale, act
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, a, bl, u, aux = ctx.saved_tensors
        dy = dy.contiguous()
        M, N = dy.shape
        if ctx.act != G.ACT_NONE:
            dz = torch.empty_like(dy)
            C().act_bwd_colsum(dy, aux, dz, None, M, N, ctx.act)
        else:
            dz = dy
        v = G.gemm(dz, bl, b_mn=True, alpha=ctx.scale)                 # [M, r] bf16
        dp = dpsgd.active()
        if dp is not None:           # DP-SGD: both adapter gradients wait for the clip factors
            dp.record(dz, u, ctx.gbl, None)
            dp.record(v, x, ctx.ga, None)
        else:
            if ctx.gbl is not None:
                _dw(dz, u, ctx.gbl)
            if ctx.ga is not None:
                _dw(v, x, ctx.ga)
        dx = None
        if ctx.needs_input_grad[1] and ctx.need_dx:
            dx = G.gemm(dz, w, b_mn=True, tail=(v, a))
        return None, dx, None, None, None, None, None, None, None, None, None


def lora_linear(x, w, b, a, bl, ga, gbl, scale: float, act=G.ACT_NONE, need_dx=True):
    """LoRA linear over a frozen ``w`` [N, K] (bf16) and ``b`` [N] (fp32 or None): ``a`` [r, K]
    and ``bl`` [N, r] are the bf16 adapter views, ``ga``/``gbl`` their fp32 gradient views
    (accumulated into; None for inference).  r is a multiple of 8 in [8, 64].  ``w`` and ``b``
    get no gradient.  The forward GEMMs are bf16 whatever ``set_precision`` says: the mx8
    forward has no low-rank tail, so it is refused."""
    if _PRECISION != "bf16":
        raise ValueError(f"lora_linear: forward precision {_PRECISION!r} is not supported; LoRA runs bf16")
    r = a.shape[0]
    if a.dim() != 2 or bl.dim() != 2 or bl.shape[1] != r or a.shape[1] != w.shape[1] or bl.shape[0] != w.shape[0]:
        raise ValueError(f"lora_linear: adapters a {tuple(a.shape)} / bl {tuple(bl.shape)} do not fit "
                         f"w {tuple(w.shape)}")
    if r % 8 != 0 or not 8 <= r <= 64:
        raise ValueError(f"lora_linear: rank must be a multiple of 8 in [8, 64], got {r}")
    # `anchor` makes the output join the autograd graph when the adapters train, even where x
    # carries no gradient (the first adapted projection after a frozen embedding)
    anchor = torch.zeros(1, device=x.device, requires_grad=(ga is not None or gbl is not None)
                         and torch.is_grad_enabled())
    return LoRALinearFn.apply(anchor, x, w, b, a, bl, ga, gbl, float(scale), act, need_dx)


class LinearXentFn(Function):
    """Classifier head fused with softmax-cross-entropy (mean over rows); also counts hits.

    The forward writes dlogits of the mean loss and their column sums into scratch buffers; the
    backward scales both by the upstream gradient ``gout`` on the device (no host read, so it can
    be graph-captured) and only then touches ``gw`` / ``gb``.  A forward that is never
    backpropagated leaves the gradient buffer alone."""

    @staticmethod
    def forward(ctx, h, w, b, gw, gb, labels, correct):
        h = h.contiguous()
        M, n_cls = h.shape[0], w.shape[0]
        ncp = (n_cls + 7) // 8 * 8
        dl = torch.zeros(M, ncp, device=h.device, dtype=BF)
        loss = torch.zeros(1, device=h.device, dtype=torch.float32)
        db = torch.zeros(n_cls, device=h.device, dtype=torch.float32) if gb is not None else None
        G.gemm_xent(h, w, labels, n_classes=n_cls, bias=b, dlogits=dl, grad_scale=1.0 / M,
                    loss_sum=loss, correct=correct, colsum=db)
        ctx.save_for_backward(h, w, dl, db)
        ctx.gw, ctx.gb, ctx.n_cls = gw, gb, n_cls
        return loss / M

    @staticmethod
    def backward(ctx, gout):
        h, w, dl, db = ctx.saved_tensors
        # dl * gout rounds once to bf16 (exact for gout == 1); the ncp-wide rows keep the
        # 16-byte row pitch the GEMMs need, and the pad columns stay zero
        dlv = torch.mul(dl, gout).to(BF)[:, :ctx.n_cls]
        dp = dpsgd.active()
        if dp is not None:           # DP-SGD: the head's gradients wait for the clip factors
            dp.record(dlv, h, ctx.gw, ctx.gb)
        else:
            if ctx.gb is not None:
                ctx.gb.addcmul_(db, gout)
            if ctx.gw is not None:
                _dw(dlv, h, ctx.gw)
        dh = G.gemm(dlv, w, b_mn=True) if ctx.needs_input_grad[0] else None
        return dh, None, None, None, None, None, None


def linear_xent(h, w, b, gw, gb, labels, correct=None):
    return LinearXentFn.apply(h, w, b, gw, gb, labels, correct)


def _lm_logits(h, w):
    """fp32 logits h @ w^T [M, V] (bf16 operands, whatever set_precision says) with a row pitch
    rounded up to 4 floats, as xent_rows reads it."""
    M, V = h.shape[0], w.shape[0]
    buf = torch.empty(M, (V + 3) // 4 * 4, device=h.device, dtype=torch.float32)
    return G.gemm(h, w, out=buf[:, :V])


class LMXentFn(Function):
    """Language-model head: logits = h @ w^T over the whole vocabulary, then the mean token
    cross-entropy (csrc/kernels/nn_kernels.cu, xent_rows).  The forward writes dlogits of the mean
    loss (grad_scale = 1 / M, a host constant, so the call can be graph-captured); the backward
    scales them by ``gout`` on the device, accumulates ``gw += dlogits^T h`` (so a tied embedding's
    gradient collects both contributions) and returns dh = dlogits @ w."""

    @staticmethod
    def forward(ctx, h, w, gw, targets, correct):
        h = h.contiguous()
        M, V = h.shape[0], w.shape[0]
        logits = _lm_logits(h, w)
        dl = torch.empty(M, (V + 7) // 8 * 8, device=h.device, dtype=BF)
        rows = torch.empty(M, device=h.device, dtype=torch.float32)
        C().xent_rows(logits, V, targets, rows, correct, dl, 1.0 / M)
        del logits
        ctx.save_for_backward(h, w, dl)
        ctx.gw, ctx.V = gw, V
        return rows.sum(0, keepdim=True) / M       # a fixed-order reduction: deterministic

    @staticmethod
    def backward(ctx, gout):
        h, w, dl = ctx.saved_tensors
        _no_dpsgd("lm_xent", ctx.gw)
        dlv = torch.mul(dl, gout).to(BF)[:, :ctx.V]   # pad columns stay zero, the row pitch 16-byte aligned
        if ctx.gw is not None:
            _dw(dlv, h, ctx.gw)
        dh = G.gemm(dlv, w, b_mn=True) if ctx.needs_input_grad[0] else None
        return dh, None, None, None, None


def _check_targets(who: str, h, targets):
    if targets.dtype != torch.int32 or targets.numel() != h.shape[0]:
        raise ValueError(f"{who}: targets must be int32 with one entry per row of h; got {targets.dtype} "
                         f"[{targets.numel()}] for {h.shape[0]} rows")


def lm_xent(h, w, gw, targets, correct=None):
    """Mean next-token cross-entropy of h [M, K] bf16 under the output matrix w [V, K] bf16 (no bias;
    e.g. a tied word embedding), targets int32 [M].  ``gw`` (fp32 [V, K] or None) accumulates the
    weight gradient; ``correct`` (int32 [1] or None) += #(argmax == target).  The logits are
    materialised in fp32, M x V."""
    _check_targets("lm_xent", h, targets)
    return LMXentFn.apply(h, w, gw, targets, correct)


@torch.no_grad()
def lm_hits(h, w, targets, correct, rows_per_chunk: int = 2048):
    """correct += #(argmax(h @ w^T) == target) over the rows of h, ``rows_per_chunk`` rows at a time
    so the fp32 logits take at most rows_per_chunk x V floats.  The chunking is fixed by the shapes,
    so the sequence can be captured in a CUDA graph."""
    _check_targets("lm_hits", h, targets)
    if rows_per_chunk <= 0:
        raise ValueError(f"lm_hits: rows_per_chunk must be > 0, got {rows_per_chunk}")
    h = h.contiguous()
    V = w.shape[0]
    for r in range(0, h.shape[0], rows_per_chunk):
        hc = h[r:r + rows_per_chunk]
        C().xent_rows(_lm_logits(hc, w), V, targets[r:r + rows_per_chunk], None, correct, None, 1.0)
    return correct


_IMPLICIT = os.environ.get("BFLC_CONV_IMPLICIT", "1") != "0"


def _pix_tile(pix: int, OH: int, OW: int) -> bool:
    """Can `pix` consecutive output pixels be fetched as one TMA box of whole image rows?"""
    if OW > pix or pix % OW:
        return False
    rows = pix // OW
    return OH % rows == 0 if rows <= OH else rows % OH == 0


def conv_is_implicit(H, W, Cin, kh, kw, stride, pad, Kp) -> bool:
    """Implicit-GEMM eligibility (csrc/kernels/gemm_sm100.cu, ConvView): 64-channel K blocks and
    pixel tiles made of whole image rows; everything else takes the im2col path."""
    OH, OW = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
    return (_IMPLICIT and _PRECISION == "bf16" and Cin % 64 == 0 and Kp == kh * kw * Cin
            and _pix_tile(128, OH, OW) and _pix_tile(64, OH, OW) and OW * stride <= 256)


def _conv_rows_gemm(flip, act_src, w, out, N, GH, GW, Cc, OH, OW, kh, kw, stride, pad, n_out, bias=None,
                    act=G.ACT_NONE, pre=None):
    """Mode-1 implicit GEMM (rows = pixels).  Few output tiles but a long reduction (the deep,
    small-image ResNet layers) would leave most SMs idle and run the rest at the 128 x 64 tile's
    L2-feed limit: split the taps x channels reduction over CTAs into an fp32 workspace
    (red.add), then cast -- 128-column tiles on every SM."""
    M, kb = N * OH * OW, kh * kw * Cc // 64
    tiles = ((M + 127) // 128) * ((n_out + 127) // 128)
    sms = _sms()
    sk = min(sms // tiles, kb // 4) if 2 * tiles <= sms else 1
    if sk >= 2 and bias is None and act == G.ACT_NONE and pre is None and n_out % 4 == 0:
        ws = torch.zeros(M, n_out, device=out.device, dtype=torch.float32)
        C().conv_gemm(1, flip, act_src, w, ws, N, GH, GW, Cc, OH, OW, kh, kw, stride, pad, n_out, None, 0,
                      None, None, 0, None, sk, False)
        C().cast_f32_to_bf16(ws.view(-1), out.view(-1))
    else:
        C().conv_gemm(1, flip, act_src, w, out, N, GH, GW, Cc, OH, OW, kh, kw, stride, pad, n_out, bias, act,
                      pre, None, 0, None, 1, False)


class ConvImplicitFn(Function):
    """NHWC convolution as an implicit GEMM: the wgmma GEMM's TMA producer fetches each
    (filter tap, 64 channels) K block as a tap-shifted 4-D box of the activation itself, the
    border zero-filled by the TMA unit -- no im2col buffer in forward, input-gradient
    (stride 1) or weight-gradient."""

    @staticmethod
    def forward(ctx, x, w, b, gw, gb, kh, kw, stride, pad, act, need_dx=True):
        x = x.contiguous()
        N, H, W, Cin = x.shape
        Cout = w.shape[0]
        OH, OW = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
        y = torch.empty(N * OH * OW, Cout, device=x.device, dtype=BF)
        pre = torch.empty_like(y) if act == G.ACT_GELU else None
        _conv_rows_gemm(0, x, w, y, N, H, W, Cin, OH, OW, kh, kw, stride, pad, Cout, b, act, pre)
        ctx.save_for_backward(x, w, y if act == G.ACT_RELU else pre)
        ctx.gw, ctx.gb, ctx.act, ctx.need_dx = gw, gb, act, need_dx
        ctx.geom = (N, Cin, H, W, kh, kw, stride, pad, OH, OW)
        return y.view(N, OH, OW, Cout)

    @staticmethod
    def backward(ctx, dy):
        x, w, aux = ctx.saved_tensors
        _no_dpsgd("conv2d", ctx.gw, ctx.gb)
        N, Cin, H, W, kh, kw, stride, pad, OH, OW = ctx.geom
        Cout = w.shape[0]
        dy = dy.contiguous().view(-1, Cout)
        rows = dy.shape[0]
        if ctx.act != G.ACT_NONE:
            dz = torch.empty_like(dy)
            C().act_bwd_colsum(dy, aux, dz, ctx.gb, rows, Cout, ctx.act)
        else:
            dz = dy
            if ctx.gb is not None:
                C().act_bwd_colsum(dy, None, None, ctx.gb, rows, Cout, 0)
        if ctx.gw is not None:
            tiles = ((Cout + 127) // 128) * ((kh * kw * Cin + 127) // 128)
            sk = max(1, min(_sms() // tiles, (rows // 64) // 2, 32))
            C().conv_gemm(2, 0, x, dz, ctx.gw, N, H, W, Cin, OH, OW, kh, kw, stride, pad, Cout, None, 0,
                          None, None, 0, None, sk, sk == 1)
        dx = None
        if ctx.needs_input_grad[0] and ctx.need_dx:
            dx = torch.empty(N, H, W, Cin, device=dy.device, dtype=BF)
            if Cout % 64 == 0 and _pix_tile(128, H, W):
                if stride == 1:
                    g, GH, GW = dz, OH, OW
                else:   # zero-stuffed dy on the input grid, then the stride-1 form
                    g, GH, GW = torch.empty(N, H, W, Cout, device=dy.device, dtype=BF), H, W
                    C().upsample_zero(dz, g, N, H, W, OH, OW, Cout, stride)
                _conv_rows_gemm(1, g, w, dx.view(-1, Cin), N, GH, GW, Cout, H, W, kh, kw, 1, pad, Cin)
            else:
                dcol = G.gemm(dz, w, b_mn=True)
                C().col2im(dcol, dx, N, Cin, H, W, kh, kw, stride, pad, OH, OW)
        return (dx,) + (None,) * 10


class Conv2dFn(Function):
    """NHWC convolution = im2col + wgmma GEMM (+bias, +activation epilogue)."""

    @staticmethod
    def forward(ctx, x, w, b, gw, gb, kh, kw, stride, pad, act, need_dx=True):
        ctx.need_dx = need_dx
        x = x.contiguous()
        N, H, W, Cin = x.shape
        Cout, Kp = w.shape
        OH, OW = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
        rows, kc = N * OH * OW, kh * kw * Cin
        col = (torch.zeros if Kp != kc else torch.empty)(rows, Kp, device=x.device, dtype=BF)
        C().im2col(x, col, N, Cin, H, W, kh, kw, stride, pad, OH, OW)
        y = torch.empty(rows, Cout, device=x.device, dtype=BF)
        pre = torch.empty_like(y) if act == G.ACT_GELU else None
        _fwd_gemm(col, w, y, b, act, pre)
        ctx.save_for_backward(col, w, y if act == G.ACT_RELU else pre)
        ctx.gw, ctx.gb, ctx.act = gw, gb, act
        ctx.geom = (N, Cin, H, W, kh, kw, stride, pad, OH, OW)
        return y.view(N, OH, OW, Cout)

    @staticmethod
    def backward(ctx, dy):
        col, w, aux = ctx.saved_tensors
        _no_dpsgd("conv2d", ctx.gw, ctx.gb)
        N, Cin, H, W, kh, kw, stride, pad, OH, OW = ctx.geom
        Cout = w.shape[0]
        dy = dy.contiguous().view(-1, Cout)
        rows = dy.shape[0]
        if ctx.act != G.ACT_NONE:
            dz = torch.empty_like(dy)
            C().act_bwd_colsum(dy, aux, dz, ctx.gb, rows, Cout, ctx.act)
        else:
            dz = dy
            if ctx.gb is not None:
                C().act_bwd_colsum(dy, None, None, ctx.gb, rows, Cout, 0)
        if ctx.gw is not None:
            _dw(dz, col, ctx.gw)
        dx = None
        if ctx.needs_input_grad[0] and ctx.need_dx:
            dcol = G.gemm(dz, w, b_mn=True)
            dx = torch.empty(N, H, W, Cin, device=dy.device, dtype=BF)
            C().col2im(dcol, dx, N, Cin, H, W, kh, kw, stride, pad, OH, OW)
        return (dx,) + (None,) * 10


def conv2d(x, w, b, gw, gb, kh, kw, stride=1, pad=0, act=G.ACT_NONE, need_dx=True):
    if conv_is_implicit(x.shape[1], x.shape[2], x.shape[3], kh, kw, stride, pad, w.shape[1]):
        return ConvImplicitFn.apply(x, w, b, gw, gb, kh, kw, stride, pad, act, need_dx)
    return Conv2dFn.apply(x, w, b, gw, gb, kh, kw, stride, pad, act, need_dx)


class BatchNormFn(Function):
    """Channels-last batch norm over [rows, C] with fused (+residual) (+ReLU)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, ggamma, gbeta, run_mean, run_var, training, relu, residual):
        shape = x.shape
        Cc = shape[-1]
        x2 = x.contiguous().view(-1, Cc)
        rows = x2.shape[0]
        y = torch.empty_like(x2)
        if training:
            mean = torch.empty(Cc, device=x.device, dtype=torch.float32)
            rstd = torch.empty_like(mean)
        else:
            mean = run_mean.clone()
            rstd = torch.rsqrt(run_var + 1e-5)
        res2 = residual.contiguous().view(-1, Cc) if residual is not None else None
        C().batchnorm_fwd(x2, y, gamma, beta, mean, rstd, run_mean if training else None,
                          run_var if training else None, rows, Cc, 1e-5, 0.1, training, relu, res2)
        ctx.save_for_backward(x2, y, gamma, mean, rstd)
        ctx.gg, ctx.gb, ctx.relu, ctx.has_res, ctx.shape = ggamma, gbeta, relu, residual is not None, shape
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        x2, y, gamma, mean, rstd = ctx.saved_tensors
        _no_dpsgd("batchnorm", ctx.gg, ctx.gb)
        Cc = x2.shape[1]
        dy2 = dy.contiguous().view(-1, Cc)
        dx = torch.empty_like(x2)
        dres = torch.empty_like(x2) if ctx.has_res else None
        gg = ctx.gg if ctx.gg is not None else torch.zeros(Cc, device=dy.device)
        gb = ctx.gb if ctx.gb is not None else torch.zeros(Cc, device=dy.device)
        C().batchnorm_bwd(dy2, x2, y, gamma, mean, rstd, dx, gg, gb, dres, x2.shape[0], Cc, ctx.relu)
        return (dx.view(ctx.shape), None, None, None, None, None, None, None, None,
                dres.view(ctx.shape) if dres is not None else None)


def batchnorm(x, gamma, beta, ggamma, gbeta, run_mean, run_var, training=True, relu=False,
              residual=None):
    return BatchNormFn.apply(x, gamma, beta, ggamma, gbeta, run_mean, run_var, training, relu, residual)


class MaxPoolFn(Function):
    @staticmethod
    def forward(ctx, x, k, stride, pad):
        x = x.contiguous()
        N, H, W, Cc = x.shape
        OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        y = torch.empty(N, OH, OW, Cc, device=x.device, dtype=BF)
        idx = torch.empty(N, OH, OW, Cc, device=x.device, dtype=torch.int32)
        C().maxpool_fwd(x, y, idx, N, Cc, H, W, k, stride, pad, OH, OW)
        ctx.save_for_backward(idx)
        ctx.in_shape = (N, H, W, Cc)
        return y

    @staticmethod
    def backward(ctx, dy):
        idx, = ctx.saved_tensors
        N, H, W, Cc = ctx.in_shape
        dxf = torch.zeros(N, H, W, Cc, device=dy.device, dtype=torch.float32)
        C().maxpool_bwd(dy.contiguous(), idx, dxf, idx.numel() // N, H * W * Cc)
        dx = torch.empty(N, H, W, Cc, device=dy.device, dtype=BF)
        C().cast_f32_to_bf16(dxf.view(-1), dx.view(-1))
        return dx, None, None, None


def maxpool2d(x, k=2, stride=2, pad=0):
    return MaxPoolFn.apply(x, k, stride, pad)


class GlobalAvgPoolFn(Function):
    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        N, H, W, Cc = x.shape
        y = torch.empty(N, Cc, device=x.device, dtype=BF)
        C().avgpool_fwd(x, y, N, H * W, Cc)
        ctx.shape = (N, H, W, Cc)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, H, W, Cc = ctx.shape
        dx = torch.empty(N, H, W, Cc, device=dy.device, dtype=BF)
        C().avgpool_bwd(dy.contiguous(), dx, N, H * W, Cc)
        return dx


def global_avgpool(x):
    return GlobalAvgPoolFn.apply(x)


class AddFn(Function):
    @staticmethod
    def forward(ctx, a, b):
        a, b = a.contiguous(), b.contiguous()
        out = torch.empty_like(a)
        C().add_bf16(a, b, out)
        return out

    @staticmethod
    def backward(ctx, g):
        return g, g


def add(a, b):
    return AddFn.apply(a, b)


class LayerNormFn(Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, ggamma, gbeta):
        x = x.contiguous()
        rows, Cc = x.shape
        y = torch.empty_like(x)
        mean = torch.empty(rows, device=x.device, dtype=torch.float32)
        rstd = torch.empty_like(mean)
        C().layernorm_fwd(x, y, gamma, beta, mean, rstd, rows, Cc, 1e-12)
        ctx.save_for_backward(x, gamma, mean, rstd)
        ctx.gg, ctx.gb = ggamma, gbeta
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, mean, rstd = ctx.saved_tensors
        _no_dpsgd("layernorm", ctx.gg, ctx.gb)
        rows, Cc = x.shape
        dx = torch.empty_like(x)
        gg = ctx.gg if ctx.gg is not None else torch.zeros(Cc, device=dy.device)
        gb = ctx.gb if ctx.gb is not None else torch.zeros(Cc, device=dy.device)
        C().layernorm_bwd(dy.contiguous(), x, gamma, mean, rstd, dx, gg, gb, rows, Cc)
        return dx, None, None, None, None


def layernorm(x, gamma, beta, ggamma=None, gbeta=None):
    return LayerNormFn.apply(x, gamma, beta, ggamma, gbeta)


class EmbeddingFn(Function):
    @staticmethod
    def forward(ctx, anchor, ids, table, pos, gtable, gpos, seq, pos_ids=None):
        rows, Cc = ids.numel(), table.shape[1]
        out = torch.empty(rows, Cc, device=table.device, dtype=BF)
        C().embedding_fwd(ids, table, pos, out, rows, seq, Cc, pos_ids)
        ctx.save_for_backward(ids, pos_ids)
        ctx.gt, ctx.gp, ctx.seq, ctx.C = gtable, gpos, seq, Cc
        return out

    @staticmethod
    def backward(ctx, dy):
        ids, pos_ids = ctx.saved_tensors
        _no_dpsgd("embedding", ctx.gt, ctx.gp)
        if ctx.gt is not None:
            C().embedding_bwd(ids, dy.contiguous(), ctx.gt, ctx.gp, ids.numel(), ctx.seq, ctx.C, pos_ids)
        return None, None, None, None, None, None, None, None


class DropoutRNG(NamedTuple):
    """Where dropout draws its masks from (csrc/include/philox.hpp).  A mask is a pure function of
    (seed, step, site, coordinates) with step = ``step[0] + add``: ``step`` is an int32 [1] device
    tensor that the kernels read when they run, so a captured CUDA graph draws new masks whenever the
    word changes, and ``add`` a host int (e.g. the mini-batch index).  The backward of a dropout call
    reads the same word as its forward: it must not change in between."""
    seed: int                 # [0, 2^64)
    step: torch.Tensor
    add: int = 0


def _check_dropout(p: float, rng, who: str):
    if not 0.0 <= p < 1.0:
        raise ValueError(f"{who}: dropout_p must lie in [0, 1), got {p}")
    if p > 0.0 and rng is None:
        raise ValueError(f"{who}: dropout_p > 0 needs a DropoutRNG")


def _drop_kw(p: float, rng, site: int) -> dict:
    if p == 0.0:
        return {}
    return dict(dropout_p=float(p), seed=int(rng.seed), step=rng.step, step_add=int(rng.add), site=int(site))


class DropoutAddFn(Function):
    """y = (x +) z * keep / (1 - p); the backward redraws the mask (nothing is saved)."""

    @staticmethod
    def forward(ctx, x, z, p, rng, site, S, seq_ids, pos_ids):
        z = z.contiguous()
        y = torch.empty_like(z)
        C().dropout_add(x.contiguous() if x is not None else None, z, y, S or 0, seq_ids, pos_ids, p, rng.seed,
                        rng.step, rng.add, site)
        ctx.args = (p, rng, site, S or 0, seq_ids, pos_ids)
        ctx.has_x = x is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        p, rng, site, S, seq_ids, pos_ids = ctx.args
        dy = dy.contiguous()
        dz = torch.empty_like(dy)
        C().dropout_add(None, dy, dz, S, seq_ids, pos_ids, p, rng.seed, rng.step, rng.add, site)
        return (dy if ctx.has_x else None), dz, None, None, None, None, None, None


def _check_rows(who: str, S, seq_ids, pos_ids):
    if (seq_ids is None) == (S is None) or (seq_ids is None) != (pos_ids is None):
        raise ValueError(f"{who}: give the row coordinates either as S (row r is position r % S of "
                         f"sequence r // S) or as seq_ids and pos_ids (packed rows)")


def dropout_add(x, z, p: float, rng: Optional[DropoutRNG], site: int, S: Optional[int] = None, seq_ids=None,
                pos_ids=None):
    """x + dropout(z) over [rows, C] bf16 (C % 8 == 0), x None for plain dropout.  Element (r, c) is
    keyed by (sequence, position, c): (r // S, r % S), or (seq_ids[r], pos_ids[r]) for packed rows,
    so a packed batch draws what the same batch right-padded draws.  p == 0 is the plain add."""
    _check_dropout(p, rng, "dropout")
    _check_rows("dropout", S, seq_ids, pos_ids)
    if p == 0.0:
        return z if x is None else add(x, z)
    return DropoutAddFn.apply(x, z, float(p), rng, int(site), S, seq_ids, pos_ids)


def dropout(z, p: float, rng: Optional[DropoutRNG], site: int, S: Optional[int] = None, seq_ids=None, pos_ids=None):
    """z * keep / (1 - p); see ``dropout_add``."""
    return dropout_add(None, z, p, rng, site, S, seq_ids, pos_ids)


def embedding(ids, table, pos, gtable, gpos, seq, pos_ids=None):
    """Word + position embedding of token ids [rows].  Row r takes position ``pos_ids[r]`` (int32
    [rows], e.g. the in-sequence positions of packed sequences), or ``r % seq`` when it is None."""
    # `anchor` makes the output join the autograd graph even though no input is a leaf
    anchor = torch.zeros(1, device=table.device, requires_grad=gtable is not None)
    return EmbeddingFn.apply(anchor, ids, table, pos, gtable, gpos, seq, pos_ids)


class FusedAttentionFn(Function):
    """Multi-head self-attention core on q, k, v of shape [B*S, H*64], heads addressed as TMA boxes
    of the projection outputs so no transpose exists (csrc/kernels/attn_sm100.cu).  Unmasked
    seq_len 128 runs one CTA per (batch, head) with the S x S matrix in registers / smem; any other
    S % 64 == 0 up to 512, a ``lengths`` mask, dropout or ``causal`` runs the tiled online-softmax
    kernels.  ``lengths`` (int32 [B]): sequence b attends to keys j < lengths[b] (right padding).
    ``drop``: keyword arguments of attention-probability dropout (tiled kernels; empty: none).
    ``causal``: query i attends to keys j <= i (not with ``lengths``)."""

    @staticmethod
    def forward(ctx, q, k, v, B, S, H, lengths=None, drop=None, causal=False):
        D = q.shape[1] // H
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        out = torch.empty_like(q)
        lse = torch.empty(B * H * S, device=q.device, dtype=torch.float32)
        drop = drop or {}
        C().attention_fwd(q, k, v, out, lse, B, S, H, 1.0 / (D ** 0.5), lengths, causal=causal, **drop)
        ctx.save_for_backward(q, k, v, out, lse, lengths)
        ctx.dims, ctx.drop, ctx.causal = (B, S, H, D), drop, causal
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse, lengths = ctx.saved_tensors
        B, S, H, D = ctx.dims
        dout = dout.contiguous()
        dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
        whole = lengths is None and S == 128 and not ctx.drop and not ctx.causal
        delta = None if whole else torch.empty_like(lse)
        C().attention_bwd(q, k, v, out, dout, lse, dq, dk, dv, B, S, H, 1.0 / (D ** 0.5), delta, lengths,
                          causal=ctx.causal, **ctx.drop)
        return dq, dk, dv, None, None, None, None, None, None


class PackedAttentionFn(Function):
    """Self-attention over packed variable-length sequences (csrc/kernels/attn_sm100.cu, packed
    mode): q, k, v are [T, H*64] with the real tokens of every sequence concatenated, sequence b
    being rows [cu_seqlens[b], cu_seqlens[b+1]).  No padded row exists, so none is computed or
    written; the lse / delta workspaces are [B*H, S_pad] fp32, S_pad = max_seqlen rounded up to 64."""

    @staticmethod
    def forward(ctx, q, k, v, cu_seqlens, max_seqlen, H, drop=None):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        B, S_pad = cu_seqlens.numel() - 1, (max_seqlen + 63) // 64 * 64
        out = torch.empty_like(q)
        lse = torch.empty(B * H * S_pad, device=q.device, dtype=torch.float32)
        drop = drop or {}
        C().attention_packed_fwd(q, k, v, out, lse, cu_seqlens, max_seqlen, H, 1.0 / 8.0, **drop)
        ctx.save_for_backward(q, k, v, out, lse, cu_seqlens)
        ctx.dims, ctx.drop = (max_seqlen, H), drop
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse, cu_seqlens = ctx.saved_tensors
        max_seqlen, H = ctx.dims
        dout = dout.contiguous()
        dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
        delta = torch.empty_like(lse)
        C().attention_packed_bwd(q, k, v, out, dout, lse, dq, dk, dv, delta, cu_seqlens, max_seqlen, H, 1.0 / 8.0,
                                 **ctx.drop)
        return dq, dk, dv, None, None, None, None


def attention_packed(q, k, v, cu_seqlens, max_seqlen: int, H: int, dropout_p: float = 0.0,
                     rng: Optional[DropoutRNG] = None, site: int = 0, causal: bool = False):
    """Self-attention over packed sequences: q, k, v [T, H*64] bf16, ``cu_seqlens`` int32 [B+1] on
    q's device (cu[0] = 0, cu[B] = T), ``max_seqlen`` (host int in [1, 512]) the longest length.
    Each sequence attends within itself only.  Rows that belong to no sequence are left unwritten.
    ``dropout_p`` > 0 drops attention probabilities as ``attention`` does, with the same masks.
    There is no causal form of the packed kernels: ``causal=True`` raises ValueError."""
    if causal:
        raise ValueError("attention_packed: the packed kernels have no causal mask (use attention(..., causal=True) "
                         "on right-padded batches without lengths)")
    _check_dropout(dropout_p, rng, "attention_packed")
    if q.shape[1] != 64 * H:
        raise ValueError(f"attention_packed: head dim must be 64; got {q.shape[1]} columns for {H} heads")
    if not 1 <= max_seqlen <= 512:
        raise ValueError(f"attention_packed: max_seqlen {max_seqlen} outside [1, 512]")
    return PackedAttentionFn.apply(q, k, v, cu_seqlens, int(max_seqlen), H, _drop_kw(dropout_p, rng, site))


class AttentionFn(Function):
    """Unfused, mask-free fallback for shapes the fused kernels do not cover (head dim != 64, or
    seq_len not a multiple of 64 in [64, 512]), and for fused=False:
    batched wgmma GEMMs + row-softmax kernel + head transposes."""

    @staticmethod
    def forward(ctx, q, k, v, B, S, H):
        D = q.shape[1] // H
        m = C()

        def heads(t):
            o = torch.empty(B * H, S, D, device=t.device, dtype=BF)
            m.transpose_0213(t.contiguous(), o, B, S, H, D)
            return o

        qh, kh, vh = heads(q), heads(k), heads(v)
        scores = G.gemm(qh, kh)                                   # [BH, S, S]
        probs = torch.empty_like(scores)
        m.softmax_fwd(scores, probs, B * H * S, S, 1.0 / (D ** 0.5))
        ctxh = G.gemm(probs, vh, b_mn=True)                       # [BH, S, D]
        out = torch.empty(B * S, H * D, device=q.device, dtype=BF)
        m.transpose_0213(ctxh, out, B, H, S, D)
        ctx.save_for_backward(qh, kh, vh, probs)
        ctx.dims = (B, S, H, D)
        return out

    @staticmethod
    def backward(ctx, dout):
        qh, kh, vh, probs = ctx.saved_tensors
        B, S, H, D = ctx.dims
        m = C()
        doh = torch.empty(B * H, S, D, device=dout.device, dtype=BF)
        m.transpose_0213(dout.contiguous(), doh, B, S, H, D)
        dv = G.gemm(probs, doh, a_mn=True, b_mn=True)             # P^T dO   [BH, S, D]
        dp = G.gemm(doh, vh)                                      # dO V^T   [BH, S, S]
        ds = torch.empty_like(dp)
        m.softmax_bwd(dp, probs, ds, B * H * S, S, 1.0 / (D ** 0.5))
        dq = G.gemm(ds, kh, b_mn=True)                            # dS K     [BH, S, D]
        dk = G.gemm(ds, qh, a_mn=True, b_mn=True)                 # dS^T Q   [BH, S, D]

        def unheads(t):
            o = torch.empty(B * S, H * D, device=t.device, dtype=BF)
            m.transpose_0213(t, o, B, H, S, D)
            return o

        return unheads(dq), unheads(dk), unheads(dv), None, None, None


def fused_attention_supported(S: int, D: int) -> bool:
    return D == 64 and S % 64 == 0 and 64 <= S <= 512


def attention(q, k, v, B, S, H, fused: bool = True, lengths=None, dropout_p: float = 0.0,
              rng: Optional[DropoutRNG] = None, site: int = 0, causal: bool = False):
    """Self-attention over q, k, v of shape [B*S, H*D].  ``lengths`` (int32 [B] on q's device, or
    None): right-padding key mask, only on the fused kernels (D == 64, S % 64 == 0, 64 <= S <= 512).
    Query rows past a sequence's length are still computed, as scaled_dot_product_attention does;
    a length <= 0 gives zero output rows.

    ``dropout_p`` > 0 (with ``rng`` and a ``site`` id) drops attention probabilities inside the
    tiled fused kernels: O = (P * keep / (1 - p)) V, the keep mask keyed by (b, h, i, j); unmasked
    S == 128 then runs the tiled kernels too.  Only on the fused kernels.

    ``causal=True``: query row i attends to keys j <= i (a decoder), on the tiled fused kernels only
    (S == 128 included), which skip the key blocks above the diagonal.  Not with ``lengths``."""
    _check_dropout(dropout_p, rng, "attention")
    ok = fused_attention_supported(S, q.shape[1] // H)
    if causal and lengths is not None:
        raise ValueError("attention: causal=True takes no lengths mask (causal attention runs on unpadded batches)")
    if causal and not (fused and ok):
        raise ValueError(f"attention: causal=True needs the fused kernels (head dim 64, seq_len a multiple of 64 "
                         f"in [64, 512]); got S={S}, fused={fused}")
    if lengths is not None and not (fused and ok):
        raise ValueError(f"attention: a lengths mask needs the fused kernels (head dim 64, "
                         f"seq_len a multiple of 64 in [64, 512]); got S={S}, fused={fused}")
    if dropout_p > 0.0 and not (fused and ok):
        raise ValueError(f"attention: dropout needs the fused kernels (head dim 64, seq_len a multiple of 64 "
                         f"in [64, 512]); got S={S}, fused={fused}")
    if fused and ok:
        return FusedAttentionFn.apply(q, k, v, B, S, H, lengths, _drop_kw(dropout_p, rng, site), bool(causal))
    return AttentionFn.apply(q, k, v, B, S, H)
