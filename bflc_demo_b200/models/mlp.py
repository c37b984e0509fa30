"""2-layer MLP 784 -> hidden -> 62 (BASELINE.json configs #1/#2), hand-scheduled: every
forward/backward GEMM is the wgmma kernel with a fused epilogue, the whole training step
is six launches and is CUDA-graph capturable (no host syncs, no allocations).

Reference parity: the reference's model is the degenerate single-layer case
``pred = x @ W + b`` with softmax-cross-entropy and plain SGD, batch 100, one pass per
round (python-sdk/main.py:109-148); ``SoftmaxRegression`` below is exactly that model.

  step(x, y):
    1. h       = relu(x @ W1^T + b1)                    GEMM  (bias+ReLU epilogue)
    2. dlogits = softmax(h @ W2^T + b2) - onehot(y)     GEMM  (xent epilogue: loss, #correct,
                                                              db2 column sums)
    3. dW2     = dlogits^T @ h                          GEMM  (MN-major A and B, split-K)
    4. dh      = (dlogits @ W2) * (h > 0)               GEMM  (MN-major B, ReLU-bwd mask, db1)
    5. dW1     = dh^T @ x                               GEMM  (MN-major A and B, split-K)
    6. SGD / Adam over the flat buffer (+ bf16 shadow refresh + grad zeroing)
"""
from __future__ import annotations

from typing import Optional

import torch

from .._native import C
from ..engine.base import step_rows
from ..ops import gemm as G
from .flat import ParamSpec


def sf_bytes(rows: int, K: int) -> int:
    """Bytes of the MXFP8 scale-chunk array of a [rows, K] operand: one 512-byte chunk per
    (128 rows, 128 K) -- csrc/include/epi_common.cuh."""
    return -(-rows // 128) * -(-K // 128) * 512


def mlp_spec(in_dim: int = 784, hidden: int = 256, n_classes: int = 62) -> ParamSpec:
    return ParamSpec([("w1", (hidden, in_dim)), ("b1", (hidden,)),
                      ("w2", (n_classes, hidden)), ("b2", (n_classes,))])


CHAIN_CLASSES = range(57, 65)   # the fused chain's 64 padded classes: ncp = (C + 7) // 8 * 8 == 64


def check_chain_shapes(in_dim: int, hidden: int, n_classes: int, batch: int, *, fp8: bool = False,
                       dpsgd: bool = False, prox: bool = False, device=None) -> None:
    """Refuses, before anything launches, the shapes the persistent trainer runs neither with DP-SGD nor
    in fp8: both need the fused chain (phase plans 3 / 4), whose tiles are hidden 256 wide and 64 classes
    wide, so 57..64 classes.  DP-SGD also needs plan 4, whose 4-CTA clusters must all be resident at once;
    only the launcher's plan decision (``mlp_round_plan``, on ``device``) knows how many the device holds."""
    if not (fp8 or dpsgd):
        return
    what = "DP-SGD in the persistent trainer" if dpsgd else "dtype fp8 (MXFP8)"
    if hidden != 256 or n_classes not in CHAIN_CLASSES:
        raise ValueError(f"{what} needs hidden == 256 and 57..64 classes, the fused chain's 64 padded columns "
                         f"(got hidden {hidden}, {n_classes} classes)")
    if dpsgd:
        with torch.cuda.device(device if device is not None else torch.cuda.current_device()):
            plan = C().mlp_round_plan(batch, in_dim, hidden, n_classes, fp8=fp8, dpsgd=True, prox=prox)
        if not plan["ok"]:
            raise ValueError(f"{what} runs in phase plan 4 only, and this device cannot run batch {batch} at "
                             f"in_dim {in_dim} in it: its grid of 4-CTA clusters exceeds the SMs or the "
                             f"clusters the device holds at once ({plan['error']})")


def softmax_regression_spec(n_features: int = 5, n_class: int = 2) -> ParamSpec:
    """The reference model: W[n_features, n_class] stored [out, in] + b (H:7-8, M:113-120)."""
    return ParamSpec([("w", (n_class, n_features)), ("b", (n_class,))])


class FlatMLP:
    """Fused-kernel trainer over flat buffers.  ``master``/``shadow``/``grad`` are 1-D tensors
    of ``spec.total`` elements (fp32 / bf16 / fp32); they may live in the symmetric heap."""

    def __init__(self, spec: ParamSpec, master: torch.Tensor, shadow: torch.Tensor,
                 grad: torch.Tensor, batch: int, *, optimizer: str = "sgd", lr: float = 1e-3,
                 loss_sum: Optional[torch.Tensor] = None, correct: Optional[torch.Tensor] = None,
                 step_dev_ptr: int = 0, fp8: bool = False, prox_mu: float = 0.0,
                 anchor: Optional[torch.Tensor] = None, dpsgd_clip: float = 0.0, dpsgd_noise: float = 0.0,
                 dpsgd_seed: int = 0):
        """``prox_mu`` > 0 (FedProx): every step adds ``prox_mu * (w - anchor)`` to the gradient;
        ``anchor`` is an fp32 tensor like ``master``, the global model the round started from.

        ``dpsgd_clip`` > 0: DP-SGD in the persistent trainer (``train_epoch_fused`` only, phase plan 4 with
        the optimizer in the epilogue, hidden 256, 57..64 classes, a batch whose plan-4 grid the device holds
        as resident 4-CTA clusters; ``check_chain_shapes``): each example's gradient is clipped
        to a certified bound of ``dpsgd_clip`` and each step's averaged gradient gets Gaussian noise of
        standard deviation ``noise_sigma(dpsgd_noise, dpsgd_clip, batch)``, keyed by ``dpsgd_seed`` and the
        step word at ``step_dev_ptr`` plus the step index, as ``ops.dpsgd`` releases it.  x must be finite
        (the engine converts it from u8): only the h row of an example with a non-finite bound is masked.
        ``dpsgd_dropped`` counts such examples; ``dpsgd_dbg`` (None; a test hook) receives the per-row
        sq0, sq1, ab0, ab1 and c of every step, then the last step's released gradient.

        ``fp8`` and DP-SGD both refuse, with a ValueError, the shapes the launcher cannot run them at."""
        if prox_mu > 0 and anchor is None:
            raise ValueError("prox_mu > 0 needs the anchor (the round's global model)")
        hidden, in_dim = spec.by_name["w1"].shape
        check_chain_shapes(in_dim, hidden, spec.by_name["w2"].shape[0], batch, fp8=fp8, dpsgd=dpsgd_clip > 0,
                           prox=prox_mu > 0, device=master.device)
        self.spec, self.master, self.shadow, self.grad = spec, master, shadow, grad
        self.prox_mu = float(prox_mu)
        self.anchor = anchor if prox_mu > 0 else None
        self.p = spec.views(master)
        self.s = spec.views(shadow)
        self.g = spec.views(grad)
        self.hidden, self.in_dim = spec.by_name["w1"].shape
        self.n_classes = spec.by_name["w2"].shape[0]
        self.batch = batch
        dev = master.device
        self.h = torch.empty(batch, self.hidden, device=dev, dtype=torch.bfloat16)
        self.dh = torch.empty(batch, self.hidden, device=dev, dtype=torch.bfloat16)
        self.ncp = (self.n_classes + 7) // 8 * 8          # dlogits row stride (TMA alignment)
        self.dlogits = torch.zeros(batch, self.ncp, device=dev, dtype=torch.bfloat16)
        self.loss_sum = loss_sum if loss_sum is not None else torch.zeros(1, device=dev)
        self.correct = correct if correct is not None else torch.zeros(1, device=dev, dtype=torch.int32)
        self.optimizer, self.lr = optimizer, lr
        self.m = torch.zeros_like(master) if optimizer == "adam" else None
        self.v = torch.zeros_like(master) if optimizer == "adam" else None
        self.step_dev_ptr = step_dev_ptr
        # weight-gradient GEMMs reduce over the batch: split the reduction only when it is long
        k_blocks = (batch + 63) // 64
        self.split_k = 1 if k_blocks <= 16 else max(1, min(8, k_blocks // 8))
        self.side = torch.cuda.Stream(device=dev)
        self._ev_fork = torch.cuda.Event()
        self._ev_join = torch.cuda.Event()
        # block-scaled fp8 forward (persistent trainer only): this trainer's quantised weights (an
        # Mx8MlpLayout blob, refreshed by the optimizer epilogue), their exactly dequantised bf16
        # copy work_dq (W1 [hidden, in_dim] | W2 [64, hidden], rows >= n_classes zero) that the
        # forward GEMMs read, and the per-step dequantised e4m3 h
        self.fp8 = bool(fp8)
        self.ql = C().mx8_mlp_layout(self.in_dim, self.hidden) if self.fp8 else None
        self._x_dq: Optional[torch.Tensor] = None
        if self.fp8:
            self.work_q = torch.zeros(self.ql["total"], device=dev, dtype=torch.uint8)
            self.work_dq = torch.zeros(self.hidden * self.in_dim + 64 * self.hidden, device=dev,
                                       dtype=torch.bfloat16)
            self.h_dq = torch.zeros(batch, self.hidden, device=dev, dtype=torch.bfloat16)
        self.dpsgd_clip = float(dpsgd_clip)
        self.dpsgd_dbg: Optional[torch.Tensor] = None
        if self.dpsgd_clip > 0:
            import numpy as np
            from ..ops.dpsgd import noise_sigma
            clip32, noise32 = np.float32(dpsgd_clip), np.float32(dpsgd_noise)
            if not (np.isfinite(clip32) and clip32 > 0 and np.isfinite(noise32) and noise32 >= 0):
                raise ValueError(f"DP-SGD needs a finite clip > 0 and a finite noise >= 0 (fp32); got clip "
                                 f"{dpsgd_clip}, noise {dpsgd_noise}")
            self.dpsgd_sigma = float(noise_sigma(noise32, clip32, batch))
            self.dpsgd_seed = int(dpsgd_seed) % (1 << 64)
            self.dpsgd_dropped = torch.zeros(1, device=dev, dtype=torch.int32)
            # 32-row column sums of the clipped dh | dlogits rows per 64-row M-tile, summed in M-tile order
            self.dpsgd_ws = torch.zeros(2 * (-(-batch // 64)), self.hidden + 64, device=dev, dtype=torch.float32)

    # -------------------------------------------------------------- training
    def forward_backward(self, x: torch.Tensor, y: torch.Tensor) -> None:
        """x: bf16 [batch, in_dim], y: int32 [batch].  Accumulates grads into ``grad``."""
        B = x.shape[0]
        s, g = self.s, self.g
        h = self.h[:B]
        G.gemm(x, s["w1"], out=h, bias=self.p["b1"], act=G.ACT_RELU)
        dl = self.dlogits[:B]
        G.gemm_xent(h, s["w2"], y, n_classes=self.n_classes, bias=self.p["b2"], dlogits=dl,
                    grad_scale=1.0 / B, loss_sum=self.loss_sum, correct=self.correct,
                    colsum=g["b2"])
        # dW2 and dh are independent (both only read dlogits, h, W2): dW2 runs on a side stream
        # (a parallel branch of the captured graph) while dh -> dW1 stay on the main stream.
        main = torch.cuda.current_stream()
        self._ev_fork.record(main)
        self.side.wait_event(self._ev_fork)
        with torch.cuda.stream(self.side):
            # dW2[c, j] = sum_b dlogits[b, c] h[b, j]
            G.gemm(dl[:, :self.n_classes], h, out=g["w2"], a_mn=True, b_mn=True,
                   split_k=self.split_k)
            self._ev_join.record(self.side)
        # dh = (dlogits @ W2) * relu'(h);  db1 = colsum(dh)
        G.gemm(dl[:, :self.n_classes], s["w2"], out=self.dh[:B], b_mn=True, aux_in=h, act_bwd=1,
               colsum=g["b1"])
        # dW1 = dh^T @ x
        G.gemm(self.dh[:B], x, out=g["w1"], a_mn=True, b_mn=True, split_k=self.split_k)
        main.wait_event(self._ev_join)

    def optimizer_step(self, step_in_round: int = 1) -> None:
        if self.prox_mu > 0:
            # the recipe kernel with the default recipe is optim_step bit for bit, plus the term
            C().optim_recipe_step(self.optimizer == "adam", self.master, self.grad, self.shadow, self.m, self.v,
                                  self.lr, 0.9, 0.999, 1e-8, step_in_round, self.step_dev_ptr, 0.0, None, 0, 0, 0,
                                  None, anchor=self.anchor, prox_mu=self.prox_mu)
            return
        C().optim_step(self.optimizer == "adam", self.master, self.grad, self.shadow, self.m,
                       self.v, self.lr, 0.0, 0.9, 0.999, 1e-8, step_in_round, self.step_dev_ptr, 0,
                       True)

    def train_epoch(self, X: torch.Tensor, Y: torch.Tensor, steps: int, epoch_rows: int = 0) -> None:
        """``steps`` mini-batches of ``batch`` rows, remainder dropped (M:141-148).  ``epoch_rows`` (default
        steps * batch): the rows of one local epoch; step i reads ``engine.base.step_rows(i, batch,
        epoch_rows)``, so later epochs repeat the first one's batches."""
        if self.dpsgd_clip > 0:
            raise ValueError("DP-SGD runs in the persistent trainer only (train_epoch_fused); the per-GEMM "
                             "step has no per-example clipping")
        B = self.batch
        epoch_rows = epoch_rows or steps * B
        if epoch_rows % B or not B <= epoch_rows <= min(X.shape[0], Y.shape[0]):
            raise ValueError(f"train_epoch: an epoch of {epoch_rows} rows in batches of {B} over "
                             f"{X.shape[0]} / {Y.shape[0]} rows of x / y")
        for i in range(steps):
            rows = step_rows(i, B, epoch_rows)
            self.forward_backward(X[rows], Y[rows])
            self.optimizer_step(i + 1)

    def fused_ok(self, steps: int) -> bool:
        """Shape limits of the persistent one-launch trainer (csrc/kernels/mlp_round_sm100.cu)."""
        B, H, D = self.batch, self.hidden, self.in_dim
        mt_b, nt_h, nt_d, mt_h = -(-B // 128), -(-H // 64), -(-D // 64), -(-H // 128)
        need = max(mt_b * nt_h, mt_h * nt_d + nt_h + 1)
        return (need <= 128 and B % 8 == 0 and H % 8 == 0 and D % 8 == 0 and self.n_classes <= 64)

    def offsets(self):
        e = self.spec.by_name
        return [e["w1"].offset, e["b1"].offset, e["w2"].offset, e["b2"].offset]

    def quantize_weights(self, master: Optional[torch.Tensor] = None,
                         blob: Optional[torch.Tensor] = None) -> torch.Tensor:
        """fp32 master weights -> MXFP8 blob (e4m3 + UE8M0 scale chunks + fp32 biases), plus the
        dequantised ``work_dq`` copy when the blob is this trainer's own.  Run at the start of
        every round: the consensus kernel has just rewritten the training buffers."""
        dq = self.work_dq if blob is None else None
        blob = self.work_q if blob is None else blob
        C().quantize_mlp_blob(self.master if master is None else master, self.offsets(), self.in_dim,
                              self.hidden, self.n_classes, blob, dq)
        return blob

    def train_epoch_fused(self, X: torch.Tensor, Y: torch.Tensor, steps: int,
                          barrier_ptr: int, dbg: Optional[torch.Tensor] = None, plan: int = -1,
                          epiopt: int = -1, x_ready_ptr: int = 0, round_seq_ptr: int = 0,
                          x_q: Optional[torch.Tensor] = None, x_sf: Optional[torch.Tensor] = None,
                          x_dq: Optional[torch.Tensor] = None, fed: Optional[dict] = None, upq_off=(), n_samples: int = 0,
                          n_loss_terms: int = 0, byz_mode: int = 0, byz_scale: float = 0.0,
                          straggle_us: int = 0, epoch_rows: int = 0) -> None:
        """All ``steps`` mini-batch steps in ONE persistent kernel launch; ``barrier_ptr`` is a
        device uint32 that is zero on entry (the phase barrier).  ``dbg``: optional int64
        [steps, 32] buffer that receives %globaltimer phase stamps of CTA 0.  ``plan`` /
        ``epiopt`` pick a phase plan explicitly (0 | 3 | 4, 0 | 1; -1 = BFLC_MLP_CHAIN /
        BFLC_MLP_EPIOPT / default 4, 1) -- all plans are numerically equivalent.  0: fwd1, xent and
        dh as separate phases (any hidden size); 3: fwd1, then fwd2 -> xent -> dh chained per
        128-row tile on four CTAs; 4: as 3, with fwd1 and the chain of a tile in one 4-CTA
        cluster that hands h over on chip.  3 and 4 need hidden = 256 and fall back to 0
        otherwise.  ``x_ready_ptr`` /
        ``round_seq_ptr`` (device uint32[steps] / uint32): the producer of step s waits until
        ``x_ready[s] >= *round_seq`` (input pipeline, engine/fused.py).

        ``x_dq`` (fp8 trainers): the dequantised MXFP8 copy of X (``prep_inputs(..., dst_dq=)``);
        fwd1 / fwd2 then multiply MXFP8 operands as bf16 wgmma on exactly dequantised copies.  Given
        only ``x_q`` / ``x_sf`` (e4m3 + scale chunks), x_dq is derived from them by one dequantise
        kernel.  ``fed`` (+ ``upq_off``,
        ``n_samples``, ...): fuse UploadLocalUpdate into the last step (the optimizer epilogue
        writes the upload buffers, CTA 0 releases FLAG_TRAINED on every peer).  ``epoch_rows``
        (default steps * batch): the rows of one local epoch, E * batch; step s reads batch s mod E
        (``engine.base.step_rows``) and waits on ``x_ready[s mod E]``."""
        dp = {}
        if self.dpsgd_clip > 0:
            if plan not in (-1, 4) or epiopt == 0:
                raise ValueError(f"DP-SGD runs in phase plan 4 with the optimizer in the epilogue (got plan {plan}, "
                                 f"epiopt {epiopt})")
            dp = dict(dpsgd_clip=self.dpsgd_clip, dpsgd_sigma=self.dpsgd_sigma, dpsgd_seed=self.dpsgd_seed,
                      dpsgd_dropped=self.dpsgd_dropped, dpsgd_ws=self.dpsgd_ws, dpsgd_dbg=self.dpsgd_dbg)
        if self.fp8 and x_dq is None:
            assert x_q is not None and x_sf is not None, "fp8 trainer needs x_dq, or x_q and x_sf"
            if self._x_dq is None or self._x_dq.shape != x_q.shape:
                self._x_dq = torch.empty(x_q.shape, device=x_q.device, dtype=torch.bfloat16)
            C().mx8_dequant(x_q, x_sf, self._x_dq)
            x_dq = self._x_dq
        C().mlp_round(X, Y, self.master, self.shadow, self.grad, self.offsets(), self.h, self.dlogits,
                      self.dh, self.loss_sum, self.correct, barrier_ptr, self.batch, steps,
                      self.in_dim, self.hidden, self.n_classes, self.lr,
                      self.optimizer == "adam", self.m, self.v, self.step_dev_ptr, dbg, plan, epiopt,
                      x_ready_ptr, round_seq_ptr,
                      x_dq if self.fp8 else None, self.work_q if self.fp8 else None,
                      self.work_dq if self.fp8 else None, self.h_dq if self.fp8 else None,
                      fed, list(upq_off), n_samples, n_loss_terms,
                      byz_mode, byz_scale, straggle_us, self.anchor, self.prox_mu, epoch_rows, **dp)

    # ------------------------------------------------------------ evaluation
    def accuracy_counts(self, X: torch.Tensor, Y: torch.Tensor, shadow: Optional[torch.Tensor] = None,
                        master: Optional[torch.Tensor] = None) -> torch.Tensor:
        """#correct of (optionally another model's) weights on (X, Y) -> int32 [1] (K6)."""
        s = self.spec.views(shadow) if shadow is not None else self.s
        p = self.spec.views(master) if master is not None else self.p
        n = X.shape[0]
        h = torch.empty(n, self.hidden, device=X.device, dtype=torch.bfloat16)
        G.gemm(X, s["w1"], out=h, bias=p["b1"], act=G.ACT_RELU)
        cnt = torch.zeros(1, device=X.device, dtype=torch.int32)
        G.gemm_argmax_acc(h, s["w2"], Y, cnt, n_classes=self.n_classes, bias=p["b2"])
        return cnt


def torch_reference_step(params: dict, x: torch.Tensor, y: torch.Tensor, lr: float):
    """Plain fp32 PyTorch version of one SGD step of the same MLP (numerics oracle)."""
    w1, b1, w2, b2 = (params[k].detach().clone().requires_grad_(True) for k in ("w1", "b1", "w2", "b2"))
    h = torch.relu(x.float() @ w1.t() + b1)
    logits = h @ w2.t() + b2
    loss = torch.nn.functional.cross_entropy(logits, y.long())
    loss.backward()
    new = {k: (t - lr * t.grad).detach() for k, t in (("w1", w1), ("b1", b1), ("w2", w2), ("b2", b2))}
    grads = {"w1": w1.grad, "b1": b1.grad, "w2": w2.grad, "b2": b2.grad}
    return loss.detach(), new, grads
