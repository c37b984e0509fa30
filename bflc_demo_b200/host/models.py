"""Plain-PyTorch (CPU or any device) models for the host path, expressed over ONE flat fp32
weight vector so an update is a single array (the reference's ``delta_model`` dict of nested
lists, python-sdk/main.py:153-157, flattened).

``softmax`` is exactly the reference model: ``pred = x @ W + b``, mean softmax-cross-entropy,
``GradientDescentOptimizer(lr)``, batch 100, one pass, remainder dropped (M:109-148);
accuracy = mean(argmax == argmax) (M:182-183)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from ..models.flat import ParamSpec
from ..models.mlp import mlp_spec, softmax_regression_spec


@dataclass
class HostDPSGD:
    """DP-SGD of a host client (ops/dpsgd.py states the definition): clip norm, noise multiplier, the
    client's noise key and its optimizer-step count, which keys each step's noise and advances by one
    per local step."""
    clip: float
    noise: float
    seed: int
    step: int = 0


class HostModel:
    def __init__(self, kind: str, in_dim: int, n_classes: int, hidden: int = 256,
                 scale_inputs: float = 1.0):
        self.kind = kind
        self.spec: ParamSpec = (softmax_regression_spec(in_dim, n_classes) if kind == "softmax"
                                else mlp_spec(in_dim, hidden, n_classes))
        self.size = self.spec.total
        self.scale = scale_inputs

    def init(self, seed: int = 0, zeros: bool = False) -> torch.Tensor:
        w = torch.zeros(self.size)
        if not zeros:
            self.spec.init_(w, seed=seed)
        return w

    def _logits(self, p: dict, x: torch.Tensor) -> torch.Tensor:
        x = x.float() * self.scale
        if self.kind == "softmax":
            return x @ p["w"].t() + p["b"]
        h = torch.relu(x @ p["w1"].t() + p["b1"])
        return h @ p["w2"].t() + p["b2"]

    def dpsgd_grad(self, w: torch.Tensor, xb: torch.Tensor, yb: torch.Tensor, dp: HostDPSGD) -> torch.Tensor:
        """One DP-SGD step's gradient, (1 / B) (sum_n c_n grad l_n + z C xi), from per-example fp32
        autograd: c_n = min(1, C / ||grad l_n||), 0 for a non-finite norm; xi_i = dp_gauss(seed, step, i,
        DPSGD_SITE) over every coordinate; no noise kernel at z = 0.  Advances ``dp.step``."""
        from ..protocol.oracle import DPSGD_SITE, dp_gauss
        from torch.func import grad, vmap

        def one(wv, x, t):
            return torch.nn.functional.cross_entropy(self._logits(self.spec.views(wv), x[None]), t[None].long())

        g = vmap(grad(one), in_dims=(None, 0, 0))(w.detach(), xb, yb)          # [B, P]
        with torch.no_grad():
            n = torch.linalg.vector_norm(g, dim=1)
            c = torch.where(torch.isfinite(n), torch.clamp(dp.clip / n, max=1.0), torch.zeros_like(n))
            out = (c[:, None] * torch.nan_to_num(g, nan=0.0, posinf=0.0, neginf=0.0)).sum(0)
            if dp.noise > 0:
                xi = torch.from_numpy(dp_gauss(dp.seed, dp.step & 0xFFFFFFFF, 0, w.numel(), DPSGD_SITE))
                out = out + float(np.float32(dp.noise) * np.float32(dp.clip)) * xi
        dp.step += 1
        return out / xb.shape[0]

    def train_pass(self, w: torch.Tensor, X: torch.Tensor, y: torch.Tensor, lr: float,
                   batch: int, epochs: int = 1, prox_mu: float = 0.0,
                   dpsgd: Optional[HostDPSGD] = None) -> Tuple[torch.Tensor, float, int]:
        """-> (new weights, avg_cost over the batches, n_samples seen). One SGD step per batch.
        ``prox_mu`` > 0 (FedProx): each step adds ``prox_mu * (w - w_start)`` to the batch gradient,
        ``w_start`` the weights passed in (the global model); avg_cost stays the data loss.
        ``dpsgd``: each step's batch gradient is the DP-SGD gradient (``dpsgd_grad``) instead."""
        w_old = w.detach().clone()
        w = w.clone().requires_grad_(True)
        n_batches = X.shape[0] // batch
        if n_batches == 0:
            n_batches, batch = 1, X.shape[0]
        cost = 0.0
        for _ in range(epochs):
            for i in range(n_batches):
                xb, yb = X[i * batch:(i + 1) * batch], y[i * batch:(i + 1) * batch]
                loss = torch.nn.functional.cross_entropy(self._logits(self.spec.views(w), xb), yb.long())
                g = self.dpsgd_grad(w, xb, yb, dpsgd) if dpsgd is not None else torch.autograd.grad(loss, w)[0]
                if prox_mu > 0:
                    g = g + prox_mu * (w.detach() - w_old)
                with torch.no_grad():
                    w -= lr * g
                cost += float(loss.detach()) / (n_batches * epochs)
        return w.detach(), cost, int(X.shape[0])

    @torch.no_grad()
    def accuracy(self, w: torch.Tensor, X: torch.Tensor, y: torch.Tensor) -> float:
        pred = self._logits(self.spec.views(w), X).argmax(1)
        return float((pred == y.long()).float().mean())
