"""Plain-PyTorch (CPU or any device) models for the host path, expressed over ONE flat fp32
weight vector so an update is a single array (the reference's ``delta_model`` dict of nested
lists, python-sdk/main.py:153-157, flattened).

``softmax`` is exactly the reference model: ``pred = x @ W + b``, mean softmax-cross-entropy,
``GradientDescentOptimizer(lr)``, batch 100, one pass, remainder dropped (M:109-148);
accuracy = mean(argmax == argmax) (M:182-183)."""
from __future__ import annotations

from typing import Tuple

import torch

from ..models.flat import ParamSpec
from ..models.mlp import mlp_spec, softmax_regression_spec


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

    def train_pass(self, w: torch.Tensor, X: torch.Tensor, y: torch.Tensor, lr: float,
                   batch: int, epochs: int = 1, prox_mu: float = 0.0) -> Tuple[torch.Tensor, float, int]:
        """-> (new weights, avg_cost over the batches, n_samples seen). One SGD step per batch.
        ``prox_mu`` > 0 (FedProx): each step adds ``prox_mu * (w - w_start)`` to the batch gradient,
        ``w_start`` the weights passed in (the global model); avg_cost stays the data loss."""
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
                g, = torch.autograd.grad(loss, w)
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
