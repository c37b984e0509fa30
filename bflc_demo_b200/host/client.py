"""Client runtime: the role loop of ``run_one_node`` and the sponsor of ``run_sponsor``
(python-sdk/main.py:84-276, 280-340) against any object exposing the six ledger methods
(local C++ ``Ledger``, gloo-replicated ledger, or the RPC proxy).

Fixed reference defects (SURVEY.md 2.2): ``trained_epoch`` only advances when the ledger
accepted the upload (M:162-163 vs C:239-244); a failed call does not leave a dead client in
the loop (M:165-167); the sponsor owns its client handle (M:340)."""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import numpy as np
import torch

from ..data.synthetic import Shard
from .models import HostDPSGD, HostModel

ROLE_TRAINER, ROLE_COMM = 1, 2


def _status_ok(s) -> bool:
    name = getattr(s, "name", None) or str(s)
    return name in ("OK", "AGGREGATED") or s in (0, 8)


@dataclass
class Client:
    node_id: int
    ledger: object
    shard: Shard
    model: HostModel
    lr: float = 0.001
    batch_size: int = 100
    max_epoch: int = 1000
    byzantine: bool = False
    byzantine_scale: float = 5.0
    prox_mu: float = 0.0              # FedProx: proximal term toward the round's global model
    dpsgd: Optional[HostDPSGD] = None  # DP-SGD local training (this client's key and step count)
    trained_epoch: int = -1
    registered: bool = False
    log: Optional[Callable[[str], None]] = None
    stats: Dict[str, int] = field(default_factory=lambda: dict(trained=0, scored=0, rejected=0))

    def _say(self, msg: str):
        if self.log:
            self.log(f"node_{self.node_id} {msg}")

    # P6 local_training (M:103-169)
    def local_training(self) -> bool:
        w_old, epoch = self.ledger.QueryGlobalModel()
        w_old = torch.as_tensor(np.asarray(w_old), dtype=torch.float32)
        w_new, avg_cost, n = self.model.train_pass(w_old, self.shard.x, self.shard.y, self.lr,
                                                   self.batch_size, prox_mu=self.prox_mu, dpsgd=self.dpsgd)
        delta = (w_old - w_new) / self.lr
        if self.byzantine:  # fault injection: sign-flipped, scaled update
            delta = -self.byzantine_scale * delta
        st = self.ledger.UploadLocalUpdate(self.node_id, delta.numpy(), n, float(avg_cost), epoch)
        if _status_ok(st):
            self.trained_epoch = epoch
            self.stats["trained"] += 1
            return True
        name = getattr(st, "name", str(st))
        if name in ("QUOTA_FULL", "DUPLICATE", "NOT_TRAINER"):
            self.trained_epoch = epoch  # nothing more to do this round
        self.stats["rejected"] += 1
        return False

    # P8 local_scoring (M:196-228) with P7 local_testing on the member's own shard (M:191)
    def local_scoring(self) -> bool:
        updates = self.ledger.QueryAllUpdates()
        if len(updates) == 0:
            return False
        w_g, epoch = self.ledger.QueryGlobalModel()
        w_g = torch.as_tensor(np.asarray(w_g), dtype=torch.float32)
        scores = {}
        for u in updates:
            cand = w_g - self.lr * torch.as_tensor(np.asarray(u["delta"]), dtype=torch.float32)
            scores[int(u["sender"])] = self.model.accuracy(cand, self.shard.x, self.shard.y)
        st = self.ledger.UploadScores(self.node_id, epoch, scores)
        if _status_ok(st):
            self.trained_epoch = epoch
            self.stats["scored"] += 1
            return True
        return False

    # P10 main_loop body (M:243-265): one poll.  Returns "done" | "idle" | "trained" | "scored"
    def poll(self) -> str:
        if not self.registered:
            self.ledger.RegisterNode(self.node_id)
            self.registered = True
            self._say("registered successfully")
        role, epoch = self.ledger.QueryState(self.node_id)
        if epoch > self.max_epoch:
            return "done"
        if epoch <= self.trained_epoch:
            return "idle"
        did = "idle"
        if role & ROLE_TRAINER:
            if self.local_training():
                did = "trained"
        if role & ROLE_COMM:
            if self.local_scoring():
                did = "scored"
        return did


@dataclass
class Sponsor:
    """P11: polls the global model and evaluates it on the held-out test set (M:280-340)."""
    ledger: object
    test: Shard
    model: HostModel
    test_epoch: int = 0
    history: List[tuple] = field(default_factory=list)
    log: Optional[Callable[[str], None]] = print

    def poll(self) -> Optional[float]:
        w, epoch = self.ledger.QueryGlobalModel()
        if epoch > self.test_epoch:
            acc = self.model.accuracy(torch.as_tensor(np.asarray(w), dtype=torch.float32),
                                      self.test.x, self.test.y)
            self.test_epoch = epoch
            self.history.append((epoch, acc))
            if self.log:
                self.log("Epoch: %03d, test_acc: %.4f" % (epoch, acc))  # M:327-328
            return acc
        return None
