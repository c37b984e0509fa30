"""LoRA fine-tuning of a frozen BERT / GPT base: the trained parameters are low-rank adapters.

``LoRANet(base, rank, alpha, targets)`` is a ``FlatNet`` whose ``ParamSpec`` holds the adapters
only (``{enc|dec}{i}.{t}.lora_a`` [r, K] and ``.lora_b`` [N, r] for every targeted projection t of
every layer, plus BERT's new task head ``cls.w`` / ``cls.b``).  The engine, the heap layout, the
consensus kernel, DP, the server optimizers and FedProx all work on ``spec.total`` floats, so the
whole protocol runs on the adapter vector: only the adapters train and travel.

The base model (an fp32 master and its bf16 shadow) stays in each device's memory, held by the net
and bound next to the adapters.  Its weights, layer norms, embeddings and (GPT) tied head are frozen:
their gradient views are ``None``, so nothing accumulates into them, and a targeted projection runs
``ops.nn.lora_linear``, ``y = act(x W^T + (alpha / r) (x A^T) B^T + b)``.  The adapter genesis is A
uniform in +-1/sqrt(fan_in) (as ``ParamSpec.init_``) and B = 0, so the genesis LoRA model computes
exactly the base model.
"""
from __future__ import annotations

import hashlib
import json
import os
from typing import Dict, NamedTuple, Optional, Sequence

import torch

from .flat import ParamSpec
from .nets import BertBase, Bound, FlatNet, GPT, ResNet18

BF = torch.bfloat16

TARGETS = ("q", "k", "v", "o", "ff1", "ff2")
RANKS = tuple(range(8, 65, 8))


class Adapter(NamedTuple):
    """One projection's adapter views: ``a`` [r, K] and ``bl`` [N, r] bf16, their fp32 gradient
    views (None for inference) and the scale alpha / r."""
    a: torch.Tensor
    bl: torch.Tensor
    ga: Optional[torch.Tensor]
    gbl: Optional[torch.Tensor]
    scale: float


def parse_targets(targets) -> tuple:
    """"q,v" or an iterable of names -> the validated tuple in canonical order."""
    names = [t.strip() for t in targets.split(",")] if isinstance(targets, str) else [str(t) for t in targets]
    names = [t for t in names if t]
    bad = sorted(set(names) - set(TARGETS))
    if bad or not names:
        raise ValueError(f"LoRA targets must be a non-empty subset of {','.join(TARGETS)}; got {targets!r}")
    return tuple(t for t in TARGETS if t in names)


def check_rank(rank: int) -> int:
    if int(rank) != rank or int(rank) not in RANKS:
        raise ValueError(f"LoRA rank must be a multiple of 8 in [8, 64]; got {rank}")
    return int(rank)


def base_digest(master: torch.Tensor) -> str:
    """sha256 of the base fp32 master's bytes (hex): ranks and checkpoints compare it."""
    return hashlib.sha256(master.detach().to("cpu", torch.float32).contiguous().numpy().tobytes()).hexdigest()


def model_shape(net) -> Optional[dict]:
    """The shape fields of a BERT / GPT net (what a base checkpoint must match), else None."""
    if not isinstance(net, (BertBase, GPT)):
        return None
    return dict(family=type(net).__name__, layers=net.L, hidden=net.Hd, heads=net.heads, ffn=net.ffn,
             max_pos=net.max_pos, n_classes=net.n_classes, vocab=net.spec.by_name["emb.word"].shape[0])


class LoRANet(FlatNet):
    def __init__(self, base: FlatNet, rank: int, alpha: float = 0.0, targets: Sequence[str] | str = ("q", "v"),
                 base_master: Optional[torch.Tensor] = None, base_seed: int = 1234):
        if not isinstance(base, (BertBase, GPT)):
            raise ValueError(f"LoRA needs a BERT or GPT base model, got {type(base).__name__}")
        self.base, self.rank = base, check_rank(rank)
        self.alpha = float(alpha) if alpha else float(self.rank)
        if not self.alpha > 0.0:
            raise ValueError(f"LoRA alpha must be > 0 (0: the rank); got {alpha}")
        self.scale = self.alpha / self.rank
        self.targets = parse_targets(targets)
        self.n_classes = base.n_classes
        self.is_gpt = isinstance(base, GPT)
        pre = "dec" if self.is_gpt else "enc"
        bspec = base.spec.by_name
        self.adapted: Dict[str, tuple] = {}     # projection -> (lora_a name, lora_b name)
        ents = []
        for i in range(base.L):
            for t in self.targets:
                proj = f"{pre}{i}.{t}"
                N, K = bspec[f"{proj}.w"].shape
                ents.extend([(f"{proj}.lora_a", (self.rank, K)), (f"{proj}.lora_b", (N, self.rank))])
                self.adapted[proj] = (f"{proj}.lora_a", f"{proj}.lora_b")
        if not self.is_gpt:                     # a new task head trains with the adapters
            ents.extend([("cls.w", bspec["cls.w"].shape), ("cls.b", bspec["cls.b"].shape)])
        self.spec = ParamSpec(ents)
        self.head = base.head
        if base_master is not None:
            base_master = base_master.detach().to("cpu", torch.float32).contiguous()
            if base_master.numel() != base.spec.total:
                raise ValueError(f"LoRA base has {base_master.numel()} parameters, the {type(base).__name__} "
                                 f"spec {base.spec.total}")
        self._base_cpu = base_master
        self.base_seed = int(base_seed)
        self._base: Dict[torch.device, tuple] = {}   # device -> (fp32 master, bf16 shadow)

    # ------------------------------------------------------------------ base model
    @classmethod
    def base_from_checkpoint(cls, path: str, model: str, base: FlatNet) -> torch.Tensor:
        """The global model of a ``run.py --checkpoint`` file of a full (non-LoRA) run of ``model``
        with ``base``'s shape.  A multi-rank run writes ``path.rank<i>`` files holding the same global
        model; ``path.rank0`` is read when ``path`` itself does not exist.  Refuses another model, a
        LoRA run, another parameter count, and (when the checkpoint records it) another shape."""
        src = path if os.path.exists(path) or not os.path.exists(f"{path}.rank0") else f"{path}.rank0"
        blob = torch.load(src, map_location="cpu", weights_only=True)
        cfg = json.loads(blob["config"]) if isinstance(blob.get("config"), str) else {}
        if cfg.get("model") != model:
            raise ValueError(f"LoRA base checkpoint {src} is a {cfg.get('model')!r} run, not {model!r}")
        if cfg.get("lora_rank", 0):
            raise ValueError(f"LoRA base checkpoint {src} is itself a LoRA run: the base must be a full model")
        if int(blob["n_params"]) != base.spec.total:
            raise ValueError(f"LoRA base checkpoint {src} has {int(blob['n_params'])} parameters; this "
                             f"{model} has {base.spec.total} (another shape?)")
        if "model_shape" in blob:
            want, got = model_shape(base), json.loads(blob["model_shape"])
            if got != want:
                raise ValueError(f"LoRA base checkpoint {src} has model shape {got}; this {model} is {want}")
        return blob["global_master"][:base.spec.total].to(torch.float32)

    def base_buffers(self, device) -> tuple:
        """(fp32 master, bf16 shadow) of the frozen base on ``device`` (made on first use)."""
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        got = self._base.get(device)
        if got is None:
            m = torch.empty(self.base.spec.total, device=device, dtype=torch.float32)
            if self._base_cpu is not None:
                m.copy_(self._base_cpu)
            else:
                self.base.init_(m, seed=self.base_seed)
            got = (m, m.to(BF))
            self._base[device] = got
        return got

    def base_digest(self, device) -> str:
        return base_digest(self.base_buffers(device)[0])

    # ------------------------------------------------------------------ FlatNet
    def init_(self, master: torch.Tensor, seed: int = 0):
        """Adapter genesis: A ~ U(+-1/sqrt(fan_in)) (ParamSpec.init_), B = 0; BERT's head as the
        base net initialises it (uniform weights, zero bias)."""
        self.spec.init_(master, seed)
        P = self.spec.views(master)
        for _, b in self.adapted.values():
            P[b].zero_()

    def bind(self, master, shadow, grad=None) -> Bound:
        bm, bs = self.base_buffers(master.device)
        P = self.base.spec.views(bm)
        S = self.base.spec.views(bs)
        Pa, Sa = self.spec.views(master), self.spec.views(shadow)
        Ga = self.spec.views(grad) if grad is not None else None
        for nm in ("cls.w", "cls.b"):
            if nm in Pa:
                P[nm], S[nm] = Pa[nm], Sa[nm]
        G = None
        if Ga is not None:
            G = {nm: None for nm in P}
            for nm in ("cls.w", "cls.b"):
                if nm in Ga:
                    G[nm] = Ga[nm]
        lora = {proj: Adapter(Sa[a], Sa[b], Ga[a] if Ga else None, Ga[b] if Ga else None, self.scale)
                for proj, (a, b) in self.adapted.items()}
        return Bound(P, S, G, lora)

    def preprocess(self, x_raw):
        return self.base.preprocess(x_raw)

    def features(self, b, x, train, rng=None):
        return self.base.features(b, x, train, rng)

    def train_features(self, b, x, rng=None):
        return self.base.train_features(b, x, rng)

    def loss(self, b, x, y, correct=None, rng=None, row_loss=None):
        return self.base.loss(b, x, y, correct, rng, row_loss)

    def correct(self, b, x, y):
        return self.base.correct(b, x, y)

    def __getattr__(self, name):
        # shape attributes the engine and data paths read (L, Hd, max_pos, vocab, pad_id, ...)
        if name.startswith("_") or name == "base":
            raise AttributeError(name)
        return getattr(self.base, name)


def lora_net_from_config(cfg, base: FlatNet, base_path: Optional[str] = None) -> "LoRANet":
    """The LoRANet that ``cfg.lora_rank`` / ``lora_alpha`` / ``lora_targets`` describe over ``base``,
    with the frozen base read from ``base_path`` (a full run's checkpoint) or, without one, the base
    net's seeded genesis (the model a full run of the same config starts from)."""
    if cfg.lora_rank == 0:
        raise ValueError("lora_net_from_config: the config has lora_rank 0 (LoRA off)")
    bm = LoRANet.base_from_checkpoint(base_path, cfg.model, base) if base_path else None
    return LoRANet(base, cfg.lora_rank, cfg.lora_alpha, cfg.lora_targets, base_master=bm,
                   base_seed=cfg.seed + 1234)


def check_net_matches_config(cfg, net) -> None:
    """Refuse a net that is not what the config says: a LoRANet needs lora_rank > 0 with the same rank,
    alpha and targets, a config with lora_rank > 0 needs a LoRANet, and a ResNet18 needs the config's
    resnet_norm."""
    if isinstance(net, ResNet18) and net.norm != cfg.resnet_norm:
        raise ValueError(f"config and net disagree on ResNet-18's norm: resnet_norm is {cfg.resnet_norm!r}, "
                         f"the net has {net.norm!r}")
    is_lora = isinstance(net, LoRANet)
    if is_lora != (cfg.lora_rank > 0):
        raise ValueError("config and net disagree on LoRA: " +
                         (f"the net is a LoRANet but lora_rank is 0" if is_lora else
                          f"lora_rank is {cfg.lora_rank} but the net ({type(net).__name__}) has no adapters; "
                          "build it with models.lora.lora_net_from_config"))
    if is_lora:
        alpha = float(cfg.lora_alpha) if cfg.lora_alpha else float(cfg.lora_rank)
        if (net.rank, net.alpha, net.targets) != (cfg.lora_rank, alpha, parse_targets(cfg.lora_targets)):
            raise ValueError(f"LoRANet (rank {net.rank}, alpha {net.alpha}, targets {','.join(net.targets)}) does "
                             f"not match the config (rank {cfg.lora_rank}, alpha {alpha}, targets {cfg.lora_targets})")
