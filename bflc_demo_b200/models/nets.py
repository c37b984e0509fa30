"""Model families of BASELINE.json on the hand-written kernels: LeNet-5 (config #3),
ResNet-18 (config #4), BERT-base (config #5), the generic MLP / softmax regression, and a GPT-2
style decoder for next-token prediction, all as *functional* models over a flat parameter buffer
(``models/flat.py``):

    net = LeNet5();  bound = net.bind(master, shadow, grad)
    loss = net.loss(bound, x, y);  loss.backward()        # grads land in the flat grad buffer
    hits = net.correct(bound_of_any_weights, x, y)        # e.g. a peer's uploaded weights

Channel / feature dims that would break TMA's 16-byte row alignment are padded to a multiple
of 8 with zero-initialised weights; a zero pad channel receives exactly zero gradient (its
activation is relu(0)=0 and the next layer's weights for it are zero), so the padded network
computes exactly the un-padded one.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from .._native import C
from ..data.packing import PackedTokens
from ..ops import gemm as G
from ..ops import nn as F
from .flat import ParamSpec

BF = torch.bfloat16


def _up8(n: int) -> int:
    return (n + 7) // 8 * 8


@dataclass
class Bound:
    P: Dict[str, torch.Tensor]            # fp32 master views (biases, norm params, running stats)
    S: Dict[str, torch.Tensor]            # bf16 shadow views (GEMM operands)
    G: Optional[Dict[str, torch.Tensor]]  # fp32 grad views or None (inference)
    # optional LoRA adapters (models/lora.py): projection name (e.g. "enc0.q") -> lora.Adapter;
    # a BERT / GPT projection with an entry runs ops.nn.lora_linear over its frozen weight
    lora: Optional[Dict[str, tuple]] = None

    def g(self, name):
        return self.G[name] if self.G is not None else None


class FlatNet:
    """Base: owns a ParamSpec, binds flat buffers, provides loss/correct on top of ``logits_in``."""
    spec: ParamSpec
    n_classes: int

    def bind(self, master, shadow, grad=None) -> Bound:
        return Bound(self.spec.views(master), self.spec.views(shadow),
                     self.spec.views(grad) if grad is not None else None)

    def init_(self, master: torch.Tensor, seed: int = 0):
        self.spec.init_(master, seed)
        self._post_init(self.spec.views(master))

    def _post_init(self, P):  # zero the padding rows/cols, set norm scales
        pass

    def preprocess(self, x_raw: torch.Tensor) -> torch.Tensor:
        raise NotImplementedError

    def features(self, b: Bound, x, train: bool):  # -> [rows, feat] bf16 input of the head
        raise NotImplementedError

    head = ("fc.w", "fc.b")

    def train_features(self, b: Bound, x, rng=None):
        """Features of the training forward; ``rng`` (ops.nn.DropoutRNG) feeds models with dropout."""
        return self.features(b, x, True)

    def loss(self, b: Bound, x, y, correct=None, rng=None, row_loss=None):
        """Mean training loss; ``row_loss`` (fp32, one entry per target, or None) receives each target's loss."""
        h = self.train_features(b, x, rng)
        w, bias = self.head
        return F.linear_xent(h, b.S[w], b.P[bias], b.g(w), b.g(bias), y, correct, row_loss)

    @torch.no_grad()
    def correct(self, b: Bound, x, y) -> torch.Tensor:
        h = self.features(b, x, False)
        w, bias = self.head
        cnt = torch.zeros(1, device=h.device, dtype=torch.int32)
        G.gemm_argmax_acc(h.contiguous(), b.S[w], y, cnt, n_classes=self.n_classes, bias=b.P[bias])
        return cnt


# ----------------------------------------------------------------------------- MLP
class MLPNet(FlatNet):
    def __init__(self, in_dim=784, hidden=256, n_classes=62):
        self.n_classes = n_classes
        self.in_dim = in_dim
        self.spec = ParamSpec([("fc1.w", (hidden, in_dim)), ("fc1.b", (hidden,)),
                               ("fc.w", (n_classes, hidden)), ("fc.b", (n_classes,))])

    def preprocess(self, x_raw):
        x = x_raw.reshape(x_raw.shape[0], -1).contiguous()
        out = torch.empty(x.shape, device=x.device, dtype=BF)
        C().cast_u8_to_bf16(x, out, 1.0 / 255.0)
        return out

    def features(self, b, x, train):
        if train:
            x = x.detach().requires_grad_(True)
        return F.linear(x, b.S["fc1.w"], b.P["fc1.b"], b.g("fc1.w"), b.g("fc1.b"), G.ACT_RELU,
                        need_dx=False)


# ----------------------------------------------------------------------------- LeNet-5
class LeNet5(FlatNet):
    """conv5x5(3->6) - pool - conv5x5(6->16) - pool - fc120 - fc84 - fc10 on 3x32x32 inputs.
    6 -> 8 channels and 84 -> 88 features are zero-padded (see module docstring)."""

    def __init__(self, n_classes=10, in_ch=3):
        self.n_classes, self.in_ch = n_classes, in_ch
        self.c1, self.c2 = 8, 16          # 6 (+2 pad), 16
        self.k1 = _up8(25 * in_ch)        # 75 -> 80
        self.k2 = 25 * self.c1            # 200
        self.f1, self.f2 = 120, 88        # 84 (+4 pad)
        self.flat = 5 * 5 * self.c2       # 400
        self.spec = ParamSpec([
            ("conv1.w", (self.c1, self.k1)), ("conv1.b", (self.c1,)),
            ("conv2.w", (self.c2, self.k2)), ("conv2.b", (self.c2,)),
            ("fc1.w", (self.f1, self.flat)), ("fc1.b", (self.f1,)),
            ("fc2.w", (self.f2, self.f1)), ("fc2.b", (self.f2,)),
            ("fc.w", (n_classes, self.f2)), ("fc.b", (n_classes,))])

    def _post_init(self, P):
        P["conv1.w"][6:].zero_(); P["conv1.w"][:, 25 * self.in_ch:].zero_()
        w2 = P["conv2.w"].view(self.c2, 25, self.c1)
        w2[:, :, 6:].zero_()
        P["fc2.w"][84:].zero_(); P["fc.w"][:, 84:].zero_()

    def preprocess(self, x_raw):  # uint8 [N, 3, 32, 32] -> bf16 NHWC
        x = x_raw.permute(0, 2, 3, 1).contiguous()
        out = torch.empty(x.shape, device=x.device, dtype=BF)
        C().cast_u8_to_bf16(x.view(-1), out.view(-1), 1.0 / 255.0)
        return out

    def features(self, b, x, train):
        if train:
            x = x.detach().requires_grad_(True)
        g = b.g
        x = F.conv2d(x, b.S["conv1.w"], b.P["conv1.b"], g("conv1.w"), g("conv1.b"), 5, 5, 1, 0,
                     G.ACT_RELU, need_dx=False)
        x = F.maxpool2d(x, 2, 2)
        x = F.conv2d(x, b.S["conv2.w"], b.P["conv2.b"], g("conv2.w"), g("conv2.b"), 5, 5, 1, 0,
                     G.ACT_RELU)
        x = F.maxpool2d(x, 2, 2)
        x = x.reshape(x.shape[0], -1)
        x = F.linear(x, b.S["fc1.w"], b.P["fc1.b"], g("fc1.w"), g("fc1.b"), G.ACT_RELU)
        return F.linear(x, b.S["fc2.w"], b.P["fc2.b"], g("fc2.w"), g("fc2.b"), G.ACT_RELU)


# ----------------------------------------------------------------------------- ResNet-18
class ResNet18(FlatNet):
    """CIFAR-style ResNet-18: conv3x3(3->64) stem, stages [64,128,256,512] x 2 BasicBlocks,
    global average pool, fc.  ~11.2 M parameters.

    ``norm="batch"``: batch norm, whose running statistics live in the flat buffer (so FedAvg averages
    them like every other parameter).  ``norm="group"``: group norm (``ops.nn.groupnorm``, 32 groups;
    every width a multiple of 32), whose statistics are per example and per forward, so the spec holds
    only gamma and beta: nothing mixes examples, and nothing but weights is averaged across clients
    with skewed shards."""

    NORMS = ("batch", "group")

    def __init__(self, n_classes=10, in_ch=3, widths=(64, 128, 256, 512), norm="batch"):
        if norm not in self.NORMS:
            raise ValueError(f"ResNet18: norm must be one of {', '.join(self.NORMS)}, got {norm!r}")
        if norm == "group" and any(c % F.GN_GROUPS for c in widths):
            raise ValueError(f"ResNet18: group norm needs every width a multiple of {F.GN_GROUPS}, got {widths}")
        self.n_classes, self.in_ch, self.widths, self.norm = n_classes, in_ch, widths, norm
        ents: List[Tuple[str, Tuple[int, ...]]] = []

        def bn(name, c):
            ents.extend([(f"{name}.gamma", (c,)), (f"{name}.beta", (c,))])
            if norm == "batch":
                ents.extend([(f"{name}.rmean", (c,)), (f"{name}.rvar", (c,))])

        self.k_stem = _up8(9 * in_ch)
        ents.append(("stem.w", (widths[0], self.k_stem)))
        bn("stem.bn", widths[0])
        self.blocks = []
        cin = widths[0]
        for si, c in enumerate(widths):
            for bi in range(2):
                stride = 2 if (si > 0 and bi == 0) else 1
                name = f"l{si}.{bi}"
                ents.append((f"{name}.c1.w", (c, 9 * cin)))
                bn(f"{name}.bn1", c)
                ents.append((f"{name}.c2.w", (c, 9 * c)))
                bn(f"{name}.bn2", c)
                down = stride != 1 or cin != c
                if down:
                    ents.append((f"{name}.down.w", (c, cin)))
                    bn(f"{name}.dbn", c)
                self.blocks.append((name, cin, c, stride, down))
                cin = c
        ents.extend([("fc.w", (n_classes, widths[-1])), ("fc.b", (n_classes,))])
        self.spec = ParamSpec(ents)

    def _post_init(self, P):
        for k, v in P.items():
            if k.endswith(".rvar"):
                v.fill_(1.0)
        P["stem.w"][:, 9 * self.in_ch:].zero_()

    preprocess = LeNet5.preprocess

    def _bn(self, b, name, x, train, relu, residual=None):
        if self.norm == "group":
            return F.groupnorm(x, b.P[f"{name}.gamma"], b.P[f"{name}.beta"], b.g(f"{name}.gamma"),
                               b.g(f"{name}.beta"), relu=relu, residual=residual)
        return F.batchnorm(x, b.P[f"{name}.gamma"], b.P[f"{name}.beta"], b.g(f"{name}.gamma"),
                           b.g(f"{name}.beta"), b.P[f"{name}.rmean"], b.P[f"{name}.rvar"],
                           training=train, relu=relu, residual=residual)

    def features(self, b, x, train):
        if train:
            x = x.detach().requires_grad_(True)
        g = b.g
        x = F.conv2d(x, b.S["stem.w"], None, g("stem.w"), None, 3, 3, 1, 1, need_dx=False)
        x = self._bn(b, "stem.bn", x, train, True)
        for name, cin, c, stride, down in self.blocks:
            idt = x
            y = F.conv2d(x, b.S[f"{name}.c1.w"], None, g(f"{name}.c1.w"), None, 3, 3, stride, 1)
            y = self._bn(b, f"{name}.bn1", y, train, True)
            y = F.conv2d(y, b.S[f"{name}.c2.w"], None, g(f"{name}.c2.w"), None, 3, 3, 1, 1)
            if down:
                idt = F.conv2d(x, b.S[f"{name}.down.w"], None, g(f"{name}.down.w"), None, 1, 1,
                               stride, 0)
                idt = self._bn(b, f"{name}.dbn", idt, train, False)
            x = self._bn(b, f"{name}.bn2", y, train, True, residual=idt)
        return F.global_avgpool(x)


# ----------------------------------------------------------------------------- BERT-base
class BertBase(FlatNet):
    """BERT-base encoder for sequence classification: 12 layers, hidden 768, 12 heads, FFN 3072,
    vocab 30522, 512 positions (seq_len 128 in config #5); post-LN, GELU; classifier on [CLS]
    through a 768->768 GELU pooler.  ~109 M parameters.

    ``pad_id``: inputs are right-padded with this token id; each sequence's length is its count of
    other ids, and attention masks the keys past it.  None: every position is a real token.

    ``packed=True`` (needs ``pad_id``): ``preprocess`` packs the batch into ``PackedTokens`` (the
    real tokens of every sample concatenated, ``data/packing.py``), so embedding, projections, FFN
    and layer norms run on the real tokens only and attention on ``cu_seqlens``.  It computes what
    the padded model computes on the real tokens.

    ``dropout`` p in [0, 1): in the training forward (``loss`` with a ``DropoutRNG``) p applies at the
    embedding output, the attention probabilities, the attention-output and FFN-output branches
    before their residual adds, and the pooled [CLS] vector.  Each site has a fixed id
    (``dropout_site``), and masks are keyed by in-sequence coordinates, so packed still computes what
    padded computes.  ``features(..., train=False)`` and ``correct`` never drop."""
    head = ("cls.w", "cls.b")
    # dropout site kinds: site id = 8 * layer + kind (embedding and pooler on layer 0)
    SITE_EMB, SITE_ATTN, SITE_ATTN_OUT, SITE_FFN_OUT, SITE_POOL = 0, 1, 2, 3, 4

    def __init__(self, n_classes=2, layers=12, hidden=768, heads=12, ffn=3072, vocab=30522,
                 max_pos=512, pad_id=None, packed=False, dropout=0.0):
        if packed and pad_id is None:
            raise ValueError("BertBase: packed=True needs a pad_id")
        if not 0.0 <= dropout < 1.0:
            raise ValueError(f"BertBase: dropout must lie in [0, 1), got {dropout}")
        self.n_classes, self.L, self.Hd, self.heads, self.ffn = n_classes, layers, hidden, heads, ffn
        self.max_pos, self.pad_id, self.packed, self.dropout = max_pos, pad_id, packed, float(dropout)
        ents: List[Tuple[str, Tuple[int, ...]]] = [
            ("emb.word", (vocab, hidden)), ("emb.pos", (max_pos, hidden)),
            ("emb.ln.gamma", (hidden,)), ("emb.ln.beta", (hidden,))]
        for i in range(layers):
            p = f"enc{i}"
            for nm in ("q", "k", "v", "o"):
                ents.extend([(f"{p}.{nm}.w", (hidden, hidden)), (f"{p}.{nm}.b", (hidden,))])
            ents.extend([(f"{p}.ln1.gamma", (hidden,)), (f"{p}.ln1.beta", (hidden,)),
                         (f"{p}.ff1.w", (ffn, hidden)), (f"{p}.ff1.b", (ffn,)),
                         (f"{p}.ff2.w", (hidden, ffn)), (f"{p}.ff2.b", (hidden,)),
                         (f"{p}.ln2.gamma", (hidden,)), (f"{p}.ln2.beta", (hidden,))])
        ents.extend([("pool.w", (hidden, hidden)), ("pool.b", (hidden,)),
                     ("cls.w", (n_classes, hidden)), ("cls.b", (n_classes,))])
        self.spec = ParamSpec(ents)

    def _post_init(self, P):
        P["emb.word"].mul_(0.02 * (self.Hd ** 0.5))  # ~N(0, 0.02)-scale embeddings
        P["emb.pos"].mul_(0.02 * (self.Hd ** 0.5))

    def preprocess(self, x_raw):  # int64 [N, S] -> int32, or PackedTokens when packed
        if self.packed:
            return PackedTokens.from_padded(x_raw, self.pad_id)
        return x_raw.to(torch.int32).contiguous()

    def _lin(self, b, name, x, act=G.ACT_NONE):
        ad = b.lora.get(name) if b.lora is not None else None
        if ad is not None:
            return F.lora_linear(x, b.S[f"{name}.w"], b.P[f"{name}.b"], ad.a, ad.bl, ad.ga, ad.gbl, ad.scale, act)
        return F.linear(x, b.S[f"{name}.w"], b.P[f"{name}.b"], b.g(f"{name}.w"), b.g(f"{name}.b"), act)

    def _ln(self, b, name, x):
        return F.layernorm(x, b.P[f"{name}.gamma"], b.P[f"{name}.beta"], b.g(f"{name}.gamma"),
                           b.g(f"{name}.beta"))

    @staticmethod
    def dropout_site(layer: int, kind: int) -> int:
        return 8 * layer + kind

    def _encoder(self, b, x, attend, residual):
        """attend(q, k, v, site); residual(x, branch, site) -> x + dropout(branch)."""
        site = self.dropout_site
        for i in range(self.L):
            p = f"enc{i}"
            q, k, v = (self._lin(b, f"{p}.{nm}", x) for nm in ("q", "k", "v"))
            a = self._lin(b, f"{p}.o", attend(q, k, v, site(i, self.SITE_ATTN)))
            x = self._ln(b, f"{p}.ln1", residual(x, a, site(i, self.SITE_ATTN_OUT)))
            h = self._lin(b, f"{p}.ff1", x, G.ACT_GELU)
            x = self._ln(b, f"{p}.ln2", residual(x, self._lin(b, f"{p}.ff2", h), site(i, self.SITE_FFN_OUT)))
        return x

    def _pool(self, b, cls_tok, p, rng):
        """Pooler on the [CLS] rows (pooled row b is sequence b, position 0 for dropout)."""
        pooled = self._lin(b, "pool", cls_tok, G.ACT_GELU)
        return F.dropout(pooled, p, rng, self.dropout_site(0, self.SITE_POOL), S=1) if p > 0.0 else pooled

    def _features_packed(self, b, pt: PackedTokens, p=0.0, rng=None):
        if pt.max_len > self.max_pos:
            raise ValueError(f"BertBase: sequence length {pt.max_len} exceeds the {self.max_pos} position embeddings")
        x = F.embedding(pt.ids, b.S["emb.word"], b.S["emb.pos"], b.g("emb.word"), b.g("emb.pos"),
                        self.max_pos, pos_ids=pt.pos_ids)
        x = self._ln(b, "emb.ln", x)
        rows = dict(seq_ids=pt.seq_ids, pos_ids=pt.pos_ids)
        if p > 0.0:
            x = F.dropout(x, p, rng, self.dropout_site(0, self.SITE_EMB), **rows)
        x = self._encoder(
            b, x,
            lambda q, k, v, site: F.attention_packed(q, k, v, pt.cu_seqlens, pt.max_len, self.heads,
                                                     dropout_p=p, rng=rng, site=site),
            lambda x, z, site: F.dropout_add(x, z, p, rng, site, **rows) if p > 0.0 else F.add(x, z))
        cls_tok = x.index_select(0, pt.cu_seqlens[:-1])
        return self._pool(b, cls_tok, p, rng)

    def train_features(self, b, x, rng=None):
        if self.dropout > 0.0 and rng is None:
            raise ValueError("BertBase: dropout > 0 needs a DropoutRNG for the training forward (loss(..., rng=))")
        return self.features(b, x, True, rng)

    def features(self, b, ids, train, rng=None):
        p = self.dropout if (train and rng is not None) else 0.0
        if isinstance(ids, PackedTokens):
            return self._features_packed(b, ids, p, rng)
        B, S = ids.shape
        if S > self.max_pos:
            raise ValueError(f"BertBase: sequence length {S} exceeds the {self.max_pos} position embeddings")
        lengths = None if self.pad_id is None else (ids != self.pad_id).sum(1, dtype=torch.int32)
        x = F.embedding(ids.reshape(-1), b.S["emb.word"], b.S["emb.pos"], b.g("emb.word"),
                        b.g("emb.pos"), S)
        x = self._ln(b, "emb.ln", x)
        if p > 0.0:
            x = F.dropout(x, p, rng, self.dropout_site(0, self.SITE_EMB), S=S)
        x = self._encoder(
            b, x,
            lambda q, k, v, site: F.attention(q, k, v, B, S, self.heads, lengths=lengths, dropout_p=p, rng=rng,
                                              site=site),
            lambda x, z, site: F.dropout_add(x, z, p, rng, site, S=S) if p > 0.0 else F.add(x, z))
        cls_tok = x.view(B, S, self.Hd)[:, 0, :]
        return self._pool(b, cls_tok, p, rng)


# ----------------------------------------------------------------------------- GPT
class GPT(FlatNet):
    """Pre-LN GPT-2 decoder for next-token prediction: token + position embeddings, per layer
    ``x += o(causal_attention(q, k, v of ln1(x)))`` and ``x += ff2(gelu(ff1(ln2(x))))``, a final
    ``ln_f`` and an output head tied to ``emb.word`` (no bias).  Defaults: 12 layers, hidden 768,
    12 heads of 64, FFN 3072, vocab 8192, 512 positions.  Inputs are int token ids [N, S] (S a
    multiple of 64 in [64, 512]); targets are the next tokens [N, S], and ``n_classes`` is the vocab.

    Attention is the fused causal kernel (csrc/kernels/attn_sm100.cu), the loss the vocabulary-wide
    cross-entropy ``ops.nn.lm_xent`` and ``correct`` counts next-token hits over every position.

    ``dropout`` p in [0, 1): in the training forward (``loss`` with a ``DropoutRNG``) p applies at the
    embedding output, the attention probabilities and both residual branches, with BertBase's site
    ids (``8 * layer + kind``).  ``features(..., train=False)`` and ``correct`` never drop."""
    SITE_EMB, SITE_ATTN, SITE_ATTN_OUT, SITE_FFN_OUT = 0, 1, 2, 3
    HITS_ROWS = 2048            # rows of fp32 logits per validation chunk

    def __init__(self, layers=12, hidden=768, heads=12, ffn=3072, vocab=8192, max_pos=512, dropout=0.0):
        if hidden != 64 * heads:
            raise ValueError(f"GPT: head dim must be 64 (hidden = 64 * heads); got hidden {hidden}, {heads} heads")
        if not 0.0 <= dropout < 1.0:
            raise ValueError(f"GPT: dropout must lie in [0, 1), got {dropout}")
        self.n_classes, self.L, self.Hd, self.heads, self.ffn = vocab, layers, hidden, heads, ffn
        self.vocab, self.max_pos, self.dropout = vocab, max_pos, float(dropout)
        ents: List[Tuple[str, Tuple[int, ...]]] = [("emb.word", (vocab, hidden)), ("emb.pos", (max_pos, hidden))]
        for i in range(layers):
            p = f"dec{i}"
            ents.extend([(f"{p}.ln1.gamma", (hidden,)), (f"{p}.ln1.beta", (hidden,))])
            for nm in ("q", "k", "v", "o"):
                ents.extend([(f"{p}.{nm}.w", (hidden, hidden)), (f"{p}.{nm}.b", (hidden,))])
            ents.extend([(f"{p}.ln2.gamma", (hidden,)), (f"{p}.ln2.beta", (hidden,)),
                         (f"{p}.ff1.w", (ffn, hidden)), (f"{p}.ff1.b", (ffn,)),
                         (f"{p}.ff2.w", (hidden, ffn)), (f"{p}.ff2.b", (hidden,))])
        ents.extend([("ln_f.gamma", (hidden,)), ("ln_f.beta", (hidden,))])
        self.spec = ParamSpec(ents)

    _post_init = BertBase._post_init
    _lin = BertBase._lin
    _ln = BertBase._ln
    dropout_site = staticmethod(BertBase.dropout_site)

    def preprocess(self, x_raw):  # int64 [N, S] -> int32
        return x_raw.to(torch.int32).contiguous()

    def train_features(self, b, x, rng=None):
        if self.dropout > 0.0 and rng is None:
            raise ValueError("GPT: dropout > 0 needs a DropoutRNG for the training forward (loss(..., rng=))")
        return self.features(b, x, True, rng)

    def features(self, b, ids, train, rng=None):
        """-> ln_f output [N * S, hidden] bf16, row n * S + t = position t of sample n."""
        p = self.dropout if (train and rng is not None) else 0.0
        B, S = ids.shape
        if S > self.max_pos:
            raise ValueError(f"GPT: sequence length {S} exceeds the {self.max_pos} position embeddings")
        site = self.dropout_site
        x = F.embedding(ids.reshape(-1), b.S["emb.word"], b.S["emb.pos"], b.g("emb.word"), b.g("emb.pos"), S)
        if p > 0.0:
            x = F.dropout(x, p, rng, site(0, self.SITE_EMB), S=S)

        def residual(x, z, kind, i):
            return F.dropout_add(x, z, p, rng, site(i, kind), S=S) if p > 0.0 else F.add(x, z)

        for i in range(self.L):
            pf = f"dec{i}"
            a = self._ln(b, f"{pf}.ln1", x)
            q, k, v = (self._lin(b, f"{pf}.{nm}", a) for nm in ("q", "k", "v"))
            att = F.attention(q, k, v, B, S, self.heads, dropout_p=p, rng=rng, site=site(i, self.SITE_ATTN),
                              causal=True)
            x = residual(x, self._lin(b, f"{pf}.o", att), self.SITE_ATTN_OUT, i)
            h = self._lin(b, f"{pf}.ff1", self._ln(b, f"{pf}.ln2", x), G.ACT_GELU)
            x = residual(x, self._lin(b, f"{pf}.ff2", h), self.SITE_FFN_OUT, i)
        return self._ln(b, "ln_f", x)

    def loss(self, b: Bound, x, y, correct=None, rng=None, row_loss=None):
        h = self.train_features(b, x, rng)
        return F.lm_xent(h, b.S["emb.word"], b.g("emb.word"), y.reshape(-1), correct, row_loss)

    @torch.no_grad()
    def correct(self, b: Bound, x, y) -> torch.Tensor:
        h = self.features(b, x, False)
        cnt = torch.zeros(1, device=h.device, dtype=torch.int32)
        return F.lm_hits(h, b.S["emb.word"], y.reshape(-1), cnt, self.HITS_ROWS)


def build_model(name: str, n_classes: int, **kw) -> FlatNet:
    name = name.lower()
    if name == "mlp":
        return MLPNet(kw.get("in_dim", 784), kw.get("hidden", 256), n_classes)
    if name in ("lenet5", "lenet"):
        return LeNet5(n_classes)
    if name == "resnet18":
        return ResNet18(n_classes, norm=kw.get("norm", "batch"))
    if name in ("bert", "bert-base", "bert_base"):
        return BertBase(n_classes, layers=kw.get("layers", 12), pad_id=kw.get("pad_id"),
                        packed=kw.get("packed", False), dropout=kw.get("dropout", 0.0))
    if name == "gpt":      # n_classes is the vocabulary
        return GPT(layers=kw.get("layers", 12), vocab=n_classes, dropout=kw.get("dropout", 0.0))
    raise ValueError(f"unknown model {name}")
