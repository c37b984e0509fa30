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

Full-model sites (``FLConfig.dpsgd_full_model``): a sequence site whose two sides are both wider than 64
(BERT / GPT projections, GPT's LM head) takes its norm in Gram form, sum_{t,t'} (p_t . p_t') (q_t . q_t'),
in ``k_pe_gram``; embeddings use its one-hot mode, GPT's tied ``emb.word`` adds the head-embedding cross
term, and layer norms have ``k_pe_ln``.  The Gram form's computed value can miss ||V||^2 by up to
kappa ab^2 (``gram_kappa``), which ``k_dpsgd_clip`` folds in under the root:
||v_n|| = sqrt(sum sq + sum_sites kappa ab^2).  Layer-norm and embedding gradients are released with
fixed-order sums (no atomics), so a full-model step is bit-reproducible too.

Convolutional sites (``FLConfig.dpsgd_conv``): a convolution is a linear site over its patch matrix P [B*R, K]
(R = OH * OW output positions per example; a bias adds a column of ones).  ``conv_norm_path`` picks, from the
shapes, the Gram form (R <= 512 and R (a + b) < a b) or product tiles.  ``record_conv`` takes the patches the
im2col path saved: 64 x 64 tiles of dz_n^T [P_n | 1] in ``k_pe_norm``, the abs term ``k_pe_rows`` over (dz, P),
and the release is the weight-gradient GEMM on the scaled rows and the masked patches with a deterministic
split-K (``gemm.gemm_dw_fixed_split``).  An implicit-GEMM convolution never forms its patches
(``record_conv_implicit``): its tile norms and its release run in the implicit weight-gradient GEMM itself, by
K groups (``conv_dw_groups``), and its abs term reads x (``dpsgd_patch_rows``).  Group norms
(``record_groupnorm``) keep ``k_gn_bwd``'s per-example fp32 partials: sq_n = sum_c pg^2 + pb^2, released as
sum_n c_n pg_n in example order; their norm is of the released partials themselves, so they need no abs term.

Poisson sampling (``FLConfig.dpsgd_sampling = "poisson"``, ``PoissonSampler``): each step runs at the capacity
``cap`` with the step's count of sampled examples as ``n_valid``; the padding slots get c = 0, so they release
exact zeros, and the loss carries the 1 / B of the expected batch size B (``norm_batch``).

Packed batches (``FLConfig.dpsgd_packed``, ``begin(segments)``): a packed BERT step's token sites have T rows,
example n owning rows [cu_seqlens[n], cu_seqlens[n + 1]) of length L_n, and its [CLS] sites (pooler, classifier)
B rows.  A site of T rows is recorded with its segmentation: every per-example kernel runs its segmented form
(``cu_seqlens`` / ``seq_ids``), whose partial for example n is a function of that example's rows only and equals
the uniform kernel on that example alone at R = L_n, bit for bit.  A site of B rows is an R = 1 site as before.
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


def clip_factors(sq: np.ndarray, ab: np.ndarray, batch: int, clip: float, kap=None, n_valid=None) -> np.ndarray:
    """fp32 mirror of ``k_dpsgd_clip``: sq [n_sq, B] and ab [n_ab, B] summed over their rows in order,
    bound = (B sqrt(sq)) (1 + gamma) + (B ab) (u + gamma); c = 0 for a non-finite bound, 1 for
    bound <= clip (bit-pattern compare), else clip / bound.  ``kap`` [n_ab] (None: no Gram site): the
    Gram slack sum_i kap_i ab_i^2 over the rows with kap_i != 0, in order, is added to sq first.
    ``n_valid`` (None: every column): columns n >= n_valid are padding slots of a Poisson batch, c = 0.
    ``batch`` is the B of the bound, the expected batch size under Poisson sampling."""
    sq, ab = np.asarray(sq, _F), np.asarray(ab, _F)
    with np.errstate(all="ignore"):
        s = np.zeros(sq.shape[1], _F)
        for row in sq:
            s = (s + row).astype(_F)
        a = np.zeros(ab.shape[1] if ab.size else sq.shape[1], _F)
        for row in ab:
            a = (a + row).astype(_F)
        if kap is not None:
            k = np.zeros_like(s)
            for ki, row in zip(np.asarray(kap, _F), ab):
                if ki != 0:
                    k = (k + (ki * (row * row).astype(_F)).astype(_F)).astype(_F)
            s = (s + k).astype(_F)
        bsz, cl = _F(batch), _F(clip)
        bound = ((np.sqrt(s) * bsz).astype(_F) * ONE_PLUS_GAMMA).astype(_F) + \
            ((a * bsz).astype(_F) * U_PLUS_GAMMA).astype(_F)
        bound = bound.astype(_F)
        c = np.where(bound.view(np.uint32) <= np.array(cl).view(np.uint32), _F(1), (cl / bound).astype(_F))
        c = np.where(np.isfinite(bound), c, _F(0)).astype(_F)
        if n_valid is not None:
            c[int(n_valid):] = _F(0)
        return c


EPS_ACC = 2.0 ** -23     # one fp32 rounding or truncation of an accumulation, the tensor cores' included


def _gamma(n: int) -> float:
    return n * EPS_ACC / (1.0 - n * EPS_ACC)


def gram_kappa(kp: int, kq: int, depth: int) -> np.float32:
    """The Gram form's slack: |computed - ||P^T Q||_F^2| <= kappa (sum_t ||p_t|| ||q_t||)^2 (DESIGN.md,
    "DP-SGD").  ``kp`` / ``kq`` the two Grams' inner dimensions (0 for an exact one-hot or gathered side; a
    site bias adds one column), ``depth`` the longest fp32 summation chain a partial passes through (tile
    reduction plus the clip kernel's sums).  The factor 2 covers the fp32 evaluation of ab and of the fold;
    rounded up to fp32."""
    k = 2.0 * ((1.0 + _gamma(kp)) * (1.0 + _gamma(kq)) * (1.0 + _gamma(depth)) - 1.0)
    return np.nextafter(_F(k), _F(np.inf)) if float(_F(k)) < k else _F(k)


def noise_sigma(noise: float, clip: float, batch: int) -> np.float32:
    """The fp32 noise scale z * C / B of one step's averaged gradient."""
    return _F(_F(_F(noise) * _F(clip)) / _F(batch))


def _rows_like(t: torch.Tensor) -> torch.Tensor:
    """An uninitialised bf16 matrix shaped like ``t`` with a 16-byte row pitch, as the GEMMs need."""
    rows, cols = t.shape
    return torch.empty(rows, (cols + 7) // 8 * 8, device=t.device, dtype=t.dtype)[:, :cols]


def _wide_narrow(a: torch.Tensor, b: torch.Tensor):
    return (b, a) if a.shape[1] <= 64 and b.shape[1] > a.shape[1] else (a, b)


_TIED_ROWS = 36 + 36 + 64   # a tied embedding at R <= 512: head Gram, one-hot Gram and their cross term


def _site_rows(shape, conv: bool) -> int:
    """sq rows one 2-D parameter can take: ceil(max / 64) norm tiles or its tied-Gram allowance, and with
    ``conv`` the 64 x 64 tiles of a convolution weight [Cout, K] with a bias column (which also cover the
    implicit-GEMM norm's 128 x 64 tiles)."""
    a, b = shape
    rows = max((max(a, b) + 63) // 64, _TIED_ROWS)
    return max(rows, ((a + 63) // 64) * ((b + 1 + 63) // 64)) if conv else rows


def conv_norm_path(R: int, a: int, b: int) -> str:
    """Which exact form takes a convolution site's per-example norms: "gram" when R <= 512 and
    R (a + b) < a b (R^2 (a + b) multiply-adds per example against R a b), else "tiles".  a = Cout, b the patch
    width with the bias column."""
    return "gram" if R <= 512 and R * (a + b) < a * b else "tiles"


class PoissonSampler:
    """DP-SGD's Poisson sample of one round's local steps (``k_dpsgd_poisson_sample``), in fixed-capacity slots.

    Record j of ``records`` S is in local step i's sample iff its Philox uniform u_j (key: the client's secret
    ``seed``, counter {j / 4, 0, *step_word + i, kDpsgdSampleSite}) is below thr = floor(q 2^32), q = batch / S
    (``oracle.poisson_threshold``); the accounted rate is ``q`` = thr / 2^32.  ``cap`` = ``poisson_capacity``: the
    sampled records fill ``idx[i, :count[i]]`` in record order, the rest point at record 0, and a step that
    samples more than ``cap`` keeps the first ``cap`` and counts in ``overflow`` (probability ``eta`` per step,
    the exact binomial tail at ``cap``).  idx and count are the client's own device memory: the sample is
    secret, like the noise."""

    def __init__(self, records: int, batch: int, steps: int, seed: int, device):
        from ..protocol.oracle import poisson_threshold
        from ..protocol.privacy import binomial_tail, poisson_capacity
        self.S, self.steps = int(records), int(steps)
        self.thr = poisson_threshold(batch, records)
        self.q = self.thr / 2.0 ** 32
        self.cap = poisson_capacity(self.S, self.q)
        self.eta = binomial_tail(self.S, self.q, self.cap)
        self.seed = int(seed) % (1 << 64)
        self.idx = torch.zeros(self.steps, self.cap, device=device, dtype=torch.int32)
        self.count = torch.zeros(self.steps, device=device, dtype=torch.int32)
        self.overflow = torch.zeros(1, device=device, dtype=torch.int32)   # overflowed steps of the last round

    def sample(self, step_word: torch.Tensor):
        """One launch: every step's sample of the round, step i keyed by *step_word + i; resets ``overflow``."""
        self.overflow.zero_()
        C().dpsgd_poisson_sample(self.seed, step_word, self.S, self.thr, self.idx, self.count, self.overflow)


class DPSGDStep:
    """Per-step DP-SGD context over a model's flat gradient buffer.  Graph-capturable: every buffer is
    allocated here, sized from ``spec`` (each 2-D parameter is at most one site: its 64 x 64 norm tiles with a
    bias column, or up to 136 Gram tile pairs for a tied embedding at 512 rows; each 1-D parameter at most one
    layer-norm or group-norm row), and the noise reads the step word on the device.

    ``batch``: examples per step (a site's rows per example is its row count / batch); ``clip`` C > 0;
    ``noise`` z >= 0 (0: clipping only, no noise kernel); ``seed`` the client's secret noise key;
    ``step_word`` the int32 [1] device word the noise is keyed by (plus ``finish``'s ``step_add``); ``conv``:
    the model has convolution sites (``FLConfig.dpsgd_conv``), whose tiles the buffers are sized for.
    ``norm_batch`` (default ``batch``): the B of the released (1 / B) (sum + noise) -- Poisson sampling runs
    ``batch`` = the capacity slots and B the expected batch size; its loss must then carry the 1 / B, and
    ``finish`` takes the step's count of real examples as ``n_valid``."""

    def __init__(self, spec, batch: int, clip: float, noise: float, seed: int, step_word: torch.Tensor,
                 device, conv: bool = False, norm_batch: Optional[int] = None):
        clip32, noise32 = _F(clip), _F(noise)
        norm_batch = batch if norm_batch is None else norm_batch
        if not (batch >= 1 and norm_batch >= 1 and math.isfinite(clip32) and clip32 > 0 and math.isfinite(noise32)
                and noise32 >= 0):
            raise ValueError(f"DP-SGD needs batch >= 1, a finite clip > 0 and a finite noise >= 0 (fp32); got "
                             f"batch {batch} (normalised by {norm_batch}), clip {clip}, noise {noise}")
        self.B, self.clip, self.noise = int(batch), float(clip32), float(noise32)
        self.norm_batch = int(norm_batch)
        self.sigma = float(noise_sigma(noise32, clip32, self.norm_batch))
        self.seed, self.step_word = int(seed) % (1 << 64), step_word
        mats = [e.shape for e in spec.entries if len(e.shape) == 2]
        vecs = [e.shape for e in spec.entries if len(e.shape) == 1]
        self.conv = bool(conv)
        rows = sum(_site_rows(s, self.conv) for s in mats) + len(vecs) or 1
        n_ab = max(2 * len(mats) + len(vecs), 1)
        self.sq = torch.zeros(rows, self.B, device=device, dtype=torch.float32)
        self.ab = torch.zeros(n_ab, self.B, device=device, dtype=torch.float32)
        self.kap = torch.zeros(n_ab, device=device, dtype=torch.float32)   # Gram slack per abs row
        self.c = torch.ones(self.B, device=device, dtype=torch.float32)
        self.dropped = torch.zeros(1, device=device, dtype=torch.int32)   # examples with a non-finite bound
        self._records: List[tuple] = []
        self._seg = None            # the collecting step's PackedTokens (begin), None for uniform rows
        self._n_sq = self._n_ab = 0
        self._kappa: dict = {}      # abs row -> (kp, kq, multiplier) of a Gram site

    # ---------------------------------------------------------------- collection
    def begin(self, segments=None):
        """Start collecting one step's sites.  ``segments``: the step's ``PackedTokens`` (a packed batch of
        exactly ``batch`` examples, at most 512 tokens each), or None for uniform rows per example."""
        global _ACTIVE
        if _ACTIVE is not None:
            raise RuntimeError("a DP-SGD step is already collecting")
        if segments is not None:
            if len(segments) != self.B:
                raise ValueError(f"DP-SGD: a packed batch of {len(segments)} examples, not the batch {self.B}")
            if not 1 <= segments.max_len <= 512:
                raise ValueError(f"DP-SGD: packed examples must have 1 to 512 tokens, got up to {segments.max_len}")
        self._seg = segments
        self._records, self._n_sq, self._n_ab, self._kappa = [], 0, 0, {}
        _ACTIVE = self

    def _rows_per_example(self, M: int) -> int:
        if self._seg is not None:
            raise ValueError("DP-SGD: this site has no segmented form for packed batches")
        if M % self.B != 0:
            raise ValueError(f"DP-SGD: a site has {M} rows, not a multiple of the batch {self.B}")
        return M // self.B

    def _layout(self, M: int):
        """(R, seg) of a site of M rows: uniform (seg None, R rows per example), or in a packed step the
        segmented rows of its T tokens (R = max_len, seg the ``PackedTokens``); a packed step's site of B rows
        (the [CLS] rows) is an R = 1 site."""
        pt = self._seg
        if pt is None:
            return self._rows_per_example(M), None
        if M == self.B:
            return 1, None
        if M == pt.T:
            return pt.max_len, pt
        raise ValueError(f"DP-SGD: a site of a packed step has {M} rows, neither the batch {self.B} nor the "
                         f"{pt.T} tokens")

    @staticmethod
    def _cu(seg) -> dict:
        return {} if seg is None else {"cu_seqlens": seg.cu_seqlens}

    def _scale_rows(self, X, lay, out, mask_only=False):
        """out = bf16(X's rows times their example's clip factor); ``lay`` a record's R or ``PackedTokens``."""
        if isinstance(lay, int):
            C().dpsgd_scale_rows(X, self.c, lay, out, mask_only=mask_only)
        else:
            C().dpsgd_scale_rows(X, self.c, 1, out, mask_only=mask_only, seq_ids=lay.seq_ids)

    def _take_ab(self) -> int:
        if self._n_ab + 1 > self.ab.shape[0]:
            raise RuntimeError("DP-SGD: more sites than the model's parameter spec allows")
        self._n_ab += 1
        return self._n_ab - 1

    def _take_sq(self, n: int) -> torch.Tensor:
        if self._n_sq + n > self.sq.shape[0]:
            raise RuntimeError("DP-SGD: more norm tiles than the model's parameter spec allows")
        self._n_sq += n
        return self.sq[self._n_sq - n:self._n_sq]

    def _gram_site(self, q: torch.Tensor, R: int, bias: float, sym: bool = True, seg=None, **p) -> None:
        out = self._take_sq(C().dpsgd_gram_pairs(R, sym))
        C().dpsgd_pe_gram(q, p.pop("q2", q), R, bias, out, sym=sym, **self._cu(seg), **p)

    def record(self, dz: torch.Tensor, op: torch.Tensor, gw: Optional[torch.Tensor], gb: Optional[torch.Tensor]):
        """A weight-gradient site gw += dz^T op (and gb += column sums of dz): launch its per-example
        norm kernels now, run the GEMM in ``finish`` on the clipped rows.  R = 1: the row identity; one
        side at most 64 wide and no bias: tiles of the product (a LoRA adapter); otherwise the Gram form,
        with op extended by a 1 where the site has a bias."""
        if gw is None and gb is None:
            return
        R, seg = self._layout(dz.shape[0])
        cu = self._cu(seg)
        bias = 1.0 if gb is not None else 0.0
        ia = self._take_ab()
        ab = self.ab[ia]
        if R == 1:
            C().dpsgd_pe_rows(dz, op, 1, bias, self._take_sq(1)[0], ab)
        else:
            wide, narrow = _wide_narrow(dz, op)
            if narrow.shape[1] <= 64 and gb is None:
                tiles = (wide.shape[1] + 63) // 64
                C().dpsgd_pe_norm(wide, narrow, R, self._take_sq(tiles), **cu)
                C().dpsgd_pe_rows(wide, narrow, R, 0.0, None, ab, **cu)
            else:
                self._gram_site(op, R, bias, seg=seg, p1=dz, p2=dz, mode=0)
                C().dpsgd_pe_rows(dz, op, R, bias, None, ab, **cu)
                self._kappa[ia] = (dz.shape[1], op.shape[1] + (gb is not None), 1)
        self._records.append(("lin", dz, op, gw, gb, R if seg is None else seg, ia))

    def record_conv(self, dz: torch.Tensor, col: torch.Tensor, gw: Optional[torch.Tensor],
                    gb: Optional[torch.Tensor]):
        """A convolution's weight gradient gw += dz^T col (and gb += column sums of dz): dz [B*R, Cout], col the
        patch matrix [B*R, K], R = OH * OW.  Per-example norms now, in the form ``conv_norm_path`` picks; the
        deterministic split-K GEMM on the clipped rows and masked patches in ``finish``."""
        if gw is None and gb is None:
            return
        if gw is None:
            raise ValueError("DP-SGD: a convolution site with a bias gradient but no weight gradient")
        self._need_conv()
        R = self._rows_per_example(dz.shape[0])
        bias = gb is not None
        a, b = dz.shape[1], col.shape[1] + int(bias)
        ia = self._take_ab()
        if conv_norm_path(R, a, b) == "gram":
            self._gram_site(col, R, float(bias), p1=dz, p2=dz, mode=0)
            self._kappa[ia] = (a, b, 1)
        else:
            C().dpsgd_pe_norm(dz, col, R, self._take_sq(C().dpsgd_norm_tiles(a, col.shape[1], bias)), bias=bias)
        C().dpsgd_pe_rows(dz, col, R, float(bias), None, self.ab[ia])
        self._records.append(("conv", dz, col, gw, gb, R, ia))

    def _need_conv(self):
        if not self.conv:
            raise RuntimeError("DP-SGD: a convolution site in a step not sized for convolutions (conv=True)")

    def record_conv_implicit(self, dz: torch.Tensor, x: torch.Tensor, geom: tuple, gw: Optional[torch.Tensor]):
        """An implicit-GEMM convolution's weight gradient gw += dW over x [N, H, W, C] and dz [N*OH*OW, Cout]
        (``geom`` = (N, C, H, W, kh, kw, stride, pad, OH, OW)), no bias: its patches are never formed.  Norms:
        R % 64 == 0 on the product-tile path, the weight-gradient GEMM's per-example mode (``conv_dw_groups``,
        one K group per example, each 128 x 64 tile squared in the epilogue); a Gram site (stages 3-4) builds
        its patches in scratch for the norm only.  The abs term is ``dpsgd_patch_rows`` from x.  ``finish``
        releases through the same GEMM on the masked x, by whole-example K groups into workspace slices."""
        if gw is None:
            return
        self._need_conv()
        N, Cin, H, W, kh, kw, stride, pad, OH, OW = geom
        R = self._rows_per_example(dz.shape[0])
        a, K = dz.shape[1], kh * kw * Cin
        ia = self._take_ab()
        m = C()
        if conv_norm_path(R, a, K) == "gram":
            col = torch.empty(dz.shape[0], K, device=x.device, dtype=x.dtype)
            m.im2col(x, col, N, Cin, H, W, kh, kw, stride, pad, OH, OW)
            self._gram_site(col, R, 0.0, p1=dz, p2=dz, mode=0)
            self._kappa[ia] = (a, K, 1)
        elif R % 64 == 0:
            out = self._take_sq(m.conv_dw_norm_tiles(a, K))
            m.conv_dw_groups(x, dz, out, N, H, W, Cin, OH, OW, kh, kw, stride, pad, self.B, True)
        else:
            col = torch.empty(dz.shape[0], K, device=x.device, dtype=x.dtype)
            m.im2col(x, col, N, Cin, H, W, kh, kw, stride, pad, OH, OW)
            m.dpsgd_pe_norm(dz, col, R, self._take_sq(m.dpsgd_norm_tiles(a, K, False)))
        m.dpsgd_patch_rows(dz, x, N, H, W, Cin, OH, OW, kh, kw, stride, pad, 0.0, self.ab[ia])
        self._records.append(("convx", dz, x, geom, gw, R, ia))

    def record_groupnorm(self, pg: torch.Tensor, pb: torch.Tensor, gg: Optional[torch.Tensor],
                         gb: Optional[torch.Tensor]):
        """A group norm's gamma / beta from its per-example partials pg, pb [B, C] (fp32, ``groupnorm_bwd``):
        sq_n = sum_c pg^2 + pb^2 now, gg += sum_n c_n pg_n (gb likewise) in example order in ``finish``."""
        if gg is None and gb is None:
            return
        if pg.shape[0] != self.B:
            raise ValueError(f"DP-SGD: a group norm has {pg.shape[0]} examples, not the batch {self.B}")
        pg = pg if gg is not None else torch.zeros_like(pg)
        pb = pb if gb is not None else torch.zeros_like(pb)
        C().dpsgd_pe_gn(pg, pb, self._take_sq(1)[0])
        self._records.append(("gn", pg, pb, gg, gb))

    def record_layernorm(self, dy: torch.Tensor, x: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor,
                         gg: Optional[torch.Tensor], gb: Optional[torch.Tensor]):
        """A layer norm's gamma / beta: per-example norms now, fixed-order release in ``finish``."""
        if gg is None and gb is None:
            return
        R, seg = self._layout(dy.shape[0])
        C().dpsgd_pe_ln(dy, x, mean, rstd, R, self._take_sq(1)[0], self.ab[self._take_ab()], **self._cu(seg))
        self._records.append(("ln", dy, x, mean, rstd, gg, gb, R if seg is None else seg))

    def record_embedding(self, dy: torch.Tensor, tables: list):
        """An embedding's gradient: ``tables`` [(ids int32 [rows], fp32 table gradient [V, C])], each row r
        adding dy_r to row ids_r.  One-hot Gram norms now (repeated ids count); a table that is also an
        earlier recorded site's gradient (GPT's tied head) adds the cross term of the two uses."""
        R, seg = self._layout(dy.shape[0])
        ents = []
        for ids, g in tables:
            if g is None:
                continue
            ia = self._take_ab()
            self._gram_site(dy, R, 0.0, seg=seg, id1=ids, id2=ids, mode=1)
            C().dpsgd_pe_rows(dy, dy[:, :0], R, 1.0, None, self.ab[ia], **self._cu(seg))     # ||e_id|| = 1
            head = next((r for r in self._records if r[0] == "lin" and r[3] is not None
                         and r[3].data_ptr() == g.data_ptr() and r[3].shape == g.shape), None)
            if head is None:
                self._kappa[ia] = (0, dy.shape[1], 1)
            else:
                _, dl, h, _, _, Rh, ih = head
                if Rh != (R if seg is None else seg):
                    raise ValueError(f"DP-SGD: a tied table's two uses have {Rh} and {R} rows per example")
                # 2 sum_{t,t'} dl_t[id_t'] (h_t . dy_t'): one parameter, one site
                self._gram_site(h, R, 0.0, sym=False, seg=seg, q2=dy, p1=dl, id2=ids, mode=2)
                # kappa (x + y)^2 <= 2 kappa x^2 + 2 kappa y^2 over the two uses' abs rows
                self._kappa[ih] = self._kappa[ia] = (dl.shape[1], h.shape[1], 2)
            ents.append((ids, g, torch.empty(ids.numel(), device=ids.device, dtype=torch.int32)))
        if ents:
            self._records.append(("emb", dy, ents, R if seg is None else seg))

    # ---------------------------------------------------------------- release
    def finish(self, grad: torch.Tensor, step_add: int, n_valid: Optional[torch.Tensor] = None):
        """Clip factors, clipped weight, bias, layer-norm and embedding gradients, then the noise over all
        of ``grad``.  ``n_valid`` (int32 [1] on the device, or None): examples n >= *n_valid are padding and
        get c = 0, so every release path turns them into exact zeros."""
        global _ACTIVE
        if _ACTIVE is not self:
            raise RuntimeError("DPSGDStep.finish without begin")
        _ACTIVE = None
        self._seg = None
        m = C()
        if self._kappa:
            # the longest fp32 chain of a Gram partial: its tile reduction, then the clip kernel's sums
            depth = 64 + self._n_sq + self._n_ab
            self.kap.zero_()
            for i, (kp, kq, mult) in self._kappa.items():
                self.kap[i].fill_(float(_F(mult) * gram_kappa(kp, kq, depth)))
        m.dpsgd_clip(self.sq[:self._n_sq], self._n_sq, self.ab[:self._n_ab], self._n_ab, self.B,
                     float(self.norm_batch), self.clip, self.c, self.dropped,
                     kap=self.kap[:self._n_ab] if self._kappa else None, n_valid=n_valid)
        for rec in self._records:
            kind, dz = rec[0], rec[1]
            if kind == "gn":
                _, pg, pb, gg, gb = rec
                cols = pg.shape[1]
                gg = gg if gg is not None else torch.zeros(cols, device=pg.device)
                gb = gb if gb is not None else torch.zeros(cols, device=pg.device)
                m.groupnorm_param(pg, pb, gg, gb, cf=self.c)
                continue
            s = _rows_like(dz)
            R = rec[-1] if kind not in ("lin", "conv", "convx") else rec[5]   # an int, or a packed step's segments
            self._scale_rows(dz, R, s)
            if kind == "convx":
                _, _, x, geom, gw, _, _ = rec
                N, Cin, H, W, kh, kw, stride, pad, OH, OW = geom
                # a dropped example's input pixels are zeroed: its patches are then exact zeros
                xm = torch.empty_like(x)
                m.dpsgd_scale_rows(x.view(-1, Cin), self.c, H * W, xm.view(-1, Cin), mask_only=True)
                if G.fixed_splits(s.shape[0], gw.shape[0], gw.shape[1], self.B, align=64):
                    G.conv_dw_fixed_split(xm, s, gw, geom, self.B)
                else:   # no run of whole examples fills 64-pixel boxes (e.g. R 16 at B 3): the patches' GEMM
                    col = torch.empty(s.shape[0], gw.shape[1], device=x.device, dtype=x.dtype)
                    m.im2col(xm, col, N, Cin, H, W, kh, kw, stride, pad, OH, OW)
                    G.gemm_dw_fixed_split(s, col, gw, G.fixed_splits(s.shape[0], gw.shape[0], gw.shape[1], self.B))
            elif kind in ("lin", "conv"):
                _, _, op, gw, gb, _, _ = rec
                if gw is not None:
                    # a dropped example's operand rows are zeroed too: they may be what is not finite
                    x = _rows_like(op)
                    self._scale_rows(op, R, x, mask_only=True)
                    if kind == "lin":
                        # one writer per output element (no split-K atomics): the same bits on every run
                        G.gemm(s, x, out=gw, a_mn=True, b_mn=True, accumulate=True)
                    else:
                        # B * R rows into few output tiles: split over whole examples, slices added in order
                        G.gemm_dw_fixed_split(s, x, gw, G.fixed_splits(s.shape[0], gw.shape[0], gw.shape[1], self.B))
                if gb is not None:
                    m.dpsgd_colsum(s, gb)
            elif kind == "ln":
                _, _, x, mean, rstd, gg, gb, _ = rec
                cols = x.shape[1]
                gg = gg if gg is not None else torch.zeros(cols, device=x.device)
                gb = gb if gb is not None else torch.zeros(cols, device=x.device)
                if isinstance(R, int):
                    m.dpsgd_ln_release(s, x, mean, rstd, self.c, R, gg, gb)
                else:
                    m.dpsgd_ln_release(s, x, mean, rstd, self.c, 1, gg, gb, seq_ids=R.seq_ids)
            else:
                for ids, g, perm in rec[2]:
                    m.dpsgd_emb_release(s, ids, perm, g)
        self._records = []
        if self.sigma > 0.0:
            m.dpsgd_noise(grad, self.seed, self.step_word, int(step_add), self.sigma)

    def abandon(self):
        """Stop collecting without releasing anything (a failed backward)."""
        global _ACTIVE
        if _ACTIVE is self:
            _ACTIVE = None
        self._records = []
        self._seg = None
