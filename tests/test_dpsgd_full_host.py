"""Full-model DP-SGD on the host: the --dpsgd-full-model opt-in and its refusals, the clip-factor mirror without
Gram sites (bit-identical to the plain bound) and with them, the Gram form's certified slack on
cancellation-heavy fixtures, and modelled mistakes that the fixtures catch."""
import numpy as np
import pytest
import torch

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.ops import dpsgd as D

F32 = np.float32


# ------------------------------------------------------------------ config and CLI
def test_full_model_opt_in_is_accepted_and_refused_as_specified():
    for m in ("bert", "gpt"):
        assert FLConfig(model=m, dpsgd_clip=1.0, dpsgd_full_model=True).validate().dpsgd_on
        with pytest.raises(ValueError, match=f"DP-SGD on {m} needs LoRA.*dpsgd_full_model"):
            FLConfig(model=m, dpsgd_clip=1.0).validate()
    bad = [dict(model="gpt", dpsgd_full_model=True),                                   # no clip
           dict(model="gpt", dpsgd_clip=1.0, dpsgd_full_model=True, lora_rank=8),       # LoRA
           dict(model="mlp", dpsgd_clip=1.0, dpsgd_full_model=True),
           dict(model="resnet18", dpsgd_clip=1.0, dpsgd_full_model=True),
           dict(model="gpt", dpsgd_clip=1.0, dpsgd_full_model=True, dtype="fp8")]
    for kw in bad:
        with pytest.raises(ValueError):
            FLConfig(**kw).validate()
    assert not FLConfig().validate().dpsgd_full_model


@pytest.mark.parametrize("argv, why", [
    (["--model", "gpt", "--dpsgd-full-model"], "--dpsgd-full-model needs --dpsgd-clip"),
    (["--model", "gpt", "--lora-rank", "8", "--dpsgd-clip", "1", "--dpsgd-full-model"], "excludes LoRA"),
    (["--model", "mlp", "--generic", "--dpsgd-clip", "1", "--dpsgd-full-model"], "applies to bert and gpt"),
    (["--model", "bert", "--packed", "--dpsgd-clip", "1", "--dpsgd-full-model"], "does not support --packed"),
    (["--model", "bert", "--dpsgd-clip", "1"], "or opt in to full-model DP-SGD"),
])
def test_cli_refuses(argv, why, capsys):
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert e.value.code == 2
    assert why in capsys.readouterr().err


# ------------------------------------------------------------------ the clip-factor mirror
def test_clip_factors_without_gram_sites_are_the_plain_bound_bit_for_bit():
    rng = np.random.default_rng(0)
    sq = rng.random((7, 16)).astype(F32) * 10
    ab = rng.random((4, 16)).astype(F32) * 30
    for clip in (0.1, 1.0, 1e30):
        plain = D.clip_factors(sq, ab, 16, clip)
        assert np.array_equal(plain.view(np.uint32), D.clip_factors(sq, ab, 16, clip, None).view(np.uint32))
        zeros = D.clip_factors(sq, ab, 16, clip, np.zeros(4, F32))     # no row carries a Gram slack
        assert np.array_equal(plain.view(np.uint32), zeros.view(np.uint32))
    kap = np.array([0, 0.01, 0, 0], F32)
    c = D.clip_factors(sq, ab, 16, 1.0, kap)
    assert (c <= D.clip_factors(sq, ab, 16, 1.0)).all() and (c < D.clip_factors(sq, ab, 16, 1.0)).any()


def test_gram_kappa_grows_with_the_inner_dimensions():
    k0 = D.gram_kappa(0, 768, 4096)
    assert 0 < k0 < D.gram_kappa(768, 3072, 4096) < D.gram_kappa(50257, 768, 4096) < 0.03
    assert float(D.gram_kappa(3072, 3072, 4096)) >= 2 * 2 * 3072 * 2.0 ** -23


# ------------------------------------------------------------------ the Gram bound in fp64
def _f32_gram(P, Q, bias, tile=64):
    """The kernel's arithmetic in numpy: fp32 Grams (a random summation order per entry), products and a
    tiled fp32 reduction."""
    Gp = (P.astype(F32) @ P.astype(F32).T).astype(F32)
    Gq = ((Q.astype(F32) @ Q.astype(F32).T).astype(F32) + F32(bias)).astype(F32)
    prod = (Gp * Gq).astype(F32)
    s = F32(0)
    R = P.shape[0]
    for i in range(0, R, tile):
        for j in range(0, R, tile):
            s = F32(s + F32(prod[i:i + tile, j:j + tile].sum(dtype=F32)))
    return s


@pytest.mark.parametrize("seed", range(6))
def test_gram_slack_bounds_the_computed_norm_on_cancelling_fixtures(seed):
    """Rows that nearly cancel: the per-example gradient is tiny next to sum_t ||p_t|| ||q_t||, so the fp32
    Gram sum misses ||V||^2 by far more than a relative rounding.  s + kappa ab^2 >= ||V||^2 holds in fp64."""
    rng = np.random.default_rng(seed)
    R, a, b = 128, 200, 96
    base_p, base_q = rng.standard_normal(a), rng.standard_normal(b)
    sign = np.where(np.arange(R) % 2 == 0, 1.0, -1.0)
    P = (sign[:, None] * base_p[None, :] + 1e-3 * rng.standard_normal((R, a))).astype(F32)
    Q = (base_q[None, :] + 1e-3 * rng.standard_normal((R, b))).astype(F32)
    P64, Q64 = P.astype(np.float64), np.hstack([Q.astype(np.float64), np.ones((R, 1))])
    V2 = float(np.sum((P64.T @ Q64) ** 2))
    s = float(_f32_gram(P, Q, 1.0))
    ab = float(np.sum(np.linalg.norm(P64, axis=1) * np.linalg.norm(Q64, axis=1)))
    kap = float(D.gram_kappa(a, b + 1, 4096))
    assert s + kap * ab * ab >= V2
    assert abs(s - V2) > 1e-6 * V2            # a fixture where the computed value alone is off


# ------------------------------------------------------------------ modelled mistakes
def _tied_fixture(seed=0, R=12, V=9, H=5):
    rng = np.random.default_rng(seed)
    dl, h = rng.standard_normal((R, V)), rng.standard_normal((R, H))
    dy, ids = rng.standard_normal((R, H)), rng.integers(0, V, R)
    E = np.eye(V)[ids]
    G = dl.T @ h + E.T @ dy                     # the one parameter's per-example gradient
    return dl, h, dy, ids, E, G


def test_mistakes_fail_the_fixtures():
    # the tied cross term dropped
    dl, h, dy, ids, E, G = _tied_fixture()
    head = np.sum((dl @ dl.T) * (h @ h.T))
    emb = np.sum((ids[:, None] == ids[None, :]) * (dy @ dy.T))
    cross = 2 * np.sum(dl[:, ids] * (h @ dy.T))
    assert np.isclose(head + emb + cross, np.sum(G ** 2))
    assert not np.isclose(head + emb, np.sum(G ** 2), rtol=1e-3)
    # repeated token ids treated as distinct (the one-hot Gram as the identity)
    ids_rep = np.array([3, 3, 3, 1, 1, 0, 5, 3, 2, 2, 3, 1])
    Er = np.eye(9)[ids_rep]
    true = np.sum((Er.T @ dy) ** 2)
    assert np.isclose(np.sum((ids_rep[:, None] == ids_rep[None, :]) * (dy @ dy.T)), true)
    assert not np.isclose(np.sum(dy ** 2), true, rtol=1e-3)
    # the Gram bias term omitted: Gq without its + 1 misses the bias gradient sum_t dz_t
    rng = np.random.default_rng(1)
    dz, x = rng.standard_normal((10, 6)), rng.standard_normal((10, 4))
    x1 = np.hstack([x, np.ones((10, 1))])
    true = np.sum((dz.T @ x1) ** 2)
    assert np.isclose(np.sum((dz @ dz.T) * (x @ x.T + 1)), true)
    assert not np.isclose(np.sum((dz @ dz.T) * (x @ x.T)), true, rtol=1e-3)
    # beta omitted from the layer-norm norm
    dy2, xh = rng.standard_normal((10, 6)), rng.standard_normal((10, 6))
    gg, gb = (dy2 * xh).sum(0), dy2.sum(0)
    assert np.sum(gg ** 2) < np.sum(gg ** 2) + np.sum(gb ** 2) * (1 - 1e-3)
    # per-site instead of per-example clipping: two sites of one example each clipped to C let the example
    # contribute up to sqrt(2) C
    clip, g1, g2 = 1.0, np.full(4, 3.0), np.full(4, 4.0)
    per_site = np.concatenate([g1 * min(1, clip / np.linalg.norm(g1)), g2 * min(1, clip / np.linalg.norm(g2))])
    full = np.concatenate([g1, g2])
    per_ex = full * min(1, clip / np.linalg.norm(full))
    assert np.linalg.norm(per_ex) <= clip * (1 + 1e-12) < np.linalg.norm(per_site)
    c = D.clip_factors(np.array([[F32(np.sum(g1 ** 2))], [F32(np.sum(g2 ** 2))]], F32), np.zeros((1, 1), F32),
                       1, clip)
    assert np.linalg.norm(c[0] * full) <= clip


def test_step_buffers_fit_a_full_model_spec():
    from bflc_demo_b200.models.nets import GPT, BertBase
    for net in (BertBase(2, layers=2), GPT(layers=2, vocab=512)):
        step = D.DPSGDStep(net.spec, 16, 1.0, 0.0, 0, torch.zeros(1, dtype=torch.int32), "cpu")
        mats = [e for e in net.spec.entries if len(e.shape) == 2]
        # every 2-D parameter can be a tied Gram site at 512 rows: 36 + 36 + 64 tile pairs
        assert step.sq.shape[0] >= 136 * len(mats) and step.kap.shape[0] == step.ab.shape[0]
