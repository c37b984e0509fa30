"""FedProx local training on the CPU: configuration and flags, the host client's ``train_pass`` against
fp64 autograd, the host simulator, and an exact fp32 model of the recipe kernel with the proximal term
(``test_gpu_prox.py`` checks the kernels against it).

The definition every path implements, per parameter and local step, mu = fp32(prox_mu):
``d = w - w0`` (w the master before the step, w0 the round's global model), ``g' = fma(mu, d, g)`` with
g the gradient as the optimizer sees it (in the recipe kernel: after the clip coefficient); the
optimizer then consumes g'.  A skipped (non-finite) recipe step skips the term too.  mu = 0 is the
path without the term.
"""
from __future__ import annotations

import math
from dataclasses import replace

import numpy as np
import pytest
import torch

from test_optim_spec_host import (F32, SH_INIT, Case, check_update, f32_fma, f32_mul, f32_sub, recipe_cases,
                                  run_update, values)

MU = 0.37


# ------------------------------------------------------------------------------ the kernel model
def prox_update(c: Case, anchor: np.ndarray, mu: float, mutant: str | None = None):
    """Outputs of ``optim_recipe_step`` with the anchor, exactly as the kernel computes them; ``mutant``
    names a kernel mistake to model instead:

    * ``anchor_is_master``: d taken against the current master (d = 0);
    * ``d_sign_flipped``: d = w0 - w;
    * ``before_coef``: the term added before the clip coefficient scales the gradient;
    * ``tail_skipped``: the scalar tail loop leaves the term out;
    * ``term_on_skipped_step``: a skipped (non-finite) step drops the data gradient but still applies
      the term, w and the moments moving by g' = fma(mu, d, 0)."""
    skipped = c.recipe and c.clip is not None and c.nonfinite
    if skipped and mutant != "term_on_skipped_step":
        return run_update(c)
    mu = F32(mu)
    coef = F32(c.coef) if c.clip is not None else F32(1)
    w0 = c.w if mutant == "anchor_is_master" else anchor
    d = f32_sub(w0, c.w) if mutant == "d_sign_flipped" else f32_sub(c.w, w0)
    if skipped:
        g = f32_fma(mu, d, np.zeros(c.n, F32))
    elif mutant == "before_coef":
        g = f32_mul(coef, f32_fma(mu, d, c.g))
    else:
        g = f32_fma(mu, d, f32_mul(coef, c.g))
    if mutant == "tail_skipped":
        tail = np.arange(c.n) >= c.n // 4 * 4
        g = np.where(tail, f32_mul(coef, c.g), g).astype(F32)
    out = run_update(replace(c, g=g, clip=None, coef=1.0, nonfinite=0))
    out["grad"] = np.zeros(c.n, F32) if c.zero_grad else c.g.astype(F32).copy()
    return out


def anchor_for(c: Case, seed: int) -> np.ndarray:
    """An anchor near w (d of every sign and scale, some d = 0 and signed zeros) of the case's size."""
    rng = np.random.default_rng(seed)
    a = (c.w + rng.standard_normal(c.n) * rng.choice([1e-3, 0.3, 5.0], c.n)).astype(F32)
    a[::7] = c.w[::7]                      # d = 0: fma(mu, 0, g) keeps g
    return a


def prox_cases(adam: bool, n: int):
    """Recipe cases with an anchor: no clip and a written clip coefficient, decay on and off, and the
    skipped step (the fixtures ``test_gpu_prox.py`` launches)."""
    cs = recipe_cases(adam, n)
    picked = [cs[0], cs[1], cs[3], cs[4]]
    out = []
    for k, c in enumerate(picked):
        c = replace(c, label=c.label + " prox")
        out.append((c, anchor_for(c, 31 * n + k)))
    c = replace(cs[1], clip="header", nonfinite=1, label=cs[1].label + " prox skipped")
    out.append((c, anchor_for(c, 7 * n)))
    return out


def as_launch(c: Case, o: dict) -> dict:
    """A model output in the form a launch returns it: a skipped step leaves the shadow untouched."""
    o = dict(o)
    if o["shadow"] is None:
        o["shadow"] = np.full(c.n, SH_INIT, np.uint16)
    return o


TEETH_N = [1, 3, 257, 4099]
MUTANTS = ["anchor_is_master", "d_sign_flipped", "before_coef", "tail_skipped", "term_on_skipped_step"]


def test_prox_cases_cover_the_term():
    """The fixtures exercise what the teeth need: a clip coefficient != 1, d != 0, a scalar tail."""
    cs = [c for adam in (False, True) for n in TEETH_N for c, _ in prox_cases(adam, n)]
    assert any(c.clip == "header" and c.coef != 1 and not c.nonfinite for c in cs)
    assert any(c.nonfinite for c in cs) and any(c.n % 4 for c in cs)


def test_mu_zero_anchor_is_the_recipe_update():
    """fma(0, d, g) = g for every finite d and nonzero g; the binding passes no anchor for mu = 0, so
    that a zero gradient keeps its sign (fma(0, d, -0) would be +0)."""
    for c, a in prox_cases(False, 257)[:2]:
        got, ref = prox_update(c, a, 0.0), run_update(c)
        nz = f32_mul(F32(c.coef if c.clip else 1), c.g) != 0      # the gradient the update sees, flushed
        assert (got["w"][nz].view(np.uint32) == ref["w"][nz].view(np.uint32)).all()
    assert math.copysign(1.0, float(f32_fma(F32(0), F32(2.0), F32(-0.0)))) == 1.0


def test_prox_model_is_sgd_on_the_proximal_loss():
    """With IEEE arithmetic the model is one SGD step on loss + mu/2 ||w - w0||^2 in fp64."""
    rng = np.random.default_rng(3)
    n = 999
    w, g, m, v = values(n, 5, moments=False)
    w = (rng.standard_normal(n)).astype(F32)
    g = (rng.standard_normal(n) * 0.1).astype(F32)
    c = Case(False, n, w, g, m, v, lr=0.05, step=1, word=None, zero_grad=True, recipe=True)
    a = (w + rng.standard_normal(n) * 0.2).astype(F32)
    got = prox_update(c, a, MU)["w"].astype(np.float64)
    ref = w.astype(np.float64) - 0.05 * (g.astype(np.float64) + float(F32(MU)) * (w.astype(np.float64) - a))
    assert np.allclose(got, ref, rtol=1e-6, atol=1e-7)


def test_kernel_model_conforms_on_the_gpu_fixtures():
    for adam in (False, True):
        for n in TEETH_N:
            for c, a in prox_cases(adam, n):
                o = prox_update(c, a, MU)
                assert check_update(c, as_launch(c, o), spec=o) == [], c.label


@pytest.mark.parametrize("mutant", MUTANTS)
def test_teeth_every_prox_mistake_fails_a_fixture(mutant):
    caught = []
    for adam in (False, True):
        for n in TEETH_N:
            for c, a in prox_cases(adam, n):
                ref = prox_update(c, a, MU)
                if check_update(c, as_launch(c, prox_update(c, a, MU, mutant)), spec=ref):
                    caught.append(c.label)
    assert caught, mutant


# ------------------------------------------------------------------------------ config and flags
BAD_VALUES = [("prox_mu", b) for b in (-0.5, float("nan"), float("inf"), 1e39)] + \
    [("non_iid_alpha", b) for b in (-0.5, float("nan"), float("inf"))]


@pytest.mark.parametrize("field,bad", BAD_VALUES)
def test_config_rejects_bad_values(field, bad):
    """prox_mu is checked on its fp32 value (1e39 overflows to inf), non_iid_alpha as a double."""
    from bflc_demo_b200.config import FLConfig
    with pytest.raises(ValueError):
        FLConfig(**{field: bad}).validate()
    FLConfig(**{field: 0.25}).validate()


def test_config_picks_prox_mu_from_env_and_json(monkeypatch):
    from bflc_demo_b200.config import FLConfig
    monkeypatch.setenv("BFLC_PROX_MU", "0.125")
    cfg = FLConfig.from_env(model="softmax", dataset="occupancy")
    assert cfg.prox_mu == 0.125
    assert FLConfig.from_json(cfg.to_json()).prox_mu == 0.125


@pytest.mark.parametrize("flag", ["--prox-mu", "--non-iid-alpha"])
@pytest.mark.parametrize("bad", ["-1", "nan", "inf"])
@pytest.mark.parametrize("entry", ["run", "sim"])
def test_bad_flag_exits_with_code_2(entry, flag, bad):
    if entry == "run":
        from bflc_demo_b200.run import main
        argv = ["--model", "mlp", flag, bad]
    else:
        from bflc_demo_b200.host.sim import main
        argv = ["--dataset", "femnist", flag, bad]
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert e.value.code == 2


# ------------------------------------------------------------------------------ host client
def _old_train_pass(model, w, X, y, lr, batch):
    """``HostModel.train_pass`` as it was before the FedProx argument (the mu = 0 reference)."""
    w = w.clone().requires_grad_(True)
    n_batches = X.shape[0] // batch
    cost = 0.0
    for i in range(n_batches):
        xb, yb = X[i * batch:(i + 1) * batch], y[i * batch:(i + 1) * batch]
        loss = torch.nn.functional.cross_entropy(model._logits(model.spec.views(w), xb), yb.long())
        g, = torch.autograd.grad(loss, w)
        with torch.no_grad():
            w -= lr * g
        cost += float(loss.detach()) / n_batches
    return w.detach(), cost


def _host_setup():
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.host.models import HostModel
    sh = femnist_like(1, 200, seed=4, alpha=0.3)[0]
    model = HostModel("mlp", 784, 62, hidden=32, scale_inputs=1 / 255.0)
    return model, model.init(seed=2), sh


def test_host_train_pass_mu_zero_is_unchanged():
    model, w, sh = _host_setup()
    ref, cost_ref = _old_train_pass(model, w, sh.x, sh.y, 0.05, 50)
    got, cost, n = model.train_pass(w, sh.x, sh.y, 0.05, 50)
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32)) and cost == cost_ref and n == 200


def test_host_train_pass_prox_matches_fp64_autograd():
    model, w, sh = _host_setup()
    mu, lr, B = 0.5, 0.05, 50
    got, _, _ = model.train_pass(w, sh.x, sh.y, lr, B, prox_mu=mu)
    w0 = w.double()
    p = w0.clone().requires_grad_(True)
    for i in range(sh.x.shape[0] // B):
        xb, yb = sh.x[i * B:(i + 1) * B], sh.y[i * B:(i + 1) * B]
        v = model.spec.views(p)
        x = xb.double() * model.scale
        h = torch.relu(x @ v["w1"].t() + v["b1"])
        loss = torch.nn.functional.cross_entropy(h @ v["w2"].t() + v["b2"], yb.long()) + \
            mu / 2 * ((p - w0) ** 2).sum()
        g, = torch.autograd.grad(loss, p)
        with torch.no_grad():
            p -= lr * g
    moved = (p.detach() - w0).abs()
    err = (got.double() - p.detach()).abs()
    assert moved.max() > 1e-3
    assert (err <= 1e-4 * moved.max() + 1e-6).all(), float(err.max())
    # the term pulls toward w0: the prox run moves less than the plain one
    plain, _, _ = model.train_pass(w, sh.x, sh.y, lr, B)
    assert (got - w).norm() < (plain - w).norm()


def test_host_sim_occupancy_with_prox_chain_verifies():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.occupancy import split_data
    from bflc_demo_b200.host.models import HostModel
    from bflc_demo_b200.host.sim import run
    cfg = FLConfig.reference_scaled(20, prox_mu=0.01)
    shards, test, _ = split_data(clients_num=cfg.clients)
    led, clients, sponsor, _ = run(cfg, shards, test, model=HostModel("softmax", 5, 2), rounds=3, log=None)
    assert led.epoch() >= 3 and led.verify_chain()
    assert all(c.prox_mu == 0.01 for c in clients)
    assert sum(c.stats["trained"] for c in clients) >= 3 * cfg.needed_updates


def test_host_sim_main_accepts_prox_flags(capsys):
    from bflc_demo_b200.host.sim import main
    main(["--rounds", "2", "--prox-mu", "0.01"])
    assert "chain ok=True" in capsys.readouterr().out


def test_sim_records_non_iid_alpha_in_its_config(monkeypatch):
    """--non-iid-alpha reaches the simulator's FLConfig (the run's record), not only the shards."""
    from bflc_demo_b200.host import sim

    class Seen(Exception):
        pass

    def fake_run(cfg, shards, test, **kw):
        raise Seen(cfg)

    monkeypatch.setattr(sim, "run", fake_run)
    with pytest.raises(Seen) as e:
        sim.main(["--dataset", "femnist", "--clients", "4", "--non-iid-alpha", "0.3", "--prox-mu", "0.02"])
    cfg = e.value.args[0]
    assert cfg.non_iid_alpha == 0.3 and cfg.prox_mu == 0.02


def test_run_rejects_non_iid_alpha_for_bert():
    from bflc_demo_b200.run import main
    with pytest.raises(SystemExit) as e:
        main(["--model", "bert", "--non-iid-alpha", "0.5"])
    assert e.value.code == 2
