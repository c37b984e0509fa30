"""Conformance of what an engine does around its kernels in one round, and from round to round, on one
GPU at world 1 (solo): which shard rows each local step reads (``engine.base.step_rows``), which inputs a
round trains on when the host sends new ones, what optimizer state and step word carry over, and the
round-level numbers the ledger records.

Three oracles:

(a) step replay -- the same trainer driven one step at a time from the host on explicit row slices
    (``FlatMLP`` over cloned buffers: one ``train_epoch_fused`` launch per step with the step word set
    to opt_step + i, which ``test_gpu_trainer_conformance.py`` ties to fp64).  The shard and model are
    that suite's saturated fixture, which makes every float-atomic sum exact, so the engine's state
    equals the replay bit for bit; the loss sum is bounded instead.
(b) epoch unrolling -- ``local_epochs = k`` on a shard trains the same model and loss as one local
    epoch on that shard repeated k times.
(c) round numbers -- the committed model is the upload (solo FedAvg), score = hits / n_val from the
    fp64 argmax, n_samples = S, the model digest, the host mirror page and the step word.

``tests/test_round_spec_host.py`` checks on the CPU that the fixture stays saturated along every
trajectory used here, and that each modelled mistake would move a bf16 weight.
"""
import numpy as np
import pytest
import torch

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.data.synthetic import Shard, cifar_like, femnist_like
from bflc_demo_b200.engine.base import parse_block_record, step_rows
from test_gpu_trainer_conformance import BF16, LR, gamma, mx8_dq, x_bf16
from test_protocol_spec_host import avg_cost_bound, digest
from test_round_spec_host import FRESH_CASES, FRESH_ROUNDS, FUSED_GRID, GRID_ROUNDS, fixture_for

pytestmark = pytest.mark.gpu

PATH_ENV = {  # run path -> (BFLC_E2E_PREFEED, BFLC_E2E_TAGS, BFLC_INPUT_PIPELINE)
    "graph": ("1", "writevalue", "1"), "e2e": ("1", "writevalue", "1"), "e2e-noprefeed": ("0", "writevalue", "1"),
    "e2e-memcpy": ("1", "memcpy", "1"), "e2e-noprefeed-memcpy": ("0", "memcpy", "1"),
    "nopipe": ("1", "writevalue", "0"), "nograph": ("1", "writevalue", "1"), "unfused": ("1", "writevalue", "1")}


def _np(t):
    return t.detach().cpu().numpy()


def fused_engine(monkeypatch, xu8, y, dtype, opt, B, le, path="graph", master=None, val_samples=0):
    """A world-1 FusedEngine on the shard (xu8, y), with ``master`` written over the genesis model
    into every buffer that holds it (as FusedEngine.__init__ writes its own genesis model)."""
    from bflc_demo_b200.engine.fused import FusedEngine
    pre, tags, pipe = PATH_ENV[path]
    monkeypatch.setenv("BFLC_E2E_PREFEED", pre)
    monkeypatch.setenv("BFLC_E2E_TAGS", tags)
    monkeypatch.setenv("BFLC_INPUT_PIPELINE", pipe)
    cfg = FLConfig.for_world(1, model="mlp", hidden=256, batch_size=B, samples_per_client=len(xu8),
                             learning_rate=LR[opt], dtype=dtype, optimizer=opt, local_epochs=le,
                             cuda_graph=path != "nograph", fused_step=path != "unfused", val_samples=val_samples)
    eng = FusedEngine(cfg, Shard(xu8, y.long(), 62))
    assert eng.fused_step == (path != "unfused")
    if master is not None:
        m = master.to(eng.dev)
        o, P, hv = eng.layout.offsets, eng.n_params, eng.heap.view
        for t in (eng.work_master, eng.global_master, *(hv(o[f"upload_master{p}"], [P], torch.float32) for p in (0, 1))):
            t.copy_(m)
        for t in (eng.work_shadow, eng.global_shadow, *(hv(o[f"upload_shadow{p}"], [P], BF16) for p in (0, 1))):
            t.copy_(m.bfloat16())
        if eng.fp8:
            for off in eng.upq_off:
                eng.trainer.quantize_weights(eng.global_master, hv(off, [eng.blob_bytes], torch.uint8))
            eng.trainer.quantize_weights()
        torch.cuda.synchronize()
    return eng


def plan_words(eng):
    """(opt_step, opt_total): the step base the last round ran with and the running total."""
    sz, pb = eng.sz, eng.plan_bytes.cpu()

    def word(off):
        return int(pb[off:off + 4].view(torch.int32)[0])
    return word(sz["plan_opt_step_off"]), word(sz["plan_opt_total_off"])


class Replay:
    """The engine's trainer replayed step by step from the host, on its own buffers."""

    def __init__(self, eng, master, m=None, v=None):
        from bflc_demo_b200.models.mlp import FlatMLP
        cfg = eng.cfg
        self.eng, self.B, self.fp8 = eng, cfg.batch_size, eng.fp8
        self.step = torch.zeros(1, device="cuda", dtype=torch.int32)
        mm = master.to("cuda").clone()
        self.tr = FlatMLP(eng.spec, mm, mm.bfloat16(), torch.zeros_like(mm), self.B, optimizer=cfg.optimizer,
                          lr=cfg.learning_rate, fp8=self.fp8, step_dev_ptr=self.step.data_ptr())
        if m is not None:
            self.tr.m.copy_(m)
            self.tr.v.copy_(v)
        self.bar = torch.zeros(1, device="cuda", dtype=torch.int32)

    def clone(self):
        tr = self.tr
        return Replay(self.eng, tr.master, tr.m, tr.v)

    def inputs(self, xu8, y):
        """The round's inputs as the engine converts them (prep_inputs), on the device."""
        from bflc_demo_b200._native import C
        xu = xu8.to("cuda")
        xb = torch.empty(xu.shape, device="cuda", dtype=BF16)
        xdq = torch.empty(xu.shape, device="cuda", dtype=BF16) if self.fp8 else None
        C().prep_inputs(xu, xb, None, None, 1.0 / 255.0, xdq)
        return xb, xdq, y.to("cuda", torch.int32)

    def round(self, xu8, y, S, steps, opt_step):
        """One round's local steps on the shard (xu8, y) from step word opt_step."""
        tr, B = self.tr, self.B
        xb, xdq, yd = self.inputs(xu8, y)
        tr.loss_sum.zero_()
        if self.fp8:
            tr.quantize_weights()
        fused = self.eng.fused_step
        self.step.fill_(opt_step)
        for i in range(steps):
            r = step_rows(i, B, S)
            if fused:
                self.step.fill_(opt_step + i)
                self.bar.zero_()
                tr.train_epoch_fused(xb[r], yd[r], 1, self.bar.data_ptr(), **({"x_dq": xdq[r]} if self.fp8 else {}))
            else:
                tr.forward_backward(xb[r], yd[r])
                tr.optimizer_step(i + 1)
        torch.cuda.synchronize()
        return float(tr.loss_sum)


def check_round(eng, rep, r, xu8, y, loss_rep, fresh_inputs):
    """Oracles (a) and (c) after round r (0 = capture()'s warm-up) trained on the shard (xu8, y)."""
    torch.cuda.synchronize()
    B, S, steps = eng.cfg.batch_size, eng.S, eng.steps
    st = eng.read_state()
    assert st["epoch"] == r + 1
    opt_step, opt_total = plan_words(eng)
    assert (opt_step, opt_total) == (r * steps, (r + 1) * steps), (r, opt_step, opt_total)
    if fresh_inputs:      # the resident inputs are the spec conversion of this round's data
        assert torch.equal(eng.x_bf.cpu(), x_bf16(_Fx(xu8))), f"round {r}: x_bf"
        assert torch.equal(eng.y.cpu(), y.to(torch.int32)), f"round {r}: y"
        if eng.fp8:
            assert torch.equal(eng.x_dq.cpu(), mx8_dq(xu8.float() * np.float32(1 / 255)).to(BF16)), f"round {r}: x_dq"
    # (a): the engine's model and optimizer state are the replay's, bit for bit
    o, P = eng.layout.offsets, eng.n_params
    up = eng.heap.view(o[f"upload_master{r & 1}"], [P], torch.float32)
    assert torch.equal(up, rep.tr.master), f"round {r}: upload != replay ({int((up != rep.tr.master).sum())} differ)"
    assert torch.equal(eng.global_master, up), f"round {r}: committed model != the upload"
    assert torch.equal(eng.global_shadow, rep.tr.shadow), f"round {r}: committed shadow"
    if eng.cfg.optimizer == "adam":
        assert torch.equal(eng.trainer.m, rep.tr.m) and torch.equal(eng.trainer.v, rep.tr.v), f"round {r}: Adam moments"
    # the loss: the replay's sum within its float-atomic reordering, and the recorded avg_cost
    loss = float(eng.loss_sum)
    assert abs(loss - loss_rep) <= gamma(steps * B + 32) * abs(loss_rep), (r, loss, loss_rep)
    ring = eng.ring_bytes.cpu().numpy()
    ep, seq, rec = parse_block_record(ring, (r % eng.cfg.ring_slots) * eng.sz["BlockRecord"], 1)
    assert (ep, seq) == (r, r + 1)
    c, b = avg_cost_bound(loss, steps * B)
    assert abs(rec["avg_cost"][0] - c) <= b, (r, rec["avg_cost"][0], c)
    # (c): n_samples is one epoch's rows whatever the local epochs; score = fp64 hits / n_val
    assert rec["n_samples"][0] == S, (rec["n_samples"], S)
    n_val = eng.n_val
    v = eng.spec.views(eng.global_master.double().cpu())
    xv = x_bf16(_Fx(xu8[:n_val])).double()
    z = torch.relu(xv @ v["w1"].bfloat16().double().t() + v["b1"]).bfloat16().double() @ v["w2"].bfloat16().double().t() + v["b2"]
    top2 = z.topk(2, dim=1)
    assert float((top2.values[:, 0] - top2.values[:, 1]).min()) > 16, "validation rows not decided by a margin"
    hits = int((top2.indices[:, 0] == y[:n_val].long()).sum())
    c, b = avg_cost_bound(hits, n_val)
    assert abs(st["median"][0] - c) <= b, (r, st["median"][0], hits, n_val)
    g = _np(eng.global_master)
    assert st["model_digest"] == digest(g) == rec["model_digest"], f"round {r}: digest"
    if eng.pipelined_input and eng.graph_pipe is not None and eng.mirror_result and r > 0 and fresh_inputs:
        mirror = _np(eng.mirror).view(np.uint8)[:eng.sz["RoundState"]]
        assert bytes(mirror) == bytes(_np(eng.state_bytes)), f"round {r}: mirror page"
    return st


class _Fx:
    """The fields x_bf16 reads off a fixture."""

    def __init__(self, xu8):
        self.xu8 = xu8


def run_fused_case(monkeypatch, path, dtype, opt, B, E, le, rounds, fresh):
    """Warm-up round + rounds - 1 more on the given run path, each checked against the replay.
    Returns the engine, its per-round states and the fixture."""
    fx = fixture_for(B, E, rounds if fresh else 1)
    S = E * B
    shards = [(fx.xu8[k * S:(k + 1) * S].contiguous(), fx.y[k * S:(k + 1) * S].contiguous())
              for k in range(rounds if fresh else 1)]
    eng = fused_engine(monkeypatch, *shards[0], dtype, opt, B, le, path, master=fx.master)
    assert eng.S == S and eng.steps == E * le
    rep = Replay(eng, fx.master)
    pinned = [(x.pin_memory(), y.to(torch.int32).pin_memory()) for x, y in shards]
    for r in range(rounds):
        k = r if fresh else 0
        before = rep.clone() if fresh and r > 0 else None
        if r == 0:
            eng.capture()
        elif fresh:
            eng.run_round_e2e(*pinned[k])
        else:
            eng.run_round()
        opt_step = r * eng.steps
        loss = rep.round(*shards[k], S, eng.steps, opt_step)
        check_round(eng, rep, r, *shards[k], loss, fresh and r > 0)
        if before is not None:   # teeth: the previous round's data trains a different model
            before.round(*shards[k - 1], S, eng.steps, opt_step)
            assert not torch.equal(before.tr.master, eng.global_master), f"round {r}: stale inputs not visible"
    assert eng.drain_blocks() == []
    if eng.pipelined_input:
        assert int(eng.in_err) == 0
    return eng, fx


@pytest.mark.parametrize("dtype,opt,B,E,le", FUSED_GRID, ids=[f"{d}-{o}-B{b}-E{e}-le{l}" for d, o, b, e, l in FUSED_GRID])
def test_fused_rounds_match_step_replay(monkeypatch, dtype, opt, B, E, le):
    """capture()'s warm-up round and a graph round on the resident shard against the replay."""
    eng, _ = run_fused_case(monkeypatch, "graph", dtype, opt, B, E, le, GRID_ROUNDS, fresh=False)
    assert eng.pipelined_input == (E <= 16)
    print(f"[round conformance] graph {dtype} {opt} B={B} E={E} local_epochs={le}: bit-equal to the replay")


@pytest.mark.parametrize("path,dtype,opt,B,E,le", FRESH_CASES,
                         ids=[f"{p}-{d}-{o}-B{b}-E{e}-le{l}" for p, d, o, b, e, l in FRESH_CASES])
def test_fused_fresh_inputs_every_round(monkeypatch, path, dtype, opt, B, E, le):
    """run_round_e2e with a new fixture slice every round: the resident inputs, the model and the
    Adam state follow that round's data on every run path."""
    eng, _ = run_fused_case(monkeypatch, path, dtype, opt, B, E, le, FRESH_ROUNDS, fresh=True)
    assert eng.pipelined_input == (path not in ("nopipe", "unfused"))
    print(f"[round conformance] {path} {dtype} {opt} B={B} E={E} local_epochs={le}: "
          f"pipelined={eng.pipelined_input}, bit-equal to the replay for {FRESH_ROUNDS} rounds")


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_pipelined_and_plain_rounds_leave_identical_state(monkeypatch, dtype):
    B, E, le, opt = 128, 4, 2, "adam"
    ends = []
    for path in ("e2e", "nopipe"):
        eng, _ = run_fused_case(monkeypatch, path, dtype, opt, B, E, le, FRESH_ROUNDS, fresh=True)
        ends.append([t.clone() for t in (eng.global_master, eng.global_shadow, eng.trainer.m, eng.trainer.v,
                                         eng.x_bf, eng.y)])
        del eng
    for a, b in zip(*ends):
        assert torch.equal(a, b)


def test_host_inputs_are_checked_against_the_resident_ones(monkeypatch):
    B, E = 128, 2
    fx = fixture_for(B, E, 1)
    eng = fused_engine(monkeypatch, fx.xu8, fx.y, "bf16", "sgd", B, 1, "e2e", master=fx.master)
    eng.capture()
    hx, hy = eng.host_x, eng.host_y
    for bad_x, bad_y in ((hx[:B].clone().pin_memory(), hy), (hx, hy[:B].clone().pin_memory()),
                         (hx.clone(), hy), (hx, hy.long().pin_memory()), (hx.t().contiguous().t(), hy)):
        with pytest.raises(ValueError, match="run_round_e2e"):
            eng.run_round_e2e(bad_x, bad_y)
    eng.run_round_e2e(hx, hy)
    assert eng.read_state()["epoch"] == 2 and eng.drain_blocks() == []


def test_trainer_refuses_inputs_shorter_than_an_epoch():
    """The binding compares x, x_dq and the labels with one local epoch's rows before launch."""
    from bflc_demo_b200.models.mlp import FlatMLP, mlp_spec
    spec = mlp_spec(784, 256, 62)
    B = 128
    m = torch.zeros(spec.total, device="cuda")
    tr = FlatMLP(spec, m, m.bfloat16(), torch.zeros_like(m), B)
    bar = torch.zeros(1, device="cuda", dtype=torch.int32)
    x = torch.zeros(2 * B, 784, device="cuda", dtype=BF16)
    y = torch.zeros(2 * B, device="cuda", dtype=torch.int32)
    for args, kw in (((x[:B], y, 2), {}), ((x, y[:B], 2), {}), ((x, y, 3), {"epoch_rows": 3 * B}),
                     ((x, y, 1), {"epoch_rows": 2 * B}), ((x, y, 4), {"epoch_rows": B + 8})):
        with pytest.raises(RuntimeError, match="mlp_round"):
            tr.train_epoch_fused(*args, bar.data_ptr(), **kw)
    torch.cuda.synchronize()
    assert int(torch.count_nonzero(m)) == 0


@pytest.mark.parametrize("dtype,opt,B,E,le", [("bf16", "sgd", 128, 2, 3), ("bf16", "adam", 512, 2, 2),
                                              ("fp8", "adam", 128, 4, 2), ("fp8", "sgd", 128, 1, 3)])
def test_local_epochs_unroll_to_a_repeated_shard(monkeypatch, dtype, opt, B, E, le):
    """(b): local_epochs = k on a shard == one local epoch on that shard repeated k times."""
    fx = fixture_for(B, E, 1)
    k = le
    a = fused_engine(monkeypatch, fx.xu8, fx.y, dtype, opt, B, k, "graph", master=fx.master)
    b = fused_engine(monkeypatch, fx.xu8.repeat(k, 1), fx.y.repeat(k), dtype, opt, B, 1, "graph", master=fx.master)
    assert a.steps == b.steps == E * k
    out = []
    for eng in (a, b):
        eng.capture()
        eng.run_round()
        torch.cuda.synchronize()
        out.append((eng.global_master.clone(), float(eng.loss_sum),
                    (eng.trainer.m.clone(), eng.trainer.v.clone()) if opt == "adam" else None))
    (wa, la, ma), (wb, lb, mb) = out
    assert torch.equal(wa, wb)
    if opt == "adam":
        assert torch.equal(ma[0], mb[0]) and torch.equal(ma[1], mb[1])
    assert abs(la - lb) <= gamma(E * k * B + 32) * abs(lb), (la, lb)


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_row_edges_tail_rows_and_short_validation(monkeypatch, opt):
    """bf16: a shard of S + 40 rows trains on its first S rows and validates all of them; then
    val_samples < len(shard) validates only the first val_samples rows."""
    B, E, le = 128, 2, 2
    fx = fixture_for(B, E + 1, 1)
    n = E * B + 40
    xu8, y = fx.xu8[:n].contiguous(), fx.y[:n].contiguous()
    for val in (0, E * B // 2 + 8):
        eng = fused_engine(monkeypatch, xu8, y, "bf16", opt, B, le, "graph", master=fx.master, val_samples=val)
        assert eng.S == E * B and not eng.pipelined_input and eng.n_val == (val or n)
        rep = Replay(eng, fx.master)
        for r in range(GRID_ROUNDS):
            if r == 0:
                eng.capture()
            else:
                eng.run_round()
            loss = rep.round(xu8, y, eng.S, eng.steps, r * eng.steps)
            check_round(eng, rep, r, xu8, y, loss, False)
        assert eng.drain_blocks() == []
        del eng


# ------------------------------------------------------------------------------ generic engine
def _generic(net_name, opt, le, shard_rows, B=64, seed=3, repeat=1):
    """A world-1 GenericFedEngine on a seeded shard (``repeat``: the shard repeated that many times)."""
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5, MLPNet
    if net_name == "mlp":
        net, shard, kw = MLPNet(784, 256, 62), femnist_like(1, shard_rows, seed=seed)[0], dict(model="mlp")
    else:
        net, shard = LeNet5(10), cifar_like(1, shard_rows, seed=seed, alpha=0.0)[0]
        kw = dict(model="lenet5", dataset="cifar10")
    if repeat > 1:
        shard = Shard(shard.x.repeat(repeat, *[1] * (shard.x.dim() - 1)), shard.y.repeat(repeat), shard.n_classes)
    cfg = FLConfig.for_world(1, batch_size=B, samples_per_client=len(shard), learning_rate=LR[opt],
                             optimizer=opt, local_epochs=le, **kw)
    return GenericFedEngine(cfg, net, shard)


def generic_replay(eng, start, m, v, opt_step, mutant=None):
    """The generic engine's local training driven from the host on cloned buffers: net.loss and
    optim_step along the row schedule, DropoutRNG keys from the step word."""
    from bflc_demo_b200.ops.nn import DropoutRNG
    cfg, B, S = eng.cfg, eng.cfg.batch_size, eng.S
    E = S // B
    master = start.clone()
    shadow = master.bfloat16()
    grad = torch.zeros_like(master)
    m = None if m is None else (torch.zeros_like(m) if mutant == "moments_reset" else m.clone())
    v = None if v is None else (torch.zeros_like(v) if mutant == "moments_reset" else v.clone())
    word = torch.full((1,), 0 if mutant == "t_restart" else opt_step, device=eng.dev, dtype=torch.int32)
    bound = eng.net.bind(master, shadow, grad)
    for i in range(eng.steps):
        j = min(i, E - 1) if mutant == "wrap_last" else 0 if mutant == "step0_rows" else i
        r = step_rows(j, B, S)
        loss = eng.net.loss(bound, eng.x[r], eng.y[r], rng=DropoutRNG(eng.dropout_seed, word, i))
        loss.backward()
        eng.mod.optim_step(cfg.optimizer == "adam", master, grad, shadow, m, v, cfg.learning_rate, 0.0, 0.9,
                           0.999, 1e-8, i + 1, word.data_ptr(), 0, True)
    torch.cuda.synchronize()
    return master, m, v


def gap(a, b, start):
    """||a - b|| relative to the round's update ||b - start|| (L2 over the parameters).

    LeNet-5's split-K weight gradients add fp32 partial sums with atomics, so two eager runs of a round
    differ.  Under SGD by an ulp here and there; under Adam the difference is heavy-tailed: where a
    gradient is noise-dominated and v is still small, m / sqrt(v) follows the noise, and one such
    weight perturbs every later step.  Between eager runs of one round on an H100 the largest
    elementwise difference ranged from 7e-9 to 9e-6, and about one run in ten took an alternative
    trajectory 1.1e-3 away in this measure.  A wrong schedule or carried state changes the update
    itself: the modelled mistakes measured 0.18 to 1.5."""
    return float((a - b).norm() / (b - start).norm())


# the smallest tolerance on ``gap`` between a nondeterministic engine round and its replay: above the
# alternative trajectory an engine round may take, far below the modelled mistakes
GAP_FLOOR = 5e-3


GENERIC = [(n, o, le) for n in ("mlp", "lenet5") for o in ("sgd", "adam") for le in (1, 2)]
N_REPLAYS = 4


@pytest.mark.parametrize("net_name,opt,le", GENERIC, ids=[f"{n}-{o}-le{l}" for n, o, l in GENERIC])
def test_generic_rounds_match_host_replay(net_name, opt, le):
    """Three rounds (capture()'s warm-up, then graph rounds), each against host replays from the round's
    committed model and the engine's Adam state.  When the replays agree bit for bit (the MLP), the
    engine must equal them, moments included; otherwise its ``gap`` to a replay is within the tolerance
    max(4x the replays' largest pairwise gap, GAP_FLOOR).  Each modelled mistake lands more than 0, at
    least 100x the replays' spread and 10x the tolerance away."""
    eng = _generic(net_name, opt, le, 256)
    assert eng.S == 256 and eng.steps == 4 * le
    adam = opt == "adam"
    for r in range(3):
        start = eng.global_master.clone()
        m0, v0 = (eng.m.clone(), eng.v.clone()) if adam else (None, None)
        eng.capture() if r == 0 else eng.run_round()
        torch.cuda.synchronize()
        opt_step, opt_total = plan_words(eng)
        assert (opt_step, opt_total) == (r * eng.steps, (r + 1) * eng.steps)
        reps = [generic_replay(eng, start, m0, v0, opt_step) for _ in range(N_REPLAYS)]
        a, am, av = reps[0]
        got = eng.global_master
        if all(torch.equal(a, x[0]) for x in reps[1:]):
            spread = tol = 0.0
            assert torch.equal(got, a), f"round {r}: {int((got != a).sum())} weights differ from the replay"
            if adam:
                assert torch.equal(eng.m, am) and torch.equal(eng.v, av), f"round {r}: Adam moments"
            how = "bit-equal"
        else:
            spread = max(gap(x[0], y[0], start) for i, x in enumerate(reps) for y in reps[i + 1:])
            tol = max(4 * spread, GAP_FLOOR)
            err = gap(got, a, start)
            assert err <= tol, (r, err, spread)
            how = f"gap {err:.3g}, replays' spread {spread:.3g}"
        mutants = ["step0_rows"] + (["wrap_last"] if le > 1 else []) + (["moments_reset", "t_restart"]
                                                                          if adam and r > 0 else [])
        for mu in mutants:
            w = generic_replay(eng, start, m0, v0, opt_step, mutant=mu)[0]
            d = gap(w, got, start)
            assert d > 0 and d >= 100 * spread and d >= 10 * tol, (r, mu, d, spread, tol)
            how += f", {mu} {d:.3g}"
        print(f"[round conformance] generic {net_name} {opt} local_epochs={le} round {r}: {how}")
    assert eng.drain_blocks() == []


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_generic_local_epochs_unroll_to_a_repeated_shard(opt):
    """(b) for the generic engine: two local epochs == the shard repeated twice, one epoch, bit for bit
    (the MLP's training is bit-reproducible)."""
    a = _generic("mlp", opt, 2, 128)
    b = _generic("mlp", opt, 1, 128, repeat=2)
    assert a.steps == b.steps == 4
    for eng in (a, b):
        eng.run_round()
    torch.cuda.synchronize()
    assert torch.equal(a.global_master, b.global_master)
    if opt == "adam":
        assert torch.equal(a.m, b.m) and torch.equal(a.v, b.v)
    la, lb = a.read_state()["global_loss"], b.read_state()["global_loss"]
    assert abs(la - lb) <= 1e-6 * abs(lb), (la, lb)


# ------------------------------------------------------------------------------ NCCL baseline
def test_baseline_local_epochs_train_full_batches_and_unroll():
    from bflc_demo_b200.engine.nccl_baseline import NcclBaselineEngine
    B, S = 128, 256
    shard = femnist_like(1, S, seed=9)[0]
    res = []
    for le, sh in ((2, shard), (1, Shard(shard.x.repeat(2, 1), shard.y.repeat(2), shard.n_classes))):
        cfg = FLConfig.for_world(1, hidden=256, batch_size=B, samples_per_client=len(sh), learning_rate=0.05,
                                 cuda_graph=False, local_epochs=le)
        eng = NcclBaselineEngine(cfg, sh, rank=0, world=1, device=0)
        assert eng.steps == 4
        rb = eng.run_round()
        torch.cuda.synchronize()
        res.append((eng.global_w.clone(), rb["global_loss"]))
        del eng
    (wa, la), (wb, lb) = res
    assert torch.equal(wa, wb)
    assert abs(la - lb) <= 1e-6 * abs(lb)
