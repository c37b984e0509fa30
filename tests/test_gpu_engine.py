"""Single-GPU end-to-end: fused engine rounds, host-ledger re-execution, learning progress,
parity with the NCCL/cuBLAS baseline engine (world = 1, solo mode)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_fused_engine_solo_rounds_learn_and_chain():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    cfg = FLConfig.for_world(1, hidden=256, batch_size=128, samples_per_client=1024,
                             learning_rate=0.05)
    shard = femnist_like(1, 1024, seed=3)[0]
    eng = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    acc0 = eng.evaluate(shard)
    eng.capture()
    losses = []
    for _ in range(8):
        losses.append(eng.run_round_e2e()["global_loss"])
    assert eng.drain_blocks() == []
    assert eng.host_ledger.n_blocks() == 9 and eng.host_ledger.verify_chain()
    assert losses[-1] < losses[0]
    assert eng.evaluate(shard) > acc0 + 0.2
    blk = eng.host_ledger.blocks()[-1]
    assert blk["from_device"] and blk["selected"] == [0] and blk["device_digest"] != 0


def test_fused_engine_two_gemm_validation():
    """hidden != 256 has no one-launch validation kernel: the committee validates with two grouped
    GEMMs (fwd1 + relu -> h_val, fwd2 + argmax epilogue).  Their counts agree with a PyTorch
    forward of the uploaded candidate to 1 % of the validation rows, round after round."""
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    cfg = FLConfig.for_world(1, hidden=128, batch_size=128, samples_per_client=1024,
                             learning_rate=0.05)
    shard = femnist_like(1, 1024, seed=3)[0]
    eng = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    assert not eng.val_chain
    eng.capture()
    o, losses = eng.layout.offsets, []
    for _ in range(4):
        eng.run_round()
        torch.cuda.synchronize()
        st = eng.read_state()
        losses.append(st["global_loss"])
        par = (st["epoch"] - 1) & 1
        w = eng.spec.views(eng.heap.view(o[f"upload_shadow{par}"], [eng.n_params], torch.bfloat16))
        b = eng.spec.views(eng.heap.view(o[f"upload_master{par}"], [eng.n_params], torch.float32))
        x = eng.x_bf[: eng.n_val].double()
        h = torch.relu(x @ w["w1"].double().t() + b["b1"].double()).to(torch.bfloat16).double()
        pred = (h @ w["w2"].double().t() + b["b2"].double()).argmax(1)
        want = int((pred == eng.y[: eng.n_val].long()).sum())
        got = int(eng.val_correct[0])
        assert abs(got - want) <= 0.01 * eng.n_val, (got, want)
        assert abs(st["median"][0] - got / eng.n_val) < 1e-6
    assert eng.drain_blocks() == []
    assert losses[-1] < losses[0]


def test_fused_matches_nccl_baseline_one_round():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    from bflc_demo_b200.engine.nccl_baseline import NcclBaselineEngine
    cfg = FLConfig.for_world(1, hidden=256, batch_size=128, samples_per_client=512,
                             learning_rate=0.05, cuda_graph=False)
    shard = femnist_like(1, 512, seed=5)[0]
    a = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    b = NcclBaselineEngine(cfg, shard, rank=0, world=1, device=0)
    a.run_round()
    torch.cuda.synchronize()
    b.x_bf.copy_(b.x_u8.to(torch.bfloat16) * (1.0 / 255.0))
    rb = b.run_round()
    sa = a.read_state()
    assert sa["epoch"] == rb["epoch"] == 1
    assert abs(sa["global_loss"] - rb["global_loss"]) < 2e-2 * max(1.0, rb["global_loss"])
    wa, wb = a.global_master, b.global_w
    assert ((wa - wb).norm() / wb.norm()).item() < 2e-2


def test_checkpoint_resume_continues_the_chain(tmp_path):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    from bflc_demo_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    cfg = FLConfig.for_world(1, hidden=256, batch_size=128, samples_per_client=512,
                             learning_rate=0.05, optimizer="adam")
    shard = femnist_like(1, 512, seed=3)[0]
    a = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    a.capture()
    for _ in range(3):
        a.run_round()
    info = save_checkpoint(str(tmp_path / "ck.pt"), a)
    assert info["epoch"] == 4 and info["blocks"] == 4
    w_saved = a.global_master.clone()
    last_hash = a.host_ledger.blocks()[-1]["hash"]
    b = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    got = load_checkpoint(str(tmp_path / "ck.pt"), b)
    assert got["epoch"] == 4 and torch.equal(b.global_master, w_saved)
    b.capture()                      # eager round 4 -> 5, then graph
    b.run_round()
    assert b.drain_blocks() == []
    blocks = b.host_ledger.blocks()
    assert len(blocks) == 6 and blocks[4]["prev_hash"] == last_hash and b.host_ledger.verify_chain()
    assert b.read_state()["epoch"] == 6
    # the end-to-end path after a restore that happened AFTER capture (run.py's order): its cached
    # epoch must be re-learnt, then the pinned mirror page takes over again
    c = FusedEngine(cfg, shard, rank=0, world=1, device=0)
    c.capture()
    c.run_round_e2e()
    load_checkpoint(str(tmp_path / "ck.pt"), c)
    assert [c.run_round_e2e()["epoch"] for _ in range(3)] == [5, 6, 7]
    assert c.drain_blocks() == [] and c.host_ledger.verify_chain()


def test_generic_engine_lenet_solo_and_tracing():
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import cifar_like
    from bflc_demo_b200.engine.generic import GenericFedEngine
    from bflc_demo_b200.models.nets import LeNet5
    from bflc_demo_b200.utils.tracing import PhaseTimer
    cfg = FLConfig.for_world(1, batch_size=64, samples_per_client=256, learning_rate=0.05,
                             model="lenet5", dataset="cifar10")
    shard = cifar_like(1, 256, seed=2, alpha=0.0)[0]
    eng = GenericFedEngine(cfg, LeNet5(10), shard, rank=0, world=1, device=0)
    acc0 = eng.evaluate(shard)
    assert 0.0 <= acc0 <= 1.0
    timer = PhaseTimer()
    losses = []
    for _ in range(6):
        with timer.phase("round"):
            eng.run_round()
        losses.append(eng.read_state()["global_loss"])
    assert eng.drain_blocks() == [] and eng.host_ledger.n_blocks() == 6
    assert losses[-1] < losses[0]          # the aggregated trainers' mean cost falls
    s = timer.summary()
    assert s["round"]["count"] == 6 and s["round"]["mean_ms"] > 0
