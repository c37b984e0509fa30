"""Host-side specification of what an engine trains on in one round, and across rounds.

* The row schedule (``engine.base.step_rows``): local step i of a round reads rows
  [(i mod E) B, (i mod E) B + B), E = S / B the whole batches of the shard, so local epoch k > 0
  repeats epoch 0's batches in order and no step reads past the epoch's rows.
* ``FLConfig`` refuses fewer than one local epoch.
* The round trajectories of ``test_gpu_round_conformance.py`` as an fp64 emulation on the trainer's
  operands (``sat_guard`` of the trainer suite): the saturated fixture keeps every float-atomic sum of
  the persistent trainer exact along each of them, which is what lets the GPU suite compare the engine
  with a step-by-step replay bit for bit.
* Teeth: each modelled mistake in the schedule, the round's data or the optimizer state carried from
  round to round moves at least one bf16 weight of the fp64 end state, so the bit-exact GPU
  comparison would catch it.
"""
import pytest
import torch

from bflc_demo_b200.config import FLConfig
from bflc_demo_b200.engine.base import step_rows
from test_gpu_trainer_conformance import rne_bf16, sat_fixture, sat_guard

# fused-engine cases: (dtype, optimizer, batch, E = batches per local epoch, local epochs)
FUSED_GRID = [(d, o, B, E, le) for d in ("bf16", "fp8") for o in ("sgd", "adam") for B in (128, 512)
              for E in (1, 2, 4) for le in (1, 2, 3)]
GRID_ROUNDS = 2          # the warm-up round of capture() and one graph round, on the resident shard
# run paths fed a fresh slice of the fixture every round: (path, dtype, optimizer, batch, E, local epochs)
E2E_PATHS = ("e2e", "e2e-noprefeed", "e2e-memcpy", "e2e-noprefeed-memcpy", "nopipe", "nograph")
FRESH_CASES = ([(p, d, o, 128, 4, 2) for p in E2E_PATHS for d in ("bf16", "fp8") for o in ("sgd", "adam")]
               + [("unfused", "bf16", o, 128, 4, 2) for o in ("sgd", "adam")]
               + [("e2e", d, "adam", 512, 2, 3) for d in ("bf16", "fp8")])
FRESH_ROUNDS = 5         # the warm-up round on slice 0, then four run_round_e2e rounds on slices 1..4

MUTANTS = ("wrap_last", "prev_data", "step0_rows", "moments_reset", "t_restart", "warmup_uncounted")


def fixture_for(B, E, rounds_of_data, seed_extra=0):
    """The saturated fixture of a case: ``rounds_of_data`` shards of E batches of B rows."""
    return sat_fixture(B, E * rounds_of_data, seed=B + 10 * E + 1000 * rounds_of_data + seed_extra)


def round_rows(B, E, le, data_round, mutant=None):
    """Row slices of one round's E * le local steps over the fixture, the round's data being its
    ``data_round``-th shard of E batches."""
    S, base = E * B, data_round * E * B
    out = []
    for i in range(E * le):
        if mutant == "wrap_last":        # later epochs repeat the last batch
            i = min(i, E - 1)
        elif mutant == "step0_rows":     # every step reads step 0's rows
            i = 0
        r = step_rows(i, B, S)
        out.append(slice(base + r.start, base + r.stop))
    return out


def trajectory(fx, fp8, opt, B, E, le, rounds, fresh, mutant=None):
    """fp64 emulation of ``rounds`` solo rounds (the first one is capture()'s warm-up): round r trains
    on shard r of the fixture when ``fresh``, else on shard 0; the committed model is the upload
    (solo FedAvg), Adam's moments carry over and its step count continues from the plan's step word,
    which the warm-up round advances too.  Returns the end state {"p", "m", "v"} (sat_guard asserts the
    fixture's guards at every step)."""
    steps = E * le
    carry = {}
    for r in range(rounds):
        data = r if fresh else 0
        if mutant == "prev_data" and fresh and r > 0:
            data = r - 1
        if mutant == "moments_reset" and "m" in carry:
            carry["m"] = {k: torch.zeros_like(t) for k, t in carry["m"].items()}
            carry["v"] = {k: torch.zeros_like(t) for k, t in carry["v"].items()}
        base = r * steps
        if mutant == "t_restart":
            base = 0
        elif mutant == "warmup_uncounted":
            base = max(r - 1, 0) * steps
        sat_guard(fx, fp8, opt, base, rows=round_rows(B, E, le, data, mutant), carry=carry)
    return carry


# ------------------------------------------------------------------------------ the schedule
def test_step_rows_wraps_whole_epochs():
    B = 32
    # E = 1: every step reads the one batch
    assert [step_rows(i, B, B) for i in range(5)] == [slice(0, B)] * 5
    # E = 3, four local epochs: batches 0 1 2 0 1 2 ...
    got = [step_rows(i, B, 3 * B).start // B for i in range(12)]
    assert got == [0, 1, 2] * 4
    # the generic engine's earlier rule (i * B) % S, for every step of several epochs
    for E in (1, 2, 5, 16):
        for i in range(4 * E):
            r = step_rows(i, B, E * B)
            assert r.start == (i * B) % (E * B) and r.stop - r.start == B
            assert r.stop <= E * B


def test_config_refuses_fewer_than_one_local_epoch():
    for le in (0, -1):
        with pytest.raises(ValueError, match="local_epochs"):
            FLConfig.for_world(1, local_epochs=le)
    with pytest.raises(ValueError, match="local_epochs"):
        FLConfig.for_world(1, local_epochs=1.5)
    assert FLConfig.for_world(1, local_epochs=3).local_epochs == 3


# --------------------------------------------------------------- trajectories of the GPU suite
@pytest.mark.parametrize("dtype,opt,B,E,le", FUSED_GRID, ids=[f"{d}-{o}-B{b}-E{e}-le{l}" for d, o, b, e, l in FUSED_GRID])
def test_sat_guard_holds_on_grid_trajectories(dtype, opt, B, E, le):
    fx = fixture_for(B, E, 1)
    trajectory(fx, dtype == "fp8", opt, B, E, le, GRID_ROUNDS, fresh=False)


FRESH_TRAJECTORIES = sorted({c[1:] for c in FRESH_CASES})


@pytest.mark.parametrize("dtype,opt,B,E,le", FRESH_TRAJECTORIES,
                         ids=[f"{d}-{o}-B{b}-E{e}-le{l}" for d, o, b, e, l in FRESH_TRAJECTORIES])
def test_sat_guard_holds_on_fresh_input_trajectories(dtype, opt, B, E, le):
    """Every run path of a (dtype, optimizer, B, E, local epochs) case is fed the same slices."""
    fx = fixture_for(B, E, FRESH_ROUNDS)
    trajectory(fx, dtype == "fp8", opt, B, E, le, FRESH_ROUNDS, fresh=True)


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_sat_guard_holds_on_the_row_edge_shards(opt):
    """A shard of S + 40 rows (cut from a fixture of E + 1 batches) trains on its first S rows."""
    B, E = 128, 2
    fx = fixture_for(B, E + 1, 1)
    trajectory(fx, False, opt, B, E, 2, GRID_ROUNDS, fresh=False)


# ------------------------------------------------------------------------------ teeth
@pytest.mark.parametrize("mutant", MUTANTS)
def test_every_modelled_mistake_moves_a_bf16_weight(mutant):
    """Bit-exact comparison on the GPU catches each mistake: its fp64 end state rounds to a different
    bf16 weight somewhere.  Adam, fresh data, E = 2 and two local epochs exercise every mutant."""
    B, E, le, rounds = 128, 2, 2, 3
    fx = fixture_for(B, E, rounds, seed_extra=5)
    want = trajectory(fx, False, "adam", B, E, le, rounds, fresh=True)
    got = trajectory(fx, False, "adam", B, E, le, rounds, fresh=True, mutant=mutant)
    moved = sum(int((rne_bf16(got["p"][k]) != rne_bf16(want["p"][k])).sum()) for k in want["p"])
    assert moved > 0, mutant
    print(f"[round spec] {mutant}: {moved} bf16 weights differ")
