"""Checkpoint / resume.  In the reference "the ledger is the checkpoint": global model + epoch +
roles persist with the chain, clients are stateless and re-register (SURVEY.md 5.4).  Here a
checkpoint is the host ledger snapshot (blocks + live state, hash-verified on load), the global
model, the device ledger page, the per-client optimizer state, and this rank's server optimizer
state (its slice of it in two-shot mode: the rest is never read on this rank).

Works for either engine on the device protocol (``engine/base.py``: ``ProtocolEngine``)."""
from __future__ import annotations

import json
import struct

import numpy as np
import torch
import torch.distributed as dist

from .._native import ledger as _ledger
from ..models.lora import model_shape


def save_checkpoint(path: str, eng) -> dict:
    """Collective (every rank calls it; each rank writes ``path`` with its rank suffix when
    world > 1).  Drains the device block ring first so the host chain is complete."""
    errs = eng.drain_blocks()
    if errs:
        raise RuntimeError(f"cannot checkpoint: host/device ledgers disagree: {errs[:2]}")
    torch.cuda.synchronize()
    st = eng.read_state()
    # Only tensors / str / int: the file loads with torch.load(weights_only=True) (no pickled
    # objects).  Byte strings are stored as uint8 tensors.
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).clone()   # noqa: E731
    opt_total, round_seq = plan_counters(eng)
    blob = dict(
        version=2, world=eng.world, rank=eng.rank, config=eng.cfg.to_json(), n_params=eng.n_params,
        epoch=st["epoch"], state_bytes=eng.state_bytes.cpu().clone(),
        global_master=eng.global_master.detach().cpu().clone(),
        ledger=u8(eng.host_ledger.snapshot()),
        # Adam: moments AND the step count t the bias correction is computed from (the plan
        # page's running total of optimizer steps on this rank)
        opt_total=opt_total, round_seq=round_seq,
    )
    for k, t in zip(("opt_m", "opt_v"), eng.opt_moments):
        if t is not None:
            blob[k] = t.detach().cpu().clone()
    for k, t in zip(("server_m", "server_v"), eng.server_state):
        blob[k] = t.detach().cpu().clone()
    # the DP noise seed: the ledger snapshot never holds it, and a resumed run needs it to draw the
    # same noise (stored as a string: it may not fit an int64)
    blob["dp_seed"] = str(int(eng.dp_seed))
    # DP-SGD: this rank's own noise key (each rank's file holds only its own), for the same reason
    if getattr(eng, "dpsgd", None) is not None:
        blob["dpsgd_seed"] = str(int(eng.dpsgd_seed))
    # LoRA: the adapters only mean something on top of the base they were trained on
    if getattr(eng, "base_digest", None):
        blob["base_digest"] = eng.base_digest
    # BERT / GPT shape fields (JSON), so a LoRA run can check a base checkpoint against its model
    net = getattr(eng, "net", None)
    shape = model_shape(getattr(net, "base", net)) if net is not None else None
    if shape is not None:
        blob["model_shape"] = json.dumps(shape, sort_keys=True)
    out = path if eng.world == 1 else f"{path}.rank{eng.rank}"
    torch.save(blob, out)
    return dict(path=out, epoch=st["epoch"], blocks=eng.host_ledger.n_blocks())


def plan_counters(eng):
    """(opt_total, round_seq) of the engine's plan page: this rank's optimizer steps so far and the
    input-pipeline generation."""
    raw = bytes(eng.plan_bytes.cpu().numpy())
    opt_total, = struct.unpack_from("<i", raw, eng.sz["plan_opt_total_off"])
    round_seq, = struct.unpack_from("<I", raw, eng.sz["plan_round_seq_off"])
    return int(opt_total), int(round_seq)


def _set_plan_counters(eng, opt_total: int, round_seq: int):
    raw = bytearray(bytes(eng.plan_bytes.cpu().numpy()))
    struct.pack_into("<i", raw, eng.sz["plan_opt_total_off"], int(opt_total))
    struct.pack_into("<i", raw, eng.sz["plan_opt_step_off"], int(opt_total))
    struct.pack_into("<I", raw, eng.sz["plan_round_seq_off"], int(round_seq))
    eng.plan_bytes.copy_(torch.frombuffer(raw, dtype=torch.uint8))


def _restore_dpsgd(blob: dict, eng):
    """DP-SGD settings must match (the accounting spans the whole run), and the client's noise key is
    adopted as DP-FedAvg's seed is: only by an engine that drew its own (dpsgd_seed None) and has not
    yet captured its training graph, which holds the key."""
    saved = json.loads(blob["config"]) if isinstance(blob.get("config"), str) else {}
    mine = (float(eng.cfg.dpsgd_constants[0]), float(eng.cfg.dpsgd_constants[1]))
    theirs = tuple(float(np.float32(saved.get(k, 0.0))) for k in ("dpsgd_clip", "dpsgd_noise"))
    if theirs != mine:
        raise ValueError(f"checkpoint was written under other DP-SGD settings than this engine's: "
                         f"(clip, noise) {theirs} there, {mine} here")
    dps = getattr(eng, "dpsgd", None)
    if dps is None or "dpsgd_seed" not in blob:
        return
    seed = int(blob["dpsgd_seed"])
    if seed != eng.dpsgd_seed:
        if eng.cfg.dpsgd_seed is not None or eng.graph_train is not None:
            raise ValueError("checkpoint was written with another DP-SGD noise key than this engine's "
                             "(construct the engine with dpsgd_seed=None and load before capture() to adopt it)")
        eng.dpsgd_seed = dps.seed = seed


def load_checkpoint(path: str, eng) -> dict:
    """Restore into a freshly constructed engine of the same config/world.  Collective."""
    src = path if eng.world == 1 else f"{path}.rank{eng.rank}"
    blob = torch.load(src, map_location="cpu", weights_only=True)
    if blob["n_params"] != eng.n_params or blob["world"] != eng.world:
        raise ValueError("checkpoint does not match this engine (n_params / world)")
    if "base_digest" in blob and blob["base_digest"] != getattr(eng, "base_digest", None):
        raise ValueError("checkpoint was trained on another LoRA base model (base sha256 differs)")
    L = _ledger()
    seed = int(blob.get("dp_seed", "0"))
    led = L.Ledger.restore(bytes(blob["ledger"].numpy()), dp_seed=seed)  # verifies the hash chain
    lc = led.config()
    # differential privacy: the same mode, clip and noise multiplier, and the same seed, so the resumed
    # run draws exactly the noise the uninterrupted one would have
    clip, noise = eng.cfg.dp_constants
    if (lc.dp_mode(), lc.dp_clip, lc.dp_noise) != (eng.cfg.dp_mode, float(clip), float(noise)):
        raise ValueError(f"checkpoint was written under other differential privacy settings than this engine's: "
                         f"ledger has (mode, clip, noise) = {(lc.dp_mode(), lc.dp_clip, lc.dp_noise)}, engine "
                         f"{(eng.cfg.dp_mode, float(clip), float(noise))}")
    if eng.cfg.dp_mode == 2 and seed != eng.dp_seed:
        if eng.cfg.dp_seed is not None or eng.consensus_captured:
            raise ValueError("checkpoint was written with another differential privacy seed than this engine's "
                             "(construct the engine with dp_seed=None and load before capture() to adopt it)")
        eng.dp_seed = seed
        eng.dp_kw = eng.layout.dp_kwargs(eng.cfg.dp_mode, clip, noise, seed)
    _restore_dpsgd(blob, eng)
    if L.agg_word(lc.aggregation, lc.trim) != L.agg_word(eng.cfg.aggregation_rule, eng.cfg.trim):
        raise ValueError("checkpoint was written under another aggregation rule than this engine's "
                         f"({eng.cfg.aggregation}, trim {eng.cfg.trim})")
    want = eng.cfg.to_ledger_config(eng.n_params)
    # the hyperparameters the optimizer uses (momentum: lr, beta1; adam / yogi: all four)
    hp = lambda c: ((c.server_opt,) + (c.server_lr, c.server_beta1, c.server_beta2, c.server_tau)[  # noqa: E731
        : (0, 2, 4, 4)[c.server_opt]])
    if hp(lc) != hp(want):
        raise ValueError(f"checkpoint was written under another server optimizer than this engine's "
                         f"({eng.cfg.server_opt}): ledger has {hp(lc)}, engine {hp(want)}")
    state = eng.server_state
    if any(blob.get(k) is None for k in ("server_m", "server_v")[: len(state)]):
        raise ValueError("checkpoint holds no server optimizer state")
    eng.host_ledger = led
    epoch = blob["epoch"]
    g = blob["global_master"].to(eng.dev)
    for t in (eng.global_master, eng.work_master):
        t.copy_(g)
    for t in (eng.global_shadow, eng.work_shadow):
        t.copy_(g.to(torch.bfloat16))
    eng.state_bytes.copy_(blob["state_bytes"])
    # epoch-tagged flags: everything up to `epoch` has happened on every rank
    n_flags = eng.sz["FLAG_COUNT"]
    flags = eng.heap.view(eng.layout.offsets["flags"], [n_flags], torch.int32)
    flags.fill_(epoch)
    for k, t in zip(("opt_m", "opt_v"), eng.opt_moments):
        if blob.get(k) is not None and t is not None:
            t.copy_(blob[k].to(eng.dev))
    for k, t in zip(("server_m", "server_v"), state):
        t.copy_(blob[k].to(eng.dev))
    # Adam's t continues where the saved run stopped, whatever warm-up rounds this engine ran
    # before the restore (FusedEngine.capture() runs one); the input-pipeline generation keeps
    # growing (tags only ever increase), so round_seq is restored only if it moves forward
    _, cur_seq = plan_counters(eng)
    _set_plan_counters(eng, blob.get("opt_total", 0), max(cur_seq, int(blob.get("round_seq", 0))))
    eng.drained = epoch
    eng._rounds = epoch
    # host-side caches of the ledger page are stale now
    eng.reset_host_caches()
    torch.cuda.synchronize()
    if eng.world > 1:
        dist.barrier(group=eng.group)
    return dict(epoch=epoch, blocks=eng.host_ledger.n_blocks())
