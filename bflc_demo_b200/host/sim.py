"""In-process simulator: N clients + sponsor against one C++ ledger, round-robin polling with
no sleeps (the reference needs >= 2 sequential 10-30 s sleeps per round, M:231-233).
``python -m bflc_demo_b200.host.sim`` reproduces the reference demo end to end on the UCI
Occupancy CSV (20 clients, committee 4, top-6 of 10, lr 1e-3, softmax regression)."""
from __future__ import annotations

import argparse
import time
from typing import List, Optional

from .._native import ledger as _ledger
from ..config import FLConfig
from ..data.occupancy import split_data
from ..data.synthetic import Shard, femnist_like
from .client import Client, Sponsor
from .models import HostDPSGD, HostModel


def host_dpsgd(cfg: FLConfig, node: int) -> Optional[HostDPSGD]:
    """Client ``node``'s DP-SGD state: the engine's per-client key rule (engine/generic.py)."""
    if not cfg.dpsgd_on:
        return None
    from ..engine.generic import resolve_dpsgd_seed
    clip, noise = cfg.dpsgd_constants
    return HostDPSGD(float(clip), float(noise), resolve_dpsgd_seed(cfg, node))


def build(cfg: FLConfig, shards: List[Shard], test: Optional[Shard], *, model: HostModel,
          genesis=None, log=None, sponsor_log=None):
    L = _ledger()
    led = L.Ledger(cfg.to_ledger_config(model.size))
    if genesis is not None:
        # non-zero genesis model: registered through a zero-lr "round -1" is not possible, so the
        # simulator seeds clients' first global via an offset applied on both sides.
        raise NotImplementedError
    clients = [Client(i, led, shards[i], model, lr=cfg.learning_rate, batch_size=cfg.batch_size,
                      max_epoch=cfg.max_epoch, byzantine=i in cfg.byzantine_ranks,
                      byzantine_scale=cfg.byzantine_scale, prox_mu=cfg.prox_mu, log=log,
                      dpsgd=host_dpsgd(cfg, i)) for i in range(cfg.clients)]
    sponsor = Sponsor(led, test, model, log=sponsor_log) if test is not None else None
    return led, clients, sponsor


def run(cfg: FLConfig, shards, test, *, model: HostModel, rounds: int, log=print):
    led, clients, sponsor = build(cfg, shards, test, model=model, log=None, sponsor_log=log)
    t0 = time.time()
    while led.epoch() < rounds:
        progressed = False
        for c in clients:
            if c.poll() not in ("idle", "done"):
                progressed = True
        if sponsor:
            sponsor.poll()
        for line in led.drain_log():
            if log and "global loss" in line:
                log(line)
        if not progressed and led.epoch() >= 0:
            # nobody could act: a stalled round (e.g. dead committee member, SURVEY.md 5.3)
            raise RuntimeError(f"round {led.epoch()} stalled: update_count={led.update_count()} "
                               f"score_count={led.score_count()}")
    dt = time.time() - t0
    return led, clients, sponsor, dt


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--dataset", default="occupancy", choices=["occupancy", "femnist"])
    ap.add_argument("--clients", type=int, default=20)
    from ..run import (add_aggregation_args, add_dp_args, add_dpsgd_args, add_local_args, add_server_opt_args,
                       dp_fields, local_fields, server_opt_fields)
    add_aggregation_args(ap)
    add_server_opt_args(ap)
    add_dp_args(ap)
    add_dpsgd_args(ap)
    add_local_args(ap)
    a = ap.parse_args(argv)
    dp = dp_fields(ap, a)
    if a.dpsgd_clip == 0 and (a.dpsgd_noise or a.dpsgd_seed is not None):
        ap.error("--dpsgd-noise / --dpsgd-seed need --dpsgd-clip")
    dp.update(dpsgd_clip=a.dpsgd_clip, dpsgd_noise=a.dpsgd_noise, dpsgd_seed=a.dpsgd_seed)
    local = local_fields(ap, a)
    if dp["dp_noise"] > 0 and dp["dp_seed"] is None:     # the host ledger draws the noise: a secret seed
        import secrets
        dp["dp_seed"] = secrets.randbits(64)
    agg = dict(aggregation=a.aggregation, trim=a.trim, **server_opt_fields(ap, a), **dp, **local)
    if a.dataset == "occupancy":
        if a.non_iid_alpha is not None:
            ap.error("--non-iid-alpha applies to --dataset femnist (occupancy keeps the reference's split)")
        cfg = FLConfig.reference_scaled(a.clients, **agg)
        shards, test, src = split_data(clients_num=cfg.clients)
        model = HostModel("softmax", 5, 2)
        print(f"data: {src}; {cfg.clients} clients, committee {cfg.committee_size}, "
              f"top-{cfg.aggregate_count} of {cfg.needed_updates}")
    else:
        cfg = FLConfig.for_world(a.clients, learning_rate=0.05, batch_size=50, **agg)
        shards = femnist_like(cfg.clients, 300, seed=1, alpha=cfg.non_iid_alpha)
        test = femnist_like(1, 1000, seed=1, only=0)[0]
        model = HostModel("mlp", 784, 62, hidden=64, scale_inputs=1 / 255.0)
    led, clients, sponsor, dt = run(cfg, shards, test, model=model, rounds=a.rounds)
    if cfg.dpsgd_on:
        from ..engine.generic import dpsgd_epsilon
        eps = max(dpsgd_epsilon(cfg, c.dpsgd.step, max(len(c.shard) // cfg.batch_size, 1))[0] for c in clients)
        print(f"DP-SGD: largest local epsilon {eps:.6g} delta {cfg.dp_delta:g} over {cfg.clients} clients")
    print(f"{a.rounds} rounds in {dt:.2f} s ({a.rounds / dt:.1f} rounds/s); chain ok="
          f"{led.verify_chain()} blocks={led.n_blocks()} counters={led.counters()}")


if __name__ == "__main__":
    main()
