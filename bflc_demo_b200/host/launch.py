"""Process launcher (reference L4, python-sdk/main.py:343-358): one ledger-server process,
``CLIENT_NUM`` client processes and one sponsor process, all on localhost.

    python -m bflc_demo_b200.host.launch --clients 20 --rounds 10

The reference staggers process starts by 3 s and clients sleep U(10, 30) s between polls
(M:62, 231-233, 350); here the poll interval is a flag (default 5 ms)."""
from __future__ import annotations

import argparse
import multiprocessing as mp
import os
import random
import tempfile
import time

from ..config import FLConfig
from ..data.occupancy import split_data
from .client import Client, Sponsor
from .models import HostModel
from . import identity
from .rpc import LedgerServer, RemoteLedger


def _server(cfg_json, model_size, q, key_dir, authkey):
    cfg = FLConfig.from_json(cfg_json)
    # signed mode: only holders of an enrolled node_<i>.pem can act, and only as client i
    srv = LedgerServer(cfg, model_size, accounts=identity.load_public_keys(key_dir, cfg.clients),
                       authkey=authkey)
    q.put(srv.address)
    srv.serve_forever()


def run_one_node(node_id, address, cfg_json, rounds, interval, key_dir, authkey):
    cfg = FLConfig.from_json(cfg_json)
    shards, _, _ = split_data(clients_num=cfg.clients)
    # set_from_account_signer(node_id), README.md:348-359
    led = RemoteLedger(address, authkey=authkey, client_id=node_id,
                       key=identity.load_account(key_dir, node_id))
    me = Client(node_id, led, shards[node_id], HostModel("softmax", 5, 2), lr=cfg.learning_rate,
                batch_size=cfg.batch_size, max_epoch=rounds - 1, prox_mu=cfg.prox_mu)
    print(f"node_{node_id} initializing....", flush=True)
    try:
        while me.poll() != "done":
            time.sleep(random.uniform(interval, 3 * interval))  # wait(), M:231-233
    except (ConnectionError, EOFError, OSError):
        pass  # the sponsor closed the ledger service: the run is over
    led.finish()


def run_sponsor(address, cfg_json, rounds, interval, authkey):
    cfg = FLConfig.from_json(cfg_json)
    _, test, _ = split_data(clients_num=cfg.clients)
    led = RemoteLedger(address, authkey=authkey)      # default account: read-only observer (M:317)
    sp = Sponsor(led, test, HostModel("softmax", 5, 2), log=lambda s: print(s, flush=True))
    while sp.test_epoch < rounds:
        sp.poll()
        time.sleep(interval)
    print("chain ok:", led.verify_chain(), "blocks:", led.n_blocks(), flush=True)
    led.shutdown()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--interval", type=float, default=0.005)
    ap.add_argument("--prox-mu", type=float, default=0.0,
                    help="FedProx: proximal term toward the round's global model (default 0: off)")
    a = ap.parse_args(argv)
    try:
        cfg = FLConfig.reference_scaled(a.clients, prox_mu=a.prox_mu)
    except ValueError as e:
        ap.error(str(e))
    cj = cfg.to_json()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    # per-run secrets: one ECDSA key per client (bin/get_batch_accounts.sh) + the socket authkey
    key_dir = tempfile.mkdtemp(prefix="bflc_accounts_")
    identity.generate_accounts(cfg.clients, key_dir)
    authkey = os.urandom(32)
    srv = ctx.Process(target=_server, args=(cj, HostModel("softmax", 5, 2).size, q, key_dir, authkey),
                      daemon=True)
    srv.start()
    address = q.get(timeout=60)
    procs = [ctx.Process(target=run_one_node,
                         args=(i, address, cj, a.rounds, a.interval, key_dir, authkey))
             for i in range(cfg.clients)]
    for p in procs:
        p.start()
    sp = ctx.Process(target=run_sponsor, args=(address, cj, a.rounds, a.interval, authkey))
    sp.start()
    sp.join()
    for p in procs:
        p.join(timeout=30)
        if p.is_alive():
            p.terminate()
    srv.join(timeout=5)
    if srv.is_alive():
        srv.terminate()


if __name__ == "__main__":
    main()
