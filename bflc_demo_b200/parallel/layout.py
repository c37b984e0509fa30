"""Byte layout of the symmetric heap (identical on every rank) -- Python mirror of
``bflc::HeapLayout`` (csrc/include/bflc_kernels.h).  The regions replace the seven JSON
strings the reference keeps in one KV table (CommitteePrecompiled.cpp:32-44): flags and
RoundState are the "epoch/roles/counters" keys, the score matrix and upload buffers are
``local_scores`` / ``local_updates``, ``global`` is ``global_model``."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List

from .._native import C


def _up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


@dataclass
class HeapLayout:
    n_params: int                     # padded to a multiple of 8 elements
    ring_slots: int = 256
    extra_bytes: int = 0              # caller-owned scratch appended after the fixed regions
    server_state: int = 0             # fp32 [n_params] vectors of server optimizer state: 0, 1 (m) or 2 (m, v)
    dp: bool = False                  # the DpPage of differentially private aggregation
    dp_adaptive: bool = False         # ... followed by the adaptive clip's DpAdapt header and clip-record ring
    offsets: Dict[str, int] = field(default_factory=dict)
    total_bytes: int = 0
    sizes: Dict[str, int] = field(default_factory=dict)

    def __post_init__(self):
        sz = C().struct_sizes()
        self.sizes = dict(sz)
        assert self.n_params % 8 == 0
        K = sz["kMaxRanks"]
        cur = 0

        def take(name: str, nbytes: int, align: int = 1024):
            nonlocal cur
            cur = _up(cur, align)
            self.offsets[name] = cur
            cur += nbytes

        take("flags", sz["FLAG_COUNT"] * 4)
        take("state", sz["RoundState"])
        take("plan", sz["RoundPlan"])
        take("scores", 2 * K * K * 4 + 2 * K * 8)   # score rows by parity + two-shot slice digests
        take("meta", 2 * K * sz["UploadMeta"])
        take("admit", 2 * sz["AdmitPage"])              # first-K-wins admission: ticket + slots, by parity
        take("ring", self.ring_slots * sz["BlockRecord"])
        f32, b16 = self.n_params * 4, self.n_params * 2
        take("work_master", f32, 4096)
        take("work_shadow", b16, 4096)
        take("upload_master0", f32, 4096)
        take("upload_master1", f32, 4096)
        take("upload_shadow0", b16, 4096)
        take("upload_shadow1", b16, 4096)
        take("global", f32, 4096)
        take("global_shadow", b16, 4096)
        take("extra", self.extra_bytes, 4096)
        # this rank's own server optimizer state (never read by a peer); after every other region so
        # a layout without it is byte for byte the one before
        assert self.server_state in (0, 1, 2)
        for name in ("server_m", "server_v")[: self.server_state]:
            take(name, f32, 4096)
        # DP norm partials (written by every peer) and the last round's norms; last, for the same reason
        if self.dp:
            take("dp", self.dp_region_bytes(), 4096)
        self.total_bytes = _up(cur, 1 << 21)

    def fed_dict(self, rank: int, n_ranks: int, peer_bases: List[int], mc_base: int) -> dict:
        o = self.offsets
        return dict(rank=rank, n_ranks=n_ranks, peer_bases=list(peer_bases), mc_base=mc_base,
                    flags_off=o["flags"], state_off=o["state"], plan_off=o["plan"],
                    scores_off=o["scores"], meta_off=o["meta"],
                    work_master_off=o["work_master"], work_shadow_off=o["work_shadow"],
                    upload_master_off=[o["upload_master0"], o["upload_master1"]],
                    upload_shadow_off=[o["upload_shadow0"], o["upload_shadow1"]],
                    global_off=o["global"], global_shadow_off=o["global_shadow"],
                    ring_off=o["ring"], n_params=self.n_params, ring_slots=self.ring_slots,
                    admit_off=o["admit"])

    def server_opt_kwargs(self, opt_id: int, constants) -> dict:
        """Keyword arguments of ``fed_consensus_aggregate`` for server optimizer ``opt_id`` (0: none,
        no arguments) with its six fp32 constants (``FLConfig.server_opt_constants``)."""
        if opt_id == 0:
            return {}
        o = self.offsets
        return dict(server_opt=opt_id, server_hp=[float(x) for x in constants], server_m_off=o["server_m"],
                    server_v_off=o.get("server_v", 0))

    def dp_kwargs(self, mode: int, clip: float, noise: float, seed: int, adaptive: bool = False) -> dict:
        """Keyword arguments of ``fed_consensus_aggregate`` for DP mode ``mode`` (0: off, no arguments); with
        ``adaptive`` the kernel modes 3 / 4, which read the clip from the DpAdapt header and write clip records
        after it, with the size of this layout's dp region (the binding refuses one without those regions)."""
        if mode == 0:
            return {}
        kw = dict(dp_mode=mode + 2 * bool(adaptive), dp_clip=float(clip), dp_noise=float(noise), dp_seed=int(seed),
                  dp_off=self.offsets["dp"])
        if adaptive:
            kw["dp_bytes"] = self.dp_region_bytes()
        return kw

    def dp_region_bytes(self) -> int:
        """Size of the dp region: the DpPage, and with adaptive clipping the DpAdapt header and clip ring."""
        sz = self.sizes
        return sz["DpPage"] + (sz["DpAdapt"] + self.ring_slots * sz["DpClipRecord"] if self.dp_adaptive else 0)

    def dp_adapt_offsets(self) -> tuple:
        """Heap byte offsets of the DpAdapt header and of the clip-record ring (adaptive clipping)."""
        head = self.offsets["dp"] + self.sizes["DpPage"]
        return head, head + self.sizes["DpAdapt"]
