"""Committee validation on CTA pairs (mlp_val_sm100.cu, mlp_val_pair_kernel): each 64-row tile's
hidden layer split across a 2-CTA cluster, h handed to the leader through distributed shared memory.

* CPU: the validation kernel compiles without a stack frame, spills or serialized wgmma;
* GPU: exact-integer conformance against fp64 (n_val tails in 64- and 128-row terms, a partial
  last K-block, 62 / 10 classes, 1 / 3 / 8 candidate slots with some inactive, bf16 and fp8-blob
  biases, the predicate off), and what the fused engine validates, round after round, in both
  dtypes, against a relaunch and an fp64 forward with a derived rounding bound."""
import os
import re
import shutil
import struct
import subprocess

import pytest
import torch

from bflc_demo_b200 import build

SRC = build.CSRC / "kernels" / "mlp_val_sm100.cu"
H = 256
BF16 = torch.bfloat16
EPI_GENERIC, EPI_ARGMAX = 0, 2


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    out = tmp_path_factory.mktemp("ptxas") / "v.o"
    inc = [f"-I{build.CSRC / d}" for d in ("include", "ledger", "runtime")]
    cmd = [nvcc, *build.GENCODE, *build.NVCC_FLAGS, *inc, "-c", str(SRC), "-o", str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    log = proc.stdout + proc.stderr
    assert proc.returncode == 0, log[-3000:]
    return log


def test_validation_kernel_spill_free(ptxas_log):
    props = re.findall(r"Function properties for \w*?\d(mlp_val\w*?kernel)E\w*\s*\n\s*"
                       r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ptxas_log)
    found = {name: tuple(map(int, rest)) for name, *rest in props}
    assert set(found) == {"mlp_val_pair_kernel"}, ptxas_log[-3000:]
    for name, (frame, st, ld) in found.items():
        assert (frame, st, ld) == (0, 0, 0), f"{name}: {frame} B stack frame, {st} / {ld} B spills"
    serialized = [ln for ln in ptxas_log.splitlines() if re.search(r"\(C75(18|20)\)", ln)]
    assert not serialized, "\n".join(serialized)


# ----------------------------------------------------------------------------------------- GPU
def C():
    from bflc_demo_b200._native import C as _C
    return _C()


def gemm_dynamic(active, map_index, bias_ptrs):
    """A device-resident GemmDynamic (bflc_kernels.h, natural alignment) with null wait flags."""
    sz = C().struct_sizes()
    kmax = sz["kMaxRanks"]
    o_map, o_bias = 4, (4 + 4 * kmax + 7) // 8 * 8
    o_flag = o_bias + 8 * kmax
    o_val = o_flag + 8 * kmax
    size = (o_val + 4 + 7) // 8 * 8
    assert size == sz["GemmDynamic"]
    buf = bytearray(size)
    struct.pack_into("<i", buf, 0, active)
    struct.pack_into(f"<{kmax}i", buf, o_map, *(list(map_index) + [0] * (kmax - len(map_index))))
    struct.pack_into(f"<{kmax}Q", buf, o_bias, *(list(bias_ptrs) + [0] * (kmax - len(bias_ptrs))))
    return torch.frombuffer(buf, dtype=torch.uint8).cuda()


def w1_map(ptr, in_dim):
    """Layer-1 map: each CTA of a pair loads 128 of the 256 hidden rows of W1."""
    return C().gemm_b_map(ptr, H, in_dim, in_dim, False, False, EPI_GENERIC, 128)


def w2_map(ptr, nc):
    return C().gemm_b_map(ptr, nc, H, H, False, False, EPI_ARGMAX, 64)


class Problem:
    """Small-integer operands: x in {0, 1}, W1 / W2 in {-1, 0, 1}, integer b1, and b2 = integer +
    a distinct multiple of 1/128 per class.  Every fp32 partial sum is exact, h is an integer
    below 256 (exact in bf16), and no two logits of a row tie, so the fp64 argmax is the only
    right answer for any summation order."""

    def __init__(self, seed, n_val, in_dim, nc, n_slots, active, fp8):
        g = torch.Generator(device="cuda").manual_seed(seed)
        dev = "cuda"
        self.n_val, self.in_dim, self.nc, self.n_slots, self.active, self.fp8 = n_val, in_dim, nc, n_slots, active, fp8
        self.x = (torch.rand(n_val, in_dim, generator=g, device=dev) < 0.25).to(BF16)
        self.w1 = [torch.randint(-1, 2, (H, in_dim), generator=g, device=dev).to(BF16) for _ in range(n_slots)]
        self.w2 = [torch.randint(-1, 2, (nc, H), generator=g, device=dev).to(BF16) for _ in range(n_slots)]
        self.b1 = [torch.randint(-4, 5, (H,), generator=g, device=dev).float() for _ in range(n_slots)]
        frac = [torch.randperm(128, generator=g, device=dev)[:nc].float() / 128 for _ in range(n_slots)]
        self.b2 = [torch.randint(-4, 5, (nc,), generator=g, device=dev).float() + f for f in frac]
        # slot z validates the weights of map perm[z]
        self.perm = torch.randperm(n_slots, generator=torch.Generator().manual_seed(seed)).tolist()
        self.ref = []
        for z in range(n_slots):
            w = self.perm[z]
            h = torch.relu(self.x.double() @ self.w1[w].double().t() + self.b1[z].double())
            assert float(h.max()) < 256
            lg = h @ self.w2[w].double().t() + self.b2[z].double()
            top2 = lg.topk(min(2, nc), dim=1).values
            assert nc == 1 or bool((top2[:, 0] > top2[:, 1]).all())
            self.ref.append(lg.argmax(1))
        # half of the rows labelled with slot 0's prediction, so hits are not rare
        rnd = torch.randint(0, nc, (n_val,), generator=g, device=dev)
        keep = torch.rand(n_val, generator=g, device=dev) < 0.5
        self.labels = torch.where(keep, self.ref[0], rnd).to(torch.int32)
        kmax = C().struct_sizes()["kMaxRanks"]
        self.kmax = kmax
        if fp8:
            # fp32 biases from the candidates' blobs (dyn bias pointers stay null)
            L = C().mx8_mlp_layout(in_dim, H)
            self.blobs = []
            for z in range(n_slots):
                b = torch.zeros(L["total"] + 16, device=dev, dtype=torch.uint8)
                b[L["b1"]:L["b1"] + 4 * H].view(torch.float32).copy_(self.b1[z])
                b[L["b2"]:L["b2"] + 4 * nc].view(torch.float32).copy_(self.b2[z])
                self.blobs.append(b)
            self.blob_ptrs = torch.tensor([b.data_ptr() for b in self.blobs] + [0] * (kmax - n_slots),
                                          dtype=torch.int64, device=dev)
            self.dyn1 = gemm_dynamic(active, self.perm, [])
            self.dyn2 = gemm_dynamic(active, [kmax + p for p in self.perm], [])
        else:
            self.dyn1 = gemm_dynamic(active, self.perm, [t.data_ptr() for t in self.b1])
            self.dyn2 = gemm_dynamic(active, [kmax + p for p in self.perm], [t.data_ptr() for t in self.b2])

    def maps(self):
        blob = bytearray(2 * self.kmax * 128)
        for i in range(self.n_slots):
            blob[i * 128:(i + 1) * 128] = w1_map(self.w1[i].data_ptr(), self.in_dim)
            j = self.kmax + i
            blob[j * 128:(j + 1) * 128] = w2_map(self.w2[i].data_ptr(), self.nc)
        return torch.frombuffer(blob, dtype=torch.uint8).cuda()

    def run(self, correct):
        C().mlp_val(self.x, self.labels, correct, self.maps(), self.dyn1.data_ptr(), self.dyn2.data_ptr(),
                    self.n_val, self.in_dim, H, self.nc, self.n_slots,
                    self.blob_ptrs.data_ptr() if self.fp8 else 0)
        torch.cuda.synchronize()


CASES = [
    # n_val, in_dim, n_classes, slots, active, fp8-blob biases
    (4096, 784, 62, 1, 1, True),
    (4096, 784, 62, 3, 2, False),
    (4032, 784, 62, 8, 8, True),
    (4032, 64, 10, 3, 3, False),
    (200, 784, 10, 8, 5, False),
    (200, 64, 62, 1, 1, True),
    (64, 784, 62, 3, 1, True),
    (64, 64, 10, 8, 6, False),
    (1, 784, 10, 3, 3, False),
    (1, 64, 62, 8, 2, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("n_val,in_dim,nc,slots,active,fp8", CASES,
                         ids=[f"n{c[0]}-k{c[1]}-c{c[2]}-s{c[3]}a{c[4]}-{'fp8' if c[5] else 'bf16'}" for c in CASES])
def test_exact_counts(n_val, in_dim, nc, slots, active, fp8):
    p = Problem(1000 + n_val + in_dim + nc + slots, n_val, in_dim, nc, slots, active, fp8)
    correct = torch.full((p.kmax,), 1000, device="cuda", dtype=torch.int32)
    p.run(correct)
    for z in range(p.kmax):
        want = 1000
        if z < active:
            want += int((p.ref[z] == p.labels.long()).sum())
        assert int(correct[z]) == want, (z, int(correct[z]), want)


@pytest.mark.gpu
def test_predicate_off_leaves_counts():
    p = Problem(77, 4096, 784, 62, 3, 3, False)
    pred = torch.zeros(1, device="cuda", dtype=torch.int32)
    correct = torch.full((p.kmax,), 1000, device="cuda", dtype=torch.int32)
    C().set_predicate(pred.data_ptr())
    try:
        p.run(correct)
    finally:
        C().set_predicate(0)
    assert bool((correct == 1000).all())
    pred.fill_(1)
    C().set_predicate(pred.data_ptr())
    try:
        p.run(correct)
    finally:
        C().set_predicate(0)
    assert int(correct[0]) == 1000 + int((p.ref[0] == p.labels.long()).sum())


def _revalidate(eng):
    """The last round's committee validation again: an eager launch on the engine's own maps,
    plan and candidate blob table."""
    K = C().struct_sizes()["kMaxRanks"]
    correct = torch.zeros(K, device="cuda", dtype=torch.int32)
    x = eng.x_dq if eng.fp8 else eng.x_bf
    C().mlp_val(x[: eng.n_val], eng.y[: eng.n_val], correct, eng.b_maps, eng.dyn_ptr[0], eng.dyn_ptr[1],
                eng.n_val, eng.in_dim, H, eng.spec.by_name["w2"].shape[0], eng.world,
                eng.plan_ptr + eng.sz["plan_cand_blob_off"] if eng.fp8 else 0)
    torch.cuda.synchronize()
    return correct


def _engine(dtype):
    from bflc_demo_b200.config import FLConfig
    from bflc_demo_b200.data.synthetic import femnist_like
    from bflc_demo_b200.engine.fused import FusedEngine
    cfg = FLConfig.for_world(1, model="mlp", hidden=H, batch_size=512, samples_per_client=4096,
                             learning_rate=1e-3, dtype=dtype, optimizer="adam", cuda_graph=True)
    eng = FusedEngine(cfg, femnist_like(1, 4096, seed=7, only=0)[0])
    # The shard's class-prototype pixels make the model confident, so almost every row's top-2
    # margin clears the rounding bound of _fp64_hit_range (noise pixels leave several percent of
    # the rows inside it).  A fixed tenth of the labels is random, so hits stay below n_val.
    g = torch.Generator().manual_seed(11)
    flip = torch.rand(eng.y.shape, generator=g) < 0.1
    rnd = torch.randint(0, eng.spec.by_name["w2"].shape[0], eng.y.shape, generator=g, dtype=torch.int32)
    eng.y.copy_(torch.where(flip, rnd, eng.y.cpu()))
    return eng


def _fp64_hit_range(eng, par):
    """[lo, lo + A]: the hits the validation kernel can report for the candidate of parity `par`.

    The weights are the bf16 W1 / W2 its maps cover (upload_shadow), the biases the fp32 ones it
    reads (bf16: upload_master; fp8: the candidate's blob), x is x_bf / x_dq.  All products of
    bf16 values are exact in fp32, so the kernel differs from exact arithmetic only by its fp32
    sums and the bf16 rounding of h.  With u = 2^-23 (one fp32 ulp per addition, which holds for
    truncating as well as round-to-nearest accumulation, in any order) and gamma_n = n u / (1 - n u):

    * fwd1: the kernel's relu(acc + b1) lies within e1 = gamma_{K+1} (sum_k |x_k W1_jk| + |b1_j|)
      of relu(z_j), z = x W1^T + b1 in fp64 (relu is 1-Lipschitz).
    * h: the kernel and the reference h_j = bf16(relu(z_j)) each round to nearest, by at most half
      a bf16 ulp, and a ulp is at most 2^-7 |v| (8 significant bits).  So the kernel's h_j lies
      within d_j = (1 + 2^-8) e1_j + 2^-7 |h_j| / (1 - 2^-8) + 2^-126 of h_j (the last term: a
      flushed subnormal), i.e. one bf16 ulp of h_j plus e1.
    * fwd2: logit c then lies within B_c = sum_j |W2_cj| d_j
      + gamma_{H+1} (sum_j (|h_j| + d_j) |W2_cj| + |b2_c|) of the fp64 logit from h_j.

    In a row whose fp64 top-2 margin exceeds 2 max_c B_c no other logit of the kernel can reach the
    top one, so the kernel's argmax is the fp64 one.  lo counts the hits among those rows; the
    other A rows may go either way."""
    o = eng.layout.offsets
    P, Hh = eng.n_params, eng.cfg.hidden
    w = eng.spec.views(eng.heap.view(o[f"upload_shadow{par}"], [P], torch.bfloat16))
    w1, w2 = w["w1"].double(), w["w2"].double()
    if eng.fp8:
        blob = eng.heap.view(eng.upq_off[par], [eng.blob_bytes], torch.uint8)
        nc = w2.shape[0]
        b1 = blob[eng.ql["b1"]:eng.ql["b1"] + 4 * Hh].view(torch.float32).double()
        b2 = blob[eng.ql["b2"]:eng.ql["b2"] + 4 * nc].view(torch.float32).double()
    else:
        m = eng.spec.views(eng.heap.view(o[f"upload_master{par}"], [P], torch.float32))
        b1, b2 = m["b1"].double(), m["b2"].double()
    x = (eng.x_dq if eng.fp8 else eng.x_bf)[: eng.n_val].double()
    y = eng.y[: eng.n_val].long()
    u = 2.0 ** -23

    def gamma(n):
        return n * u / (1 - n * u)

    K = x.shape[1]
    z = x @ w1.t() + b1
    e1 = gamma(K + 1) * (x.abs() @ w1.abs().t() + b1.abs())
    h = torch.relu(z).float().to(torch.bfloat16).double()
    d = (1 + 2.0 ** -8) * e1 + 2.0 ** -7 * h / (1 - 2.0 ** -8) + 2.0 ** -126
    logits = h @ w2.t() + b2
    bound = (d @ w2.abs().t() + gamma(Hh + 1) * ((h + d) @ w2.abs().t() + b2.abs())).amax(1)
    top2 = logits.topk(2, dim=1).values
    sure = top2[:, 0] - top2[:, 1] > 2 * bound
    lo = int(((logits.argmax(1) == y) & sure).sum())
    return lo, int((~sure).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp8", "bf16"])
def test_engine_validation_matches_fp64(dtype):
    """Round after round through FusedEngine: the engine's own val_correct equals an eager relaunch
    of the validation kernel on the same plan and candidate weights, the median score is
    val_correct / n_val, and val_correct lies in the range an fp64 forward pass with a derived
    rounding bound allows (_fp64_hit_range)."""
    eng = _engine(dtype)
    assert eng.val_chain and eng.val_bn == [128, 64]
    eng.capture()
    for _ in range(4):
        eng.run_round()
        torch.cuda.synchronize()
        st = eng.read_state()
        got = eng.val_correct.clone()
        assert int(got[0]) > 0
        assert torch.equal(_revalidate(eng), got)
        assert abs(st["median"][0] - int(got[0]) / eng.n_val) < 1e-6
        lo, undecided = _fp64_hit_range(eng, (st["epoch"] - 1) & 1)
        print(f"{dtype} epoch {st['epoch']}: {int(got[0])} hits, fp64 range [{lo}, {lo + undecided}], "
              f"{undecided} undecided rows")
        assert lo <= int(got[0]) <= lo + undecided
        assert undecided <= 0.01 * eng.n_val
    assert not eng.drain_blocks()
