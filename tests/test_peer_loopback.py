"""The peer-exchange path (ddp.py, csrc/comm.cu, the world > 1 norm finalize) on ONE device.

Every test of world > 1 that needs two GPUs skips on a one-GPU machine; these need one (or none):

Part A -- the flag kernels against exact results.  Each "peer" is a local b2_comm_alloc buffer.  The other ranks'
flags (and, where the kernel reads them, their values) are posted before the launch, and loopback.flag_launch checks on
the host that every flag the kernel polls already satisfies its epoch: a kernel never waits, and the device is idle
before and after each launch, so no two flag kernels are ever in flight together.

Part B/C -- a loopback peer group: N replicas of one model on one device, each in the real DistributedDataParallel,
over a thread-backed process group.  The flag entry points are replaced by host lockstep (loopback.Group), so no flag
kernel runs there; the reduce-and-update kernels, the copy-engine DMA form, the one-sided pulls and close() are the
library's own.  The eager step is driven with forward + backward rank by rank on the main thread and optimizer.step()
in N threads (its lazy state allocations are collective).

Part D -- planted defects in the harness, each failing its named check.

Arguments -- the flag entry points' rejections, in a child process that sees no device.

What the checks found and how close they came (H100 80 GB HBM3, 700 W power limit; `pytest -m gpu` on this file: 63
tests in 90 s):
  * b2_grad_norm_finalize at world > 1 launched its share kernel before checking the exchange's slot and peer
    pointers: a rejected call had already overwritten *total_norm, and without a device the rejection was never
    reached.  Fixed (checked first); test_argument_is_rejected[finalize-slot-64], [finalize-null-peer] and
    [finalize-null-flags] fail without the fix.
  * The range limit: at world > 1 the share of the sum of squares is exchanged as fp32, so a sum above FLT_MAX gives
    an infinite norm where world 1 (fp64 until the square root) stays finite.  It needs a gradient norm above 1.8e19,
    a run that has already diverged; pinned, not changed (test_finalize_range_limit).
  * The GradScaler consensus probe (a scalar mean at _SLOT_INF) runs in every backward under a peer group, not only
    under a GradScaler.  The loopback's backward runs rank by rank on one thread, so it answers that call from the
    rank's own value and requires it to be 0 (a finite probe); the exchange itself stays with the 2-GPU worker.  The
    loopback therefore runs no GradScaler, and its host restatement of the world > 1 finalize refuses one.
  * Part A, exact: barrier flags and counters (world 1 / 2 / 3 / 8, first / middle / last rank, slots 0 and 63, the
    epoch wrap 0xFFFFFFFF -> 0), the allgather words (4 B, 4 * 1001 B, 1 MiB) and the rank-order mean are bitwise their
    restatements, and no other word moved.  The world > 1 finalize's norm is bitwise its restatement; against float64
    the worst |norm - sqrt(S)| / bound was 0.370 (world 2), 0.162 (world 3), 0.114 (world 8).
  * Same batch on every rank, N in {2, 4, 8}: master, shadow, every optimizer state buffer, the step counter and
    optimizer.state_dict() bitwise the world-1 run's for HF AdamW, TorchAdamW, Adam(amsgrad) and SGD(momentum,
    nesterov, decay), kernel form, and DMA form for HF AdamW at every N and every optimizer at N = 4; also at H 768
    with 2 layers (N = 4).  Both sides run the reduce form (b2_bucket_reduce_*, recorded): the slim form is world 1
    under an armed backward only.
  * Same batch, N = 3 (the inexact mean): HF AdamW within AdamWRef's bound, worst ratio 0.872; TorchAdamW, Adam
    (amsgrad) and SGD bitwise torch's fused AdamW / Adam and torch.optim.SGD fed the exact fp32 mean.
  * no_sync() window at N = 3: the fold bitwise its fp32 restatement, worst 0.996 of its float64 bound (the bound is
    one bf16 rounding, which it nearly reaches); the update worst 0.968 of AdamWRef's bound.
  * clip_grad_norm_ at N = 3: the stash bitwise the rank-order mean; partial sums of squares worst 0.020 of their
    bound, the norm worst 0.046 of its bound, the coefficient bitwise torch's and read by every bucket's update; the
    update worst 0.959 of AdamWRef's bound.
  * Different batches, N = 2 and 3: the worst per-rank loss error against oracle.ddp_ref.train was 0.025 and 0.075 of
    TOL_TRAJ, loss_reduce is bitwise the rank-order fp32 mean, and the DMA form is bitwise the kernel form from
    bitwise-equal gradients.
"""
import json
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import loopback as lb
from loopback import L, interlock, flag_launch, ready
from parity import TOL_TRAJ, b2, bert_ref, make_model, state_from_hf_init, tiny_config, to_dev
from oracle import ddp_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DDP = b2.DistributedDataParallel
U32 = 0xFFFFFFFF
SENT = 0x5A5A5A5A
U = 2.0 ** -24


def i32(v):
    v &= U32
    return v - (1 << 32) if v >= (1 << 31) else v


# ======================================================================================================================
# CPU: the slice rule, the interlock
# ======================================================================================================================
def test_bucket_slice_tiles_every_bucket():
    """rank r's slice of [b, e): 8-aligned, the slices of 0..world-1 tile the bucket in rank order, and ranks past the
    end get an empty slice (those launch nothing, see _exchange_update) -- including buckets shorter than 8 * world"""
    g = torch.Generator().manual_seed(5)
    cases = [(0, 8, 8), (0, 16, 8), (8, 24, 3), (64, 64 + 8 * 5, 8), (0, 8 * 1001, 3)]
    for _ in range(400):
        b = 8 * int(torch.randint(0, 1 << 16, (1,), generator=g))
        n = 8 * int(torch.randint(0, 80 if _ % 2 else 1 << 14, (1,), generator=g))
        cases.append((b, b + n, int(torch.randint(1, 9, (1,), generator=g))))
    short = 0
    for b, e, world in cases:
        at = b
        for r in range(world):
            sb, se = DDP._bucket_slice(b, e, r, world)
            assert sb % 8 == 0 and se % 8 == 0 and b <= sb <= se <= e, (b, e, world, r, sb, se)
            assert sb == at, ("gap or overlap", b, e, world, r)
            at = se
            if se == sb:
                short += 1
        assert at == e, (b, e, world)
    assert short > 0       # some cases give the last ranks nothing


def test_interlock_rule():
    assert interlock(4, {"a": 5, "b": 9}) == 5
    assert interlock(0xFFFFFFFE, {"a": 0xFFFFFFFF}) == 0xFFFFFFFF
    assert interlock(0xFFFFFFFF, {"a": 0}) == 0          # the wrap: epoch 0 after 0xFFFFFFFF
    assert ready(0, 0xFFFFFFFF) and ready(5, 0xFFFFFFF0)
    # at the wrap a flag of 0xFFFFFFFF is one epoch short of epoch 0
    assert not ready(0xFFFFFFFF, 0)
    with pytest.raises(AssertionError, match="interlock: q1"):
        interlock(0xFFFFFFFF, {"q0": 0, "q1": 0xFFFFFFFF})


def test_planted_interlock_one_epoch_short():
    """planted defect: a flag one epoch short of what the launch will use -- the helper refuses before launching"""
    with pytest.raises(AssertionError, match="does not satisfy epoch 0x00000008: the kernel would wait; not launched"):
        interlock(7, {"flags[3]": 8, "flags[4]": 7})


# ======================================================================================================================
# CPU: argument rejections, in a child process that sees no device
# ======================================================================================================================
_CHILD = r"""
import ctypes, importlib.util, json, sys
spec = importlib.util.spec_from_file_location("b2_lib_child", sys.argv[1])
L = importlib.util.module_from_spec(spec)
spec.loader.exec_module(L)
base = 1 << 24
lib = L.load()
out = {}
def arr(world, null=None, off=0):
    return L.ptr_array([None if q == null else base + off + 0x10000 * q for q in range(max(world, 1))])
for name, entry, world, rank, slot, nbytes, null in json.loads(sys.argv[2]):
    ep = base + 0x900000
    if entry == "barrier":
        st = lib.b2_peer_barrier(arr(world, null), world, rank, slot, ep, None)
    elif entry == "allgather":
        st = lib.b2_allgather_rows(base + 0xa00000, nbytes, arr(world, null if null != "flags" else None, 0x100000),
                                   arr(world, 1 if null == "flags" else None), world, rank, slot, ep, None)
    elif entry == "mean":
        st = lib.b2_scalar_allreduce_mean(base + 0xa00000, base + 0xb00000, arr(world, null, 0x200000), arr(world),
                                          world, rank, slot, ep, None)
    else:
        st = lib.b2_grad_norm_finalize(base + 0xc00000, 4, arr(world, null if null != "flags" else None, 0x300000),
                                       arr(world, 1 if null == "flags" else None), world, rank, slot, ep, 1.0, None,
                                       None, base + 0xd00000, base + 0xd00010, base + 0xd00020, None)
    out[name] = [int(st), L.last_error()]
print(json.dumps(out))
"""
REJECT = [  # (id, entry, world, rank, slot, bytes, null peer, prefix, word in the error)
    ("barrier-world-0", "barrier", 0, 0, 0, 0, None, "peer_barrier: ", "world=0"),
    ("barrier-world-9", "barrier", 9, 0, 0, 0, None, "peer_barrier: ", "world=9"),
    ("barrier-rank", "barrier", 2, 2, 0, 0, None, "peer_barrier: ", "rank=2"),
    ("barrier-slot-64", "barrier", 2, 0, 64, 0, None, "peer_barrier: ", "slot=64"),
    ("barrier-null-peer", "barrier", 3, 0, 0, 0, 2, "peer_barrier: ", "null peer pointer for rank 2"),
    ("allgather-bytes-6", "allgather", 2, 0, 3, 6, None, "allgather_rows: ", "bytes=6"),
    ("allgather-bytes-0", "allgather", 2, 0, 3, 0, None, "allgather_rows: ", "bytes=0"),
    ("allgather-world-9", "allgather", 9, 0, 3, 64, None, "allgather_rows: ", "world=9"),
    ("allgather-rank", "allgather", 2, 5, 3, 64, None, "allgather_rows: ", "rank=5"),
    ("allgather-slot-64", "allgather", 2, 0, 64, 64, None, "allgather_rows: ", "slot=64"),
    ("allgather-null-dst", "allgather", 2, 0, 3, 64, 1, "allgather_rows(dst): ", "null peer pointer for rank 1"),
    ("allgather-null-flags", "allgather", 2, 0, 3, 64, "flags", "allgather_rows(flags): ",
     "null peer pointer for rank 1"),
    ("mean-world-0", "mean", 0, 0, 2, 0, None, "scalar_allreduce_mean: ", "world=0"),
    ("mean-world-9", "mean", 9, 0, 2, 0, None, "scalar_allreduce_mean: ", "world=9"),
    ("mean-rank", "mean", 3, 3, 2, 0, None, "scalar_allreduce_mean: ", "rank=3"),
    ("mean-slot-64", "mean", 2, 0, 64, 0, None, "scalar_allreduce_mean: ", "slot=64"),
    ("mean-null-scratch", "mean", 2, 1, 2, 0, 0, "scalar_allreduce_mean(scratch): ", "null peer pointer for rank 0"),
    ("finalize-world-0", "finalize", 0, 0, 5, 0, None, "grad_norm_finalize: ", "world=0"),
    ("finalize-world-9", "finalize", 9, 0, 5, 0, None, "grad_norm_finalize: ", "world=9"),
    ("finalize-rank", "finalize", 2, 2, 5, 0, None, "grad_norm_finalize: ", "rank=2"),
    ("finalize-slot-64", "finalize", 2, 0, 64, 0, None, "grad_norm_finalize: ", "slot=64"),
    ("finalize-null-peer", "finalize", 2, 0, 5, 0, 1, "grad_norm_finalize: ", "null peer pointer for rank 1"),
    ("finalize-null-flags", "finalize", 3, 0, 5, 0, "flags", "grad_norm_finalize: ", "null peer pointer for rank 1"),
]
ACCEPT = [  # calls that must get past every argument check (and then fail for want of a device)
    ("barrier-ok", "barrier", 8, 7, 63, 0, None),
    ("barrier-world-1", "barrier", 1, 0, 0, 0, None),
    ("allgather-ok", "allgather", 3, 2, 3, 4 * 1001, None),
    ("mean-ok", "mean", 2, 1, 2, 0, None),
    ("finalize-ok", "finalize", 8, 3, 63, 0, None),
    ("finalize-world-1-null-peers", "finalize", 1, 0, 64, 0, 0),    # world 1 exchanges nothing: no peer is read
]


@pytest.fixture(scope="module")
def child_results():
    env = dict(os.environ)
    env["CUDA_VISIBLE_DEVICES"] = ""
    lib_py = os.path.join(ROOT, "pytorch-distributed-nlp_b200", "_lib.py")
    cases = [c[:7] for c in REJECT] + ACCEPT
    r = subprocess.run([sys.executable, "-c", _CHILD, lib_py, json.dumps(cases)], env=env, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", REJECT, ids=lambda c: c[0])
def test_argument_is_rejected(child_results, case):
    st, err = child_results[case[0]]
    assert st != 0 and err.startswith(case[7]) and case[8] in err, err


@pytest.mark.parametrize("case", ACCEPT, ids=lambda c: c[0])
def test_valid_arguments_pass_the_checks(child_results, case):
    st, err = child_results[case[0]]
    assert st != 0, case[0]
    for phrase in ("world=", "slot=", "bytes=", "null", "bad args"):
        assert phrase not in err, (case[0], err)


# ======================================================================================================================
# Part A: the flag kernels on one device, every wait met before the launch
# ======================================================================================================================
class Peers:
    """world local flag pads (and optionally payload buffers) standing in for the peers, filled with a sentinel"""

    def __init__(self, world, dev, payload_bytes=0, fill=SENT):
        self.world, self.dev = world, dev
        self.flags = [lb.CommBuf(L.FLAG_SLOTS * world * 4, dev) for _ in range(world)]
        self.data = [lb.CommBuf(payload_bytes, dev) for _ in range(world)] if payload_bytes else []
        for b in self.flags + self.data:
            b.u32().fill_(i32(fill))
        self.ctr = torch.zeros(L.FLAG_SLOTS, dtype=torch.int32, device=dev)

    def post(self, rank, slot, e):
        """every flag rank `rank` polls at `slot` set to epoch e (its own word to e + 7: the kernel's store shows)"""
        own = self.flags[rank].u32()
        for q in range(self.world):
            own[slot * self.world + q] = i32(e if q != rank else e + 7)

    def flag_ptrs(self):
        return L.ptr_array([b.ptr for b in self.flags])

    def data_ptrs(self):
        return L.ptr_array([b.ptr for b in self.data])

    def snapshot(self):
        return [b.u32().cpu().clone() for b in self.flags], [b.u32().cpu().clone() for b in self.data]

    def launch(self, entry, args, rank, slot):
        return flag_launch(entry, args, (self.ctr, slot), (self.flags[rank].u32(), slot), self.world)

    def free(self):
        for b in self.flags + self.data:
            b.free()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _expect_flags(P, before, rank, slot, e):
    want = [t.clone() for t in before]
    for q in range(P.world):
        want[q][slot * P.world + rank] = i32(e)
    for q in range(P.world):
        got = P.flags[q].u32().cpu()
        bad = (got != want[q]).nonzero().flatten().tolist()
        assert not bad, ("flag words changed or missing", q, bad[:8])


BARRIER_CASES = sorted({(w, r, s) for w in (1, 2, 3, 8) for r in (0, w // 2, w - 1) for s in (0, L.FLAG_SLOTS - 1)})


@pytest.mark.gpu
@pytest.mark.parametrize("world,rank,slot", BARRIER_CASES)
def test_peer_barrier(cuda_dev, world, rank, slot):
    P = Peers(world, cuda_dev)
    try:
        P.ctr[slot] = 41
        P.post(rank, slot, 42)
        before, _ = P.snapshot()
        ctr_before = P.ctr.cpu().clone()
        e = P.launch("b2_peer_barrier", (P.flag_ptrs(), world, rank, slot, P.ctr.data_ptr() + 4 * slot, _stream()),
                     rank, slot)
        assert e == 42
        ctr_want = ctr_before.clone()
        ctr_want[slot] = 42
        assert torch.equal(P.ctr.cpu(), ctr_want), "the epoch counter moves by one, at its slot only"
        _expect_flags(P, before, rank, slot, e)
    finally:
        P.free()


@pytest.mark.gpu
def test_peer_barrier_epoch_wrap(cuda_dev):
    world, rank, slot = 3, 1, 7
    P = Peers(world, cuda_dev)
    try:
        P.ctr[slot] = i32(0xFFFFFFFE)
        args = (P.flag_ptrs(), world, rank, slot, P.ctr.data_ptr() + 4 * slot, _stream())
        P.post(rank, slot, 0xFFFFFFFF)
        before, _ = P.snapshot()
        assert P.launch("b2_peer_barrier", args, rank, slot) == 0xFFFFFFFF
        _expect_flags(P, before, rank, slot, 0xFFFFFFFF)
        # the peers' flags still read 0xFFFFFFFF: one epoch short of 0, the helper must refuse
        with pytest.raises(AssertionError, match="does not satisfy epoch 0x00000000"):
            P.launch("b2_peer_barrier", args, rank, slot)
        assert int(P.ctr[slot]) & U32 == 0xFFFFFFFF, "a refused launch changed the counter"
        P.post(rank, slot, 0)
        before, _ = P.snapshot()
        assert P.launch("b2_peer_barrier", args, rank, slot) == 0
        assert int(P.ctr[slot]) == 0
        _expect_flags(P, before, rank, slot, 0)
    finally:
        P.free()


@pytest.mark.gpu
@pytest.mark.parametrize("world,rank,words", [(1, 0, 1), (2, 1, 1), (3, 1, 1001), (8, 7, 1001), (3, 0, 1 << 18),
                                              (8, 4, 1 << 18)])
def test_allgather_rows(cuda_dev, world, rank, words):
    slot = ddp_mod_slot("_SLOT_GATHER")
    P = Peers(world, cuda_dev, payload_bytes=4 * words * world)
    try:
        src = torch.randint(-(1 << 31), (1 << 31) - 1, (words,), dtype=torch.int32, device=cuda_dev,
                            generator=torch.Generator(cuda_dev).manual_seed(words + rank))
        P.ctr[slot] = 9
        P.post(rank, slot, 10)
        fbefore, dbefore = P.snapshot()
        e = P.launch("b2_allgather_rows", (src.data_ptr(), 4 * words, P.data_ptrs(), P.flag_ptrs(), world, rank, slot,
                                           P.ctr.data_ptr() + 4 * slot, _stream()), rank, slot)
        _expect_flags(P, fbefore, rank, slot, e)
        s = src.cpu()
        for q in range(world):
            want = dbefore[q].clone()
            want[rank * words:(rank + 1) * words] = s
            assert torch.equal(P.data[q].u32().cpu(), want), ("dst of rank %d" % q)
    finally:
        P.free()


def ddp_mod_slot(name):
    return getattr(lb.ddp_mod, name)


@pytest.mark.gpu
@pytest.mark.parametrize("world,rank", [(3, 1), (8, 5), (2, 0)])
def test_scalar_allreduce_mean(cuda_dev, world, rank):
    """the rank-order fp32 sum of the posted values / (float)world, bitwise; values that cancel show the order"""
    slot = ddp_mod_slot("_SLOT_LOSS")
    P = Peers(world, cuda_dev)
    scratch = [lb.CommBuf(2 * world * 4, cuda_dev) for _ in range(world)]
    try:
        for b in scratch:
            b.u32().fill_(i32(SENT))
        src = torch.zeros(1, dtype=torch.float32, device=cuda_dev)
        dst = torch.full((1,), 7.0, dtype=torch.float32, device=cuda_dev)
        P.ctr[slot] = 100
        base = [1e8, 1.0, -1e8, 3.0, -2.5, 1e-3, 7.0, -1e8]
        for call in range(2):
            e = (int(P.ctr[slot]) + 1) & U32
            par = e & 1
            vals = [torch.tensor(v * (1 + call), dtype=torch.float32) for v in base[:world]]
            if world == 2:
                vals = [torch.tensor(1e8, dtype=torch.float32), torch.tensor(1.0 + call, dtype=torch.float32)]
            for q in range(world):
                if q != rank:
                    scratch[rank].f32()[par * world + q] = vals[q]
            src.fill_(float(vals[rank]))
            P.post(rank, slot, e)
            before = [b.u32().cpu().clone() for b in scratch]
            fbefore, _ = P.snapshot()
            got_e = P.launch("b2_scalar_allreduce_mean",
                             (src.data_ptr(), dst.data_ptr(), L.ptr_array([b.ptr for b in scratch]), P.flag_ptrs(),
                              world, rank, slot, P.ctr.data_ptr() + 4 * slot, _stream()), rank, slot)
            assert got_e == e
            want = lb.rank_mean(vals)
            assert dst.cpu()[0].view(torch.int32) == want.view(torch.int32), (call, float(dst), float(want))
            if world > 2:
                assert float(want) != float(sum(float(v) for v in vals) / world) or call, "values do not show the order"
            _expect_flags(P, fbefore, rank, slot, e)
            for q in range(world):
                w = before[q].clone()
                w[par * world + rank] = src.cpu().view(torch.int32)[0]
                assert torch.equal(scratch[q].u32().cpu(), w), ("scratch of rank %d" % q, call)
    finally:
        P.free()
        for b in scratch:
            b.free()


# ---- b2_grad_norm_finalize at world > 1 --------------------------------------------------------------------------------
class Finalize:
    """one rank's b2_grad_norm_finalize at world > 1 with the other ranks' shares and flags posted"""

    def __init__(self, world, rank, dev):
        self.world, self.rank, self.dev = world, rank, dev
        self.slot = ddp_mod_slot("_SLOT_CLIP")
        self.P = Peers(world, dev)
        self.scratch = [lb.CommBuf(2 * world * 4, dev) for _ in range(world)]
        self.out = torch.zeros(3, dtype=torch.float32, device=dev)       # norm, coef, skip

    def run(self, partials, other_shares, max_norm, grad_scale=None, found_inf=None):
        world, rank, slot = self.world, self.rank, self.slot
        e = (int(self.P.ctr[slot]) + 1) & U32
        par = e & 1
        for q in range(world):
            if q != rank:
                self.scratch[rank].f32()[par * world + q] = float(other_shares[q])
        self.P.post(rank, slot, e)
        p = partials.to(self.dev, torch.float64).contiguous()
        self.out.zero_()
        self.P.launch("b2_grad_norm_finalize",
                      (p.data_ptr(), p.numel(), L.ptr_array([b.ptr for b in self.scratch]), self.P.flag_ptrs(), world,
                       rank, slot, self.P.ctr.data_ptr() + 4 * slot, max_norm, L.ptr(grad_scale), L.ptr(found_inf),
                       self.out.data_ptr(), self.out.data_ptr() + 4, self.out.data_ptr() + 8, _stream()), rank, slot)
        return self.out.cpu()

    def free(self):
        self.P.free()
        for b in self.scratch:
            b.free()


def finalize_world1(partials, max_norm, dev, grad_scale=None, found_inf=None):
    p = partials.to(dev, torch.float64).contiguous()
    out = torch.zeros(3, dtype=torch.float32, device=dev)
    L.call("b2_grad_norm_finalize", p.data_ptr(), p.numel(), None, None, 1, 0, 0, None, max_norm, L.ptr(grad_scale),
           L.ptr(found_inf), out.data_ptr(), out.data_ptr() + 4, out.data_ptr() + 8, _stream())
    torch.cuda.synchronize()
    return out.cpu()


def restate_norm(shares32, world, grad_scale=None):
    """the finalize's arithmetic: rank-order fp32 mean of the shares, x world in fp64, sqrt, fp32 [/ scale]"""
    mean = lb.rank_mean(shares32)
    norm = torch.tensor(math.sqrt(float(mean) * world), dtype=torch.float64).to(torch.float32)
    return norm / grad_scale if grad_scale is not None else norm


def exact_partials(total_units, n, g):
    """n fp64 slot sums, dyadic (k * 2^-30), summing exactly to total_units * 2^-30 in any order"""
    cuts = torch.sort(torch.randint(0, total_units, (n - 1,), generator=g)).values.tolist()
    edges = [0] + cuts + [total_units]
    return torch.tensor([(edges[i + 1] - edges[i]) * 2.0 ** -30 for i in range(n)], dtype=torch.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("world,rank", [(2, 1), (3, 2), (8, 0)])
def test_grad_norm_finalize_world_gt1(cuda_dev, world, rank):
    """total_norm within |norm - sqrt(S)| <= ((world + 3) / 2) u sqrt(S), S = the fp64 sum of the shares (positive):
    the shares' fp32 rounding (u each), the world-term fp32 sum ((world - 1) u), 1/world (u), x world in fp64 (exact:
    a 24-bit mantissa times at most 8), sqrt halving the relative error, and the final fp32 rounding (u).  clip_coef is
    bitwise torch's formula on that norm; skip as at world 1"""
    g = torch.Generator().manual_seed(world * 10 + rank)
    F_ = Finalize(world, rank, cuda_dev)
    worst = 0.0
    try:
        for trial in range(6):
            units = int(torch.randint(1 << 34, 1 << 44, (1,), generator=g))
            partials = exact_partials(units, 37, g)
            own = units * 2.0 ** -30
            shares64 = [float(torch.rand((), generator=g, dtype=torch.float64) * 3e4) for _ in range(world)]
            shares64[rank] = own
            shares32 = [torch.tensor(s, dtype=torch.float64).to(torch.float32) for s in shares64]
            max_norm = [1.0, 1e6, 0.5][trial % 3]
            out = F_.run(partials, shares32, max_norm)
            want = restate_norm(shares32, world)
            assert out[0].view(torch.int32) == want.view(torch.int32), (float(out[0]), float(want))
            ref = math.sqrt(sum(shares64))
            bound = (world + 3) / 2 * U * ref * (1 + 1e-6)
            err = abs(float(out[0]) - ref)
            assert err <= bound, (err, bound)
            worst = max(worst, err / bound)
            coef = lb.torch_clip_coef(out[0], max_norm)
            assert out[1].view(torch.int32) == coef.view(torch.int32), (float(out[1]), float(coef))
            assert float(out[2]) == 0.0
        # GradScaler: the norm of the unscaled gradients (a power-of-two scale: exact), found_inf skips
        gs = torch.full((1,), 65536.0, device=cuda_dev)
        for fi_v in (0.0, 1.0):
            fi = torch.full((1,), fi_v, device=cuda_dev)
            out = F_.run(partials, shares32, 1.0, grad_scale=gs, found_inf=fi)
            want = restate_norm(shares32, world, 65536.0)
            assert out[0].view(torch.int32) == want.view(torch.int32)
            assert out[1].view(torch.int32) == lb.torch_clip_coef(out[0], 1.0).view(torch.int32)
            w1 = finalize_world1(partials, 1.0, cuda_dev, gs, fi)
            assert float(out[2]) == float(w1[2]) == fi_v
        # a NaN share: a NaN norm and coefficient; skipped only under a GradScaler, as at world 1 with a NaN slot
        nan_shares = list(shares32)
        nan_shares[(rank + 1) % world] = torch.tensor(float("nan"))
        nan_partials = partials.clone()
        nan_partials[3] = float("nan")
        for scale in (None, gs):
            out = F_.run(partials, nan_shares, 1.0, grad_scale=scale,
                         found_inf=torch.zeros(1, device=cuda_dev) if scale is not None else None)
            w1 = finalize_world1(nan_partials, 1.0, cuda_dev, scale,
                                 torch.zeros(1, device=cuda_dev) if scale is not None else None)
            assert math.isnan(float(out[0])) and math.isnan(float(out[1])) and math.isnan(float(w1[0]))
            assert float(out[2]) == float(w1[2]) == (1.0 if scale is not None else 0.0)
    finally:
        F_.free()
    print("finalize world %d: worst |norm - sqrt(S)| / bound = %.3f" % (world, worst))


@pytest.mark.gpu
def test_finalize_range_limit(cuda_dev):
    """Pinned behaviour: at world > 1 each rank's share of the sum of squares is exchanged as fp32, so a share above
    FLT_MAX (3.4e38, a gradient norm above 1.8e19) is inf and so is the norm; world 1 keeps the sum in fp64 until the
    square root and stays finite.  Only a run that has already diverged gets there (its coefficient is then 0 rather
    than ~1e-19 at world 1), so it is not changed."""
    partials = torch.tensor([6e38, 4e38], dtype=torch.float64)
    w1 = finalize_world1(partials, 1.0, cuda_dev)
    assert math.isfinite(float(w1[0])) and abs(float(w1[0]) - math.sqrt(1e39)) <= 1e-6 * math.sqrt(1e39)
    F_ = Finalize(2, 0, cuda_dev)
    try:
        out = F_.run(partials, [None, torch.tensor(1.0)], 1.0)
    finally:
        F_.free()
    assert math.isinf(float(out[0])) and float(out[1]) == 0.0


# ======================================================================================================================
# Part B / C: the loopback peer group
# ======================================================================================================================
NODROP = dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
_STATE = {}


def initial_state(cfg, key):
    if key not in _STATE:
        _STATE[key] = state_from_hf_init(cfg, seed=123)
    return _STATE[key]


def groups(m):
    no_decay = ["bias", "LayerNorm.weight"]
    return [{"params": [p for n, p in m.named_parameters() if not any(nd in n for nd in no_decay)],
             "weight_decay": 0.01},
            {"params": [p for n, p in m.named_parameters() if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]


OPTIMIZERS = {
    "hf_adamw": lambda m: b2.AdamW(groups(m), lr=1e-3),
    "torch_adamw": lambda m: b2.TorchAdamW(groups(m), lr=1e-3, weight_decay=0.01),
    "adam_amsgrad": lambda m: b2.Adam(groups(m), lr=1e-3, amsgrad=True),
    "sgd": lambda m: b2.SGD(groups(m), lr=1e-2, momentum=0.9, nesterov=True),
}


def fwd_bwd(model, batch, dev):
    d = to_dev(batch, dev)
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    loss = F.cross_entropy(out[1], d["label"])
    loss.backward()
    return loss.detach()


def gathered_master(models, world):
    """the fp32 masters as the owners hold them: every slice from the rank that updates it"""
    lay = models[0]._layout
    out = torch.empty_like(models[0]._flat)
    for (b, e, _label) in lay.buckets:
        for q in range(world):
            sb, se = DDP._bucket_slice(b, e, q, world)
            out[sb:se] = models[q]._flat[sb:se]
    return out


def check_ownership(rec, lay, world):
    """the recorded update ranges tile every bucket exactly once, each is the rank's _bucket_slice, 8-aligned; empty
    slices launch nothing"""
    ups = [u for u in rec.updates if u["world"] == world]
    for u in ups:
        assert u["end"] > u["begin"], "ownership: rank %d launched the empty range [%d, %d)" % (
            u["rank"], u["begin"], u["end"])
        assert any(b <= u["begin"] and u["end"] <= e for (b, e, _l) in lay.buckets), \
            "ownership: rank %d's range [%d, %d) lies in no bucket" % (u["rank"], u["begin"], u["end"])
    for (b, e, label) in lay.buckets:
        mine = sorted([u for u in ups if b <= u["begin"] < e], key=lambda u: u["begin"])
        for q in range(world):
            sb, se = DDP._bucket_slice(b, e, q, world)
            got = [(u["begin"], u["end"]) for u in mine if u["rank"] == q]
            want = [(sb, se)] if se > sb else []
            assert got == want, "ownership: bucket %s rank %d updated %s, its slice is %s" % (label, q, got, want)
            assert all(x % 8 == 0 for g in got for x in g), "ownership: unaligned range"
        at = b
        for u in mine:
            assert u["begin"] == at, "ownership: bucket %s not tiled exactly once at %d" % (label, at)
            at = u["end"]
        assert at == e, "ownership: bucket %s ends at %d, not %d" % (label, at, e)


def check_delivery(models, world, grads_before):
    """shadow == bf16(gathered master) on every rank, bitwise; gradient buffers untouched by the step"""
    want = gathered_master(models, world).to(torch.bfloat16)
    for r, m in enumerate(models):
        eng = m._engine
        bad = (eng.shadow.view(torch.int16) != want.view(torch.int16)).nonzero().flatten()
        assert bad.numel() == 0, "delivery: rank %d's shadow differs from bf16(master) at %d elements, first %s" % (
            r, bad.numel(), bad[:4].tolist())
        assert torch.equal(eng.grads.view(torch.int16), grads_before[r]), "rank %d's gradients changed" % r


def state_buffers(opt):
    opt._gather_state()
    st = opt._dev_state
    return {k: st[k] for k in opt._flat_keys if st.get(k) is not None}


def run_group(world, make_opt, batches_per_step, dma, cfg, key, monkeypatch, plant=None, ref=True, check=True,
              clip=None):
    """Steps N loopback replicas (and, with ref, one unwrapped world-1 replica on rank 0's batches) eagerly; returns
    what the checks need.  Each step checks ownership and delivery and runs loss_reduce.  make_opt: a name of
    OPTIMIZERS or a factory.  A rank's batch may be a list of micro-batches: all but the last run inside no_sync().
    clip: max_norm of a clip_grad_norm_ before every step (collective: in N threads)."""
    dev = torch.device("cuda", 0)
    state = initial_state(cfg, key)
    make_opt = OPTIMIZERS[make_opt] if isinstance(make_opt, str) else make_opt
    monkeypatch.setenv("B2_DDP_DMA", "1" if dma else "0")
    res = {"losses": [], "loss_mean": [], "forms": set(), "ref_forms": set(), "grads": [], "passes": [], "clip": [],
           "updates": []}
    forms = ("b2_bucket_reduce", "b2_adamw_background", "b2_sgd_background", "b2_adam_background")
    with lb.Group(world, plant=plant) as g:
        models = [make_model(cfg, state, dev) for _ in range(world)]
        wrappers, opts = g.wrap(models, make_opt)
        res["init_master"] = models[0]._flat.clone()
        res["decay"] = opts[0]._decay_flags_cpu.clone()
        if ref:
            rmodel = make_model(cfg, state, dev)
            ropt = make_opt(rmodel)
        for s, batches in enumerate(batches_per_step):
            losses, passes = [], []
            g.rec.clear()
            g.rec.snap_accum = True
            for r in range(world):
                g.fake.local.rank = g.driving = r
                micro = batches[r] if isinstance(batches[r], list) else [batches[r]]
                for b in micro[:-1]:
                    with wrappers[r].no_sync():
                        fwd_bwd(wrappers[r], b, dev)
                losses.append(fwd_bwd(wrappers[r], micro[-1], dev))
            g.rec.snap_accum = False
            torch.cuda.synchronize()
            res["passes"].append(list(g.rec.accum))
            res["losses"].append([float(x) for x in losses])
            res["loss_mean"].append(g.run(lambda r: wrappers[r].loss_reduce(losses[r]).cpu()))
            grads = [m._engine.grads.view(torch.int16).clone() for m in models]
            res["grads"].append(grads)
            if clip is not None:
                g.run(lambda r: b2.clip_grad_norm_(wrappers[r].parameters(), clip))
                torch.cuda.synchronize()
                res["clip"].append([dict({k: o._clip_buf[k].clone() for k in ("stash", "partials", "norm", "coef")},
                                         ranges=list(o._clip_buf["ranges"]), stash_off=list(o._clip_buf["stash_off"]),
                                         slot_off=list(o._clip_buf["slot_off"]),
                                         coef_ptr=o._clip_buf["coef"].data_ptr(),
                                         stash_ptr=o._clip_buf["stash"].data_ptr()) for o in opts])
            g.rec.clear()
            g.step(opts)
            res["updates"].append(list(g.rec.updates))
            res["forms"] |= {n for n in g.rec.names if n.startswith(forms)}
            if check:
                check_ownership(g.rec, models[0]._layout, world)
                check_delivery(models, world, grads)
            if ref:
                g.rec.clear()
                fwd_bwd(rmodel, batches[0], dev)
                assert torch.equal(rmodel._engine.grads.view(torch.int16), grads[0]) or \
                    any(batches[r] is not batches[0] for r in range(world))
                ropt.step()
                torch.cuda.synchronize()
                res["ref_forms"] |= {n for n in g.rec.names if n.startswith(forms)}
        res["master"] = gathered_master(models, world)
        res["shadows"] = [m._engine.shadow.clone() for m in models]
        res["state"] = [{k: v.clone() for k, v in state_buffers(o).items()} for o in opts]
        res["steps"] = [int(o._dev_state["step"]) for o in opts]
        # (copies: the state dicts are views into the peer buffers, which close() frees)
        res["model_sd"] = [{k: v.clone() for k, v in m.state_dict().items()} for m in models]
        res["opt_sd"] = [clone_sd(o.state_dict()) for o in opts]
        if ref:
            res["ref_master"] = rmodel._flat.clone()
            res["ref_shadow"] = rmodel._engine.shadow.clone()
            res["ref_state"] = {k: v.clone() for k, v in state_buffers(ropt).items()}
            res["ref_step"] = int(ropt._dev_state["step"])
            res["ref_opt_sd"] = clone_sd(ropt.state_dict())
        # close(): every replica keeps working on private buffers with the same values
        g.close()
        comm_ptrs = set()
        for m in models:
            assert m._ddp is None
        for r, m in enumerate(models):
            assert torch.equal(m._flat, res["master"]), "close(): rank %d's masters changed" % r
            assert torch.equal(m._engine.shadow, res["shadows"][r])
            comm_ptrs.add(m._flat.data_ptr())
        assert len(comm_ptrs) == world, "close(): replicas share a master buffer"
        for o, st in zip(opts, res["state"]):
            for k, v in st.items():
                assert torch.equal(o._dev_state[k], v), "close(): state %s changed" % k
        res["logits_after_close"] = []
        b0 = batches_per_step[0][0]
        d = to_dev(b0[-1] if isinstance(b0, list) else b0, dev)
        for m in models:
            m.eval()
            with torch.no_grad():
                res["logits_after_close"].append(m(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                                                   attention_mask=d["attention_mask"]).logits.clone())
    # loss_reduce: the rank-order fp32 mean of the ranks' losses, the same on every rank
    for s, per_rank in enumerate(res["loss_mean"]):
        want = lb.rank_mean([torch.tensor(x, dtype=torch.float32) for x in res["losses"][s]])
        for r, v in enumerate(per_rank):
            assert v.reshape(()).view(torch.int32) == want.view(torch.int32), ("loss_reduce", s, r, float(v))
    return res


def clone_sd(sd):
    return {"state": {i: {k: v.clone() if isinstance(v, torch.Tensor) else v for k, v in e.items()}
                      for i, e in sd["state"].items()}, "param_groups": sd["param_groups"]}


def _same_batches(cfg, world, steps=3):
    return [[bert_ref.synthetic_batch(cfg, 4, 128, 7000 + 10 * s, padded=(s % 2 == 1))] * world for s in range(steps)]


def _assert_sd_equal(a, b, what):
    assert a["param_groups"] == b["param_groups"], what
    assert a["state"].keys() == b["state"].keys(), what
    for i in a["state"]:
        for k, v in a["state"][i].items():
            w = b["state"][i][k]
            if isinstance(v, torch.Tensor):
                assert torch.equal(v.cpu(), w.cpu()), (what, i, k)
            else:
                assert v == w, (what, i, k)


@pytest.fixture
def deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(prev)


SAME_BATCH = [(w, o, dma) for w in (2, 4, 8) for o in OPTIMIZERS for dma in (False, True)
              if dma is False or o == "hf_adamw" or w == 4]


@pytest.mark.gpu
@pytest.mark.parametrize("world,opt_name,dma", SAME_BATCH,
                         ids=lambda x: str(x) if not isinstance(x, bool) else ("dma" if x else "kernel"))
def test_same_batch_is_world_1(cuda_dev, monkeypatch, deterministic, world, opt_name, dma):
    """The same batch on every rank: N g is exact in fp32 for a bf16 g and 1/N a power of two, so masters, shadows,
    every state buffer, the step counters and optimizer.state_dict() are bitwise those of one replica stepped alone.
    The backward runs the fixed-order form, so every replica's gradients are bitwise the reference's."""
    cfg = tiny_config(**NODROP)
    res = run_group(world, opt_name, _same_batches(cfg, world), dma, cfg, "tiny", monkeypatch)
    # both sides run the reduce form of the update
    assert res["forms"] and all(f.startswith("b2_bucket_reduce") for f in res["forms"]), res["forms"]
    assert res["ref_forms"] == res["forms"], (res["ref_forms"], res["forms"])
    assert torch.equal(res["master"], res["ref_master"]), "masters differ from world 1"
    for r in range(world):
        assert torch.equal(res["shadows"][r].view(torch.int16), res["ref_shadow"].view(torch.int16)), r
        assert res["steps"][r] == res["ref_step"]
        assert res["state"][r].keys() == res["ref_state"].keys()
        for k, v in res["state"][r].items():
            assert torch.equal(v, res["ref_state"][k]), ("state", r, k)
        _assert_sd_equal(res["opt_sd"][r], res["ref_opt_sd"], "optimizer.state_dict() of rank %d" % r)
        _assert_sd_equal(res["opt_sd"][r], res["opt_sd"][0], "ranks' optimizer.state_dict()")
        for k, v in res["model_sd"][r].items():
            if k in res["model_sd"][0] and "position_ids" not in k:
                assert torch.equal(v, res["model_sd"][0][k]), ("model.state_dict()", r, k)
        assert torch.equal(res["logits_after_close"][r], res["logits_after_close"][0])


@pytest.mark.gpu
def test_state_dict_is_the_owners_slices(cuda_dev, monkeypatch):
    """model.state_dict() on every rank (one-sided) equals the owners' master slices, concatenated"""
    cfg = tiny_config(**NODROP)
    world = 3
    batches = [[bert_ref.synthetic_batch(cfg, 4, 128, 500 + 10 * s + r) for r in range(world)] for s in range(2)]
    res = run_group(world, "hf_adamw", batches, False, cfg, "tiny", monkeypatch, ref=False)
    m = b2.BertForSequenceClassification(cfg)
    views = {}
    for name in m._params_by_name:
        off, shape = m._layout.entries[name]
        views[name] = res["master"][off:off + m._params_by_name[name].numel()].view(shape)
    for r in range(world):
        sd = res["model_sd"][r]
        for name, v in views.items():
            assert torch.equal(sd[name], v), (r, name)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_different_batches_match_oracle(cuda_dev, monkeypatch, deterministic, world):
    """Different batches per rank, dropout off: the per-rank losses within TOL_TRAJ of oracle.ddp_ref.train (as the
    2-GPU worker checks) and the final masters within its 2e-4; and the DMA form is bitwise the kernel form.  The
    backward runs the fixed-order form, so both runs start every step from the same gradients (checked)."""
    cfg = tiny_config(**NODROP)
    steps = 3
    batches = [[bert_ref.synthetic_batch(cfg, 4, 128, 7000 + 10 * s + r, padded=(s % 2 == 1)) for r in range(world)]
               for s in range(steps)]
    state = initial_state(cfg, "tiny")
    ref = {k: v.clone() for k, v in state.items()}
    hist = ddp_ref.train(ref, cfg, batches)
    def build(m):
        return b2.build_optimizer(m, type("A", (), {"weight_decay": 0.01, "learning_rate": 3e-5}))

    kern = run_group(world, build, batches, False, cfg, "tiny", monkeypatch, ref=False)
    dma = run_group(world, build, batches, True, cfg, "tiny", monkeypatch, ref=False)
    worst = 0.0
    for s in range(steps):
        for r in range(world):
            err = abs(kern["losses"][s][r] - float(hist[s]["loss_per_rank"][r]))
            worst = max(worst, err / TOL_TRAJ)
            assert err <= TOL_TRAJ, (s, r, err)
        err = abs(float(kern["loss_mean"][s][0]) - float(hist[s]["loss_mean"]))
        assert err <= TOL_TRAJ, ("loss_reduce", s, err)
    for k, v in ref.items():
        assert float((kern["model_sd"][0][k].cpu() - v).abs().max()) <= 2e-4, k
    for s in range(steps):
        for r in range(world):
            assert torch.equal(kern["grads"][s][r], dma["grads"][s][r]), ("gradients differ between the runs", s, r)
    assert torch.equal(kern["master"], dma["master"]), "DMA form differs from the kernel form"
    for r in range(world):
        assert torch.equal(kern["shadows"][r], dma["shadows"][r])
        for k in kern["state"][r]:
            assert torch.equal(kern["state"][r][k], dma["state"][r][k]), k
    print("world %d oracle trajectory: worst |dloss| / TOL_TRAJ = %.3f" % (world, worst))


# ---- N = 3: the only world whose fp32 mean is inexact -----------------------------------------------------------------
TORCH_TWINS = {  # torch's own optimizers with the hyperparameters of OPTIMIZERS, per parameter and group
    "torch_adamw": (lambda gs: torch.optim.AdamW(gs, lr=1e-3, weight_decay=0.01, fused=True), ("exp_avg", "exp_avg_sq")),
    "adam_amsgrad": (lambda gs: torch.optim.Adam(gs, lr=1e-3, amsgrad=True, fused=True),
                     ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")),
    "sgd": (lambda gs: torch.optim.SGD(gs, lr=1e-2, momentum=0.9, nesterov=True, foreach=False), ("momentum_buffer",)),
}
BF_U = 2.0 ** -8     # bf16 unit roundoff


def bf(g16):
    return g16.view(torch.bfloat16).float()


def rank_order_mean(grads):
    """what the reduce kernels form from the ranks' bf16 gradients: fp32 sum in rank order, times fl(1 / world)"""
    acc = torch.zeros_like(grads[0])
    for x in grads:
        acc = acc + x
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(len(grads)), dtype=torch.float32)
    return acc * inv.to(acc.device)


def ratio(got, want, bound):
    err = (got.double() - want).abs()
    assert bool((err <= bound).all()), "worst error is %.3g x its bound" % float((err / bound.clamp_min(1e-300)).max())
    return float((err / bound.clamp_min(1e-300)).max())


def adamw_ref(res, world, extra=0):
    from test_step_kernels import AdamWRef
    dev = res["init_master"].device
    dec = res["decay"].bool().repeat_interleave(8).to(dev)
    sel = torch.arange(res["init_master"].numel(), device=dev)
    return AdamWRef(res["init_master"], dec, sel, 1e-3, 0.01, 1, world, extra=extra)


def adamw_ratios(res, ref):
    m, v, w = ref.gather("exp_avg"), ref.gather("exp_avg_sq"), ref.gather("w")
    out = [ratio(res["master"], w, ref.ew)]
    for r in range(len(res["state"])):
        out.append(ratio(res["state"][r]["exp_avg"], m, ref.em))
        out.append(ratio(res["state"][r]["exp_avg_sq"], v, ref.ev))
    return max(out)


@pytest.mark.gpu
@pytest.mark.parametrize("opt_name", list(OPTIMIZERS))
def test_same_batch_world3(cuda_dev, monkeypatch, deterministic, opt_name):
    """The same batch on N = 3 ranks: the mean fl(3 g * fl(1/3)) is within 2u of g, not g.  HF AdamW: the masters and
    moments within test_step_kernels.AdamWRef's float64 bound (world 3 carries the mean's rounding).  TorchAdamW, Adam
    (amsgrad) and SGD: masters and state bitwise torch.optim.AdamW / Adam (fused=True, torch._fused_adamw_ /
    _fused_adam_) and torch.optim.SGD(foreach=False) fed that exact fp32 mean."""
    cfg = tiny_config(**NODROP)
    world = 3
    res = run_group(world, opt_name, _same_batches(cfg, world), False, cfg, "tiny", monkeypatch, ref=False)
    assert res["forms"] and all(f.startswith("b2_bucket_reduce") for f in res["forms"]), res["forms"]
    for grads in res["grads"]:
        assert all(torch.equal(g, grads[0]) for g in grads), "the ranks' gradients differ"
    if opt_name == "hf_adamw":
        ref = adamw_ref(res, world)
        for grads in res["grads"]:
            ref.step(bf(grads[0]).double())
        print("N = 3 same batch, HF AdamW: worst error / AdamWRef bound = %.3f" % adamw_ratios(res, ref))
        return
    make, keys = TORCH_TWINS[opt_name]
    mcpu = b2.BertForSequenceClassification(cfg)
    lay = mcpu._layout

    def view(flat, name):
        off, shape = lay.entries[name]
        return flat[off:off + mcpu._params_by_name[name].numel()].view(shape)

    names = list(mcpu._params_by_name)
    params = {n: torch.nn.Parameter(view(res["init_master"], n).clone()) for n in names}
    nd = lambda n: any(x in n for x in ("bias", "LayerNorm.weight"))
    topt = make([{"params": [params[n] for n in names if not nd(n)], "weight_decay": 0.01},
                 {"params": [params[n] for n in names if nd(n)], "weight_decay": 0.0}])
    for grads in res["grads"]:
        mean = rank_order_mean([bf(g) for g in grads])
        for n in names:
            params[n].grad = view(mean, n).clone()
        topt.step()
    for n in names:
        assert torch.equal(view(res["master"], n), params[n].detach()), ("master", n)
        for k in keys:
            for r in range(world):
                assert torch.equal(view(res["state"][r][k], n), topt.state[params[n]][k]), (k, n, r)


@pytest.mark.gpu
def test_no_sync_window_world3(cuda_dev, monkeypatch, deterministic):
    """Two passes inside no_sync() and a third outside (ACCUM STORE, ADD, FOLD) on each of N = 3 ranks, different
    micro-batches, two steps.  The folded gradient is bitwise bf16((g1 + g2) + g3) in fp32, and within
    2^-8 |S| + 2u (|g1| + |g2| + |g3|) of the float64 sum S (one bf16 rounding, two fp32 additions).  The update of
    that window is within AdamWRef's float64 bound of HF AdamW fed the float64 mean of the folded gradients."""
    cfg = tiny_config(**NODROP)
    world, steps = 3, 2
    batches = [[[bert_ref.synthetic_batch(cfg, 4, 128, 900 + 100 * s + 10 * r + k, padded=(k == 1)) for k in range(3)]
                for r in range(world)] for s in range(steps)]
    res = run_group(world, "hf_adamw", batches, False, cfg, "tiny", monkeypatch, ref=False)
    ref = adamw_ref(res, world)
    worst = 0.0
    for s in range(steps):
        passes = res["passes"][s]
        for r in range(world):
            mine = [p for p in passes if p[0] == r]
            assert [p[1] for p in mine] == [L.ACCUM_STORE, L.ACCUM_ADD, L.ACCUM_FOLD], [p[1] for p in mine]
            g1, g2, g3 = (p[4].float() for p in mine)
            folded = bf(res["grads"][s][r])
            assert torch.equal(folded, ((g1 + g2) + g3).to(torch.bfloat16).float()), ("fold", s, r)
            S = g1.double() + g2.double() + g3.double()
            bound = BF_U * S.abs() + 2 * U * (g1.abs() + g2.abs() + g3.abs()).double() + 2.0 ** -133
            worst = max(worst, ratio(folded, S, bound))
        ref.step(sum(bf(g).double() for g in res["grads"][s]) / world)
    upd = adamw_ratios(res, ref)
    print("N = 3 no_sync window: fold worst / bound = %.3f, update worst / AdamWRef bound = %.3f" % (worst, upd))


@pytest.mark.gpu
def test_clip_grad_norm_world3(cuda_dev, monkeypatch, deterministic):
    """clip_grad_norm_ at N = 3 (in N threads, as it is collective), two steps of HF AdamW, different batches.
    * every rank's stash is bitwise the rank-order fp32 mean of its slice of every bucket;
    * its partial sums of squares are within 8u of float64's sum of the squared means (fp32 fmaf over 8 elements per
      slot, then fp64);
    * the norm is the same on every rank and within ((world + 3) / 2 + 4) u sqrt(S) of float64's (the partials' 8u
      halved by the square root, plus the exchange's bound of test_grad_norm_finalize_world_gt1); the coefficient is
      bitwise torch's formula on it and below 1;
    * every bucket's update reads that rank's coefficient and stash slice, and the masters and moments are within
      AdamWRef's bound of HF AdamW fed coef x mean."""
    cfg = tiny_config(**NODROP)
    world, steps, max_norm = 3, 2, 0.05
    batches = [[bert_ref.synthetic_batch(cfg, 4, 128, 3000 + 10 * s + r) for r in range(world)] for s in range(steps)]
    res = run_group(world, "hf_adamw", batches, False, cfg, "tiny", monkeypatch, ref=False, clip=max_norm)
    lay = b2.BertForSequenceClassification(cfg)._layout
    ref = adamw_ref(res, world, extra=1)
    w_part, w_norm = 0.0, 0.0
    for s in range(steps):
        mean = rank_order_mean([bf(g) for g in res["grads"][s]])
        S = float((mean.double() ** 2).sum())
        clips = res["clip"][s]
        norm = clips[0]["norm"].cpu()
        for r, c in enumerate(clips):
            assert c["norm"].cpu().view(torch.int32) == norm.view(torch.int32), ("norm differs between ranks", r)
            assert c["coef"].cpu().view(torch.int32) == clips[0]["coef"].cpu().view(torch.int32)
            want_r = 0.0
            for idx, (b, e) in enumerate(c["ranges"]):
                assert (b, e) == DDP._bucket_slice(*lay.buckets[idx][:2], r, world)
                if e > b:
                    got = c["stash"][c["stash_off"][idx]:c["stash_off"][idx] + e - b]
                    assert torch.equal(got, mean[b:e]), ("stash", s, r, idx)
                    want_r += float((mean[b:e].double() ** 2).sum())
            p = float(c["partials"].sum())
            bound = 8.01 * U * want_r + 1e-300
            assert abs(p - want_r) <= bound, ("partials", s, r, p, want_r)
            w_part = max(w_part, abs(p - want_r) / bound)
        bound = ((world + 3) / 2 + 4.01) * U * math.sqrt(S)
        err = abs(float(norm) - math.sqrt(S))
        assert err <= bound, ("norm", s, err, bound)
        w_norm = max(w_norm, err / bound)
        coef = clips[0]["coef"].cpu()
        assert coef.view(torch.int32) == lb.torch_clip_coef(norm, max_norm).view(torch.int32)
        assert float(coef) < 1.0, "the test does not clip"
        ups = res["updates"][s]
        assert len(ups) == sum(1 for c in clips for (b, e) in c["ranges"] if e > b)
        for u in ups:
            c = clips[u["rank"]]
            idx = next(i for i, (b, e) in enumerate(lay.buckets[j][:2] for j in range(len(lay.buckets)))
                       if b <= u["begin"] < e)
            assert u["coef"] == c["coef_ptr"], ("the update does not read the coefficient", u["rank"], idx)
            assert u["grad_f32"] == c["stash_ptr"] + 4 * c["stash_off"][idx], ("stash slice", u["rank"], idx)
        ref.step(mean.double() * float(coef))
    upd = adamw_ratios(res, ref)
    print("N = 3 clip: partials worst / bound = %.3f, norm worst / bound = %.3f, update worst / AdamWRef bound = %.3f"
          % (w_part, w_norm, upd))


@pytest.mark.gpu
def test_same_batch_hidden_768(cuda_dev, monkeypatch, deterministic):
    """H 768, 2 layers, N = 4: bitwise world 1 (the fused dense + LayerNorm forward runs at this width)"""
    cfg = tiny_config(hidden_size=768, num_attention_heads=12, intermediate_size=3072, **NODROP)
    res = run_group(4, "hf_adamw", _same_batches(cfg, 4, steps=2), False, cfg, "h768", monkeypatch)
    assert torch.equal(res["master"], res["ref_master"])
    for r in range(4):
        assert torch.equal(res["shadows"][r], res["ref_shadow"])


# ======================================================================================================================
# Part D: planted defects, each failing its named check
# ======================================================================================================================
@pytest.mark.gpu
def test_planted_shifted_slice_fails_ownership(cuda_dev, monkeypatch):
    cfg = tiny_config(**NODROP)
    with pytest.raises(AssertionError, match="ownership: bucket embeddings rank 0"):
        run_group(3, "hf_adamw", _same_batches(cfg, 3, steps=1), False, cfg, "tiny", monkeypatch,
                  plant={"shift_slice": (0, 0, 8)}, ref=False)


@pytest.mark.gpu
def test_planted_dropped_shadow_fails_delivery(cuda_dev, monkeypatch):
    cfg = tiny_config(**NODROP)
    with pytest.raises(AssertionError, match="delivery: rank 2's shadow differs"):
        run_group(3, "hf_adamw", _same_batches(cfg, 3, steps=1), False, cfg, "tiny", monkeypatch,
                  plant={"drop_shadow": (1, 2)}, ref=False)


@pytest.mark.gpu
def test_planted_skipped_barrier_fails_lockstep(cuda_dev, monkeypatch):
    cfg = tiny_config(**NODROP)
    with pytest.raises(lb.Divergence, match=r"rank \d reached b2_peer_barrier slot [01] \(_SLOT_\w+\), "
                                            r"rank \d reached b2_peer_barrier slot [01] \(_SLOT_\w+\)") as ex:
        run_group(3, "hf_adamw", _same_batches(cfg, 3, steps=1), False, cfg, "tiny", monkeypatch,
                  plant={"skip_slot": (1, lb.ddp_mod._SLOT_GRADS_READY)}, ref=False)
    # whichever rank reports it, the message names the skipping rank 1 at _SLOT_UPDATE_DONE against _SLOT_GRADS_READY
    msg = str(ex.value)
    assert "rank 1 reached b2_peer_barrier slot 1 (_SLOT_UPDATE_DONE)" in msg and "(_SLOT_GRADS_READY)" in msg, msg
