"""The packed attention kernels at bins of 256, 384 and 512 tokens (b2_attention_{fwd,bwd}_packed_seq: the kSeg forms
of attention_fwd_kernel / attention_bwd_kernel, which visit only the 128-row blocks a segment reaches).  GPU.

* float64: ctx, lse and d_qkv of every (segment, head) against HF's attention in float64 at test_attention_reference's
  rounding-derived bounds, dropout off and on (the Philox replica of tests/parity.py with b the bin and seq the bin
  length).  The layouts: the Trainer's bins of a long-text batch, segments straddling the 128-row block boundaries,
  one S-token segment, S one-token segments, and unused rows (before a segment, after one, and whole blocks of them).
* One segment equals the padded kernel.  A bin holding one sequence gives what b2_attention_fwd / _bwd give the padded
  row, bit for bit with dropout on: ctx and lse of its rows, dK and dV of its keys.  dQ is the sum of the same
  per-key-block fp32 partials, added by atomics in no fixed order: the fp32 accumulators may differ by what reordering
  nkv additions can change, 2 nkv U sum_j |partial_j| (dq_reorder_bound), and the bf16 dQ by that plus one bf16 step.
* Isolation.  Rewriting the other segments' Q / K / V and dO with other finite values leaves a segment's ctx, lse, dK,
  dV (and dQ, for a segment inside one key block: its only nonzero dQ contribution) bit-identical, and its dQ
  accumulator within the reordering bound otherwise; with dO zero outside one segment, every other row of d_qkv is
  exactly zero.  Block skipping must not break either.
* Containment.  Segment words pack_batch never builds (an end past the bin, lo > hi, a key block whose first key's
  segment starts after its last key's ends) keep every read and dQ atomic inside their bin: the next bin's outputs are
  bit-identical to a run in which the malformed bin is well formed.  The malformed bin comes first, so a stray access
  would land in the next bin's rows, inside the buffers.
"""
import pytest
import torch

from parity import attn_keep_mask, packed_visibility
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.packing import pack_batch
from test_attention import SEED, SITE, STEP, attn_bwd, attn_fwd, contiguous, stream
from test_attention_reference import check_outputs
from test_packing_long import long_batch, long_config

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
U = 2.0 ** -24


def seg_words(bins, S):
    """int32 [len(bins), S] segment words; a bin is a list of (lo, hi); other rows are unused (a segment of their own)"""
    ar = torch.arange(S, dtype=torch.int32)
    out = (ar | ((ar + 1) << 16)).repeat(len(bins), 1)
    for b, segs in enumerate(bins):
        for lo, hi in segs:
            out[b, lo:hi] = lo | (hi << 16)
    return out


def long_layout(S):
    """every edge in one multi-bin batch of S-token bins"""
    cfg = long_config()
    batch = long_batch(cfg, 12, S, lo=4, hi=S // 2, S=S, long_rows=[(0, S - 1), (1, S // 2 + 3)])
    tr = pack_batch(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"], S)["segments"]
    straddle, total = [], 0                      # 100, 60, 200, ... cut at S: ends at rows 100, 160, 360, 450
    for n in (100, 60, 200, 90, 62):
        straddle.append(min(n, S - total))
        total += straddle[-1]
    own = seg_words([contiguous([S]), contiguous([1] * S), contiguous([n for n in straddle if n > 0]),
                     [(0, 20), (70, S - 30)], contiguous([3, 30, 2]), [(S - 200, S)], [(130, 131), (250, min(S, 260))]], S)
    return torch.cat([tr, own]).contiguous()


def fwd(qkv, seg, S, nh, p):
    dev = qkv.device
    rs = torch.tensor([SEED, STEP], dtype=torch.int64, device=dev)
    B = seg.shape[0]
    ctx = torch.empty(B * S, nh * 64, dtype=bf, device=dev)
    lse = torch.empty(B * nh * S, dtype=torch.float32, device=dev)
    L.call("b2_attention_fwd_packed_seq", qkv.data_ptr(), seg.data_ptr(), B, S, nh, 64, p, rs.data_ptr(), SITE,
           ctx.data_ptr(), lse.data_ptr(), None, stream())
    return ctx, lse.view(B, nh, S)


def bwd(qkv, seg, ctx, dctx, lse, S, nh, p):
    dev = qkv.device
    rs = torch.tensor([SEED, STEP], dtype=torch.int64, device=dev)
    B = seg.shape[0]
    dqkv = torch.zeros(B * S, 3 * nh * 64, dtype=bf, device=dev)
    dq_acc = torch.empty(B * S, nh * 64, dtype=torch.float32, device=dev)
    L.call("b2_attention_bwd_packed_seq", qkv.data_ptr(), seg.data_ptr(), ctx.data_ptr(), dctx.data_ptr(),
           lse.data_ptr(), B, S, nh, 64, p, rs.data_ptr(), SITE, dqkv.data_ptr(), dq_acc.data_ptr(), None, None,
           stream())
    return dqkv, dq_acc


def run(qkv, dctx, seg, S, nh, p):
    """ctx, lse [B, nh, S], d_qkv, and the fp32 dQ accumulator the backward left"""
    ctx, lse = fwd(qkv, seg, S, nh, p)
    dqkv, acc = bwd(qkv, seg, ctx, dctx, lse, S, nh, p)
    torch.cuda.synchronize()
    return ctx, lse, dqkv, acc


def padded_bwd(qkv, ctx, dctx, lse, mask, B, S, nh, p):
    """b2_attention_bwd; returns d_qkv and its fp32 dQ accumulator"""
    dev = qkv.device
    rs = torch.tensor([SEED, STEP], dtype=torch.int64, device=dev)
    dqkv = torch.zeros(B * S, 3 * nh * 64, dtype=bf, device=dev)
    dq_acc = torch.empty(B * S, nh * 64, dtype=torch.float32, device=dev)
    L.call("b2_attention_bwd", qkv.data_ptr(), mask.data_ptr(), ctx.data_ptr(), dctx.data_ptr(), lse.data_ptr(), B, S,
           nh, 64, p, rs.data_ptr(), SITE, dqkv.data_ptr(), dq_acc.data_ptr(), None, None, stream())
    torch.cuda.synchronize()
    return dqkv, dq_acc


def dq_reorder_bound(qkv, dctx, vis, B, S, nh, p):
    """[B*S, nh*64] float64: how far two fp32 sums of the same nkv per-key-block dQ partials, added in different
    orders, can lie apart: 2 (nkv - 1) U sum_j |partial_j| <= 2 nkv U (|dS| @ |K|).  |dS| is bounded without
    cancellation, 0.125 P (sc keep |dP| + |delta|), in float64 from the same operands and the kernels' keep mask; x 1.25
    covers the kernel's P, dP and bf16 dS tile lying off the float64 values (by well under 1 % where they matter)"""
    H, nkv = nh * 64, S // 128
    hd = lambda t: t.double().view(B, S, nh, 64).transpose(1, 2)
    q, k, v = (hd(qkv[:, i * H:(i + 1) * H]) for i in range(3))
    do = hd(dctx)
    s = torch.where(vis[:, None], (q @ k.transpose(-1, -2)) * 0.125, -torch.inf)
    P = torch.nan_to_num(torch.softmax(s, -1))
    del s
    keep = attn_keep_mask(B, nh, S, SEED, STEP, SITE, p, qkv.device)
    kf = keep.double() / (1.0 - p) if keep is not None else torch.ones(1, dtype=torch.float64, device=qkv.device)
    dp = do @ v.transpose(-1, -2)
    delta = (P * kf * dp).sum(-1, keepdim=True)
    mag = 0.125 * P * (kf * dp.abs() + delta.abs())
    del P, dp
    bound = 2 * nkv * U * 1.25 * (mag @ k.abs()) + 2.0 ** -120
    return bound.transpose(1, 2).reshape(B * S, H)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("S", [256, 384, 512])
def test_long_packed_vs_float64(cuda_dev, S, p):
    torch.manual_seed(S + int(10 * p))
    nh = 4
    seg = long_layout(S).to(cuda_dev)
    B = seg.shape[0]
    qkv = torch.randn(B * S, 3 * nh * 64, device=cuda_dev).to(bf)
    dctx = torch.randn(B * S, nh * 64, device=cuda_dev).to(bf)
    ctx, lse, dqkv, _ = run(qkv, dctx, seg, S, nh, p)
    keep = attn_keep_mask(B, nh, S, SEED, STEP, SITE, p, cuda_dev)
    check_outputs("packed S=%d p=%g" % (S, p), qkv, dctx, packed_visibility(seg), B, S, nh, p, keep, ctx, lse,
                  dqkv).assert_ok()


def _bf16_step(x):
    """one bf16 rounding step (ulp) at |x|"""
    e = torch.floor(torch.log2(x.float().abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


@pytest.mark.parametrize("S,n", [(256, 256), (384, 300), (512, 512), (512, 200)])
def test_one_segment_equals_the_padded_kernel(cuda_dev, S, n):
    """a bin holding one n-token sequence against the padded kernel on that row (mask = n ones), dropout on; dO of the
    padded rows is zero in both, as in the model (nothing reads those rows)"""
    torch.manual_seed(n)
    nh, p, B = 4, 0.1, 3
    H = nh * 64
    qkv = torch.randn(B * S, 3 * H, device=cuda_dev).to(bf)
    dctx = torch.randn(B * S, H, device=cuda_dev).to(bf)
    valid = (torch.arange(S, device=cuda_dev) < n).repeat(B)
    dctx[~valid] = 0
    seg = seg_words([[(0, n)]] * B, S).to(cuda_dev)
    mask = (torch.arange(S) < n).to(torch.int64).repeat(B, 1).to(cuda_dev)
    ctx_p, lse_p, dq_p, acc_p = run(qkv, dctx, seg, S, nh, p)
    ctx_d, lse_d = attn_fwd(qkv, B, S, nh, p, mask=mask)
    dq_d, acc_d = padded_bwd(qkv, ctx_d, dctx, lse_d, mask, B, S, nh, p)
    rows = valid
    assert torch.equal(ctx_p[rows], ctx_d[rows])
    assert torch.equal(lse_p[..., :n], lse_d[..., :n])
    assert torch.equal(dq_p[rows, H:], dq_d[rows, H:])              # dK | dV
    bound = dq_reorder_bound(qkv, dctx, packed_visibility(seg), B, S, nh, p)[rows]
    err = (acc_p[rows].double() - acc_d[rows].double()).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    err16 = (dq_p[rows, :H].double() - dq_d[rows, :H].double()).abs()
    tol16 = bound + _bf16_step(dq_d[rows, :H].double().abs() + bound).double()
    assert bool((err16 <= tol16).all()), float((err16 / tol16).max())
    print("S=%d n=%d: dQ accumulators differ in %d of %d elements, worst %.3g of the reordering bound"
          % (S, n, int((err > 0).sum()), err.numel(), float((err / bound).max())))


@pytest.mark.parametrize("S", [256, 512])
def test_segments_are_isolated(cuda_dev, S):
    torch.manual_seed(S + 1)
    nh, p = 4, 0.1
    H = nh * 64
    layout = [(0, 100), (100, 120), (120, 300 if S == 512 else 200), (S - 40, S)]   # rows between: unused
    seg = seg_words([layout, [(0, 60), (60, S)]], S).to(cuda_dev)
    B = seg.shape[0]
    qkv = torch.randn(B * S, 3 * H, device=cuda_dev).to(bf)
    dctx = torch.randn(B * S, H, device=cuda_dev).to(bf)
    base = run(qkv, dctx, seg, S, nh, p)
    bound = dq_reorder_bound(qkv, dctx, packed_visibility(seg), B, S, nh, p)
    # targets: (bin, lo, hi, inside one 128-key block)
    for b, lo, hi, one_block in [(0, 100, 120, True), (0, 120, layout[2][1], False), (1, 0, 60, True),
                                 (1, 60, S, False)]:
        rows = torch.zeros(B, S, dtype=torch.bool, device=cuda_dev)
        rows[b, lo:hi] = True
        rows = rows.view(-1)
        q2 = torch.where(rows[:, None], qkv, (torch.randn_like(qkv, dtype=torch.float32) * 3).to(bf))
        d2 = torch.where(rows[:, None], dctx, torch.randn_like(dctx, dtype=torch.float32).to(bf))
        ctx, lse, dqkv, acc = run(q2, d2, seg, S, nh, p)
        assert torch.equal(ctx[rows], base[0][rows]), (b, lo, hi)
        assert torch.equal(lse[b, :, lo:hi], base[1][b, :, lo:hi]), (b, lo, hi)
        assert torch.equal(dqkv[rows, H:], base[2][rows, H:]), (b, lo, hi)
        if one_block:
            assert torch.equal(dqkv[rows, :H], base[2][rows, :H]), (b, lo, hi)
        else:   # the same partials, added in another order
            err = (acc[rows].double() - base[3][rows].double()).abs()
            assert bool((err <= bound[rows]).all()), (b, lo, hi, float((err / bound[rows]).max()))
            err16 = (dqkv[rows, :H].double() - base[2][rows, :H].double()).abs()
            tol16 = bound[rows] + _bf16_step(base[2][rows, :H].double().abs() + bound[rows]).double()
            assert bool((err16 <= tol16).all()), (b, lo, hi)
        # dO only on the target: no gradient anywhere else
        d3 = torch.where(rows[:, None], dctx, torch.zeros_like(dctx))
        _, _, g, _ = run(qkv, d3, seg, S, nh, p)
        assert bool((g[~rows] == 0).all()), (b, lo, hi)


@pytest.mark.parametrize("S", [256, 512])
def test_malformed_segments_stay_inside_their_bin(cuda_dev, S):
    torch.manual_seed(S + 2)
    nh, p = 4, 0.1
    H = nh * 64
    good = seg_words([[(0, 50)], contiguous([128] * (S // 128))], S)
    bad = good.clone()
    bad[0, 60:70] = 60 | ((S + 300) << 16)          # ends past the bin
    bad[0, 100:110] = 105 | (20 << 16)              # lo > hi: sees nothing
    bad[0, 127] = 127 | ((S + 300) << 16)           # key block 0: its last key's segment ends past the bin
    bad[0, S - 128] = (S - 1) | ((S - 1) << 16)     # last key block: first key's segment starts after ...
    bad[0, S - 1] = 0 | (1 << 16)                   # ... its last key's ends
    qkv = torch.randn(2 * S, 3 * H, device=cuda_dev).to(bf)
    dctx = torch.randn(2 * S, H, device=cuda_dev).to(bf)
    ref = run(qkv, dctx, good.to(cuda_dev), S, nh, p)
    got = run(qkv, dctx, bad.to(cuda_dev), S, nh, p)
    nxt = slice(S, 2 * S)                           # bin 1: one-block segments, so its dQ has one partial per row
    assert torch.equal(got[0][nxt], ref[0][nxt])
    assert torch.equal(got[1][1], ref[1][1])
    assert torch.equal(got[2][nxt], ref[2][nxt])
    assert torch.equal(got[3][nxt], ref[3][nxt])
    for t in got:
        assert bool(torch.isfinite(t.float()).all())
