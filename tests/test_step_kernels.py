"""The embedding, head, loss, optimizer and bookkeeping kernels in the forms the training step calls them (GPU).

Edges, kernel by kernel:
  embed.cu     vocabulary 21128, H 256-1024, padded [32, 128] and packed bins (position ids, pos32); one hot id in
               more than 128 tokens spread over many 128-token scan blocks, ids seen once, id vocab-1, id 0 as the pad
               row and as an ordinary row; 1-4 token types (4: the filtered-colsum fallback); fp32 and bf16 dy; both
               word-row paths at their exact scratch boundary; the owner table re-armed after every call.
  head.cu      pooler groups of 8 rows with a ragged last group, packed cls rows (unsorted, the last row of the last
               bin); b2_head_bwd_split with fp32 / bf16 d_hidden on one stream and on a second stream; the mean
               cross-entropy beyond one 256-thread block's first sweep, with ignored labels and logits near +-80.
  optim.cu     the mean over 1-8 peer gradient buffers, shadow fan-out with NULL entries, slices,
               GradScaler scale / found_inf, a grid-stride loop that wraps; the background form on a ragged slice;
               the fp32 -> bf16 bias-gradient finish with the engine's segment table; the two casts.
  layernorm.cu the warp-pair backward at the engine's row counts (the operand ring and the row-sum exchange wrap),
               the forward on offset and constant rows, b2_colsum_finish.

References run in float64 on the GPU.  Where a kernel keeps a bf16 intermediate (pre_ln, pooled, scratch_dx) the
reference starts from it, so every bound is the rounding the kernel itself does: U = 2^-24 per fp32 operation,
times the length of the longest chain of fp32 additions behind a value, plus UB = 2^-8 (half a bf16 ulp) where the
result is stored as bf16.  Exact results are compared bitwise.  Each check asserts error <= bound element-wise.

Measured worst error / bound on an H100 80GB HBM3 (700 W), per check family: every bf16 store 0.95-0.996 (the
half-ulp rounding itself dominates: scratch_dx, d_word, d_pos, y, pooled, the head gradients, colsum_finish, the LN
column sums in bf16); d_type 0.85; LN fp32 dx 0.26 and fp32 accumulated column sums 0.05-0.22; LN mean / rstd
0.03 / 0.13; logits 0.025; cross-entropy loss 0.05; AdamW exp_avg / exp_avg_sq 0.37, master 0.88; the background
AdamW form matched the regular kernel bit for bit.  With B2_PARITY_REPORT set, every check appends its ratio there.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from parity import philox_keep_mask, report, tiny_config
from oracle import adamw_ref
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import _Layout
from pytorch_distributed_nlp_b200.packing import pack_batch

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
f64 = torch.float64
SEED, STEP = 1234, 5
U = 2.0 ** -24       # fp32 unit roundoff
UB = 2.0 ** -8       # bf16 unit roundoff (round to nearest even: half an ulp, relative)
INT_MAX = 2 ** 31 - 1
EPS = float(np.float32(1e-12))
SENT = -3.0          # sentinel fill: exactly representable in bf16 and fp32


def stream():
    return torch.cuda.current_stream().cuda_stream


def rng_state(dev, step=STEP):
    return torch.tensor([SEED, step], dtype=torch.int64, device=dev)


def rnd(shape, dev, scale=1.0, shift=0.0, gen=None):
    return (torch.randn(*shape, device=dev, generator=gen) * scale + shift).to(bf)


def drop_scale(p):
    """the kernels' 1/(1-p), computed in fp32"""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p))) if p > 0 else 1.0


def keep_mask(rows, H, site, p, dev, step=STEP):
    """fp64 [rows, H]: scale where the Philox stream keeps an element, 0 where it drops it"""
    k = torch.from_numpy(philox_keep_mask(rows * H, SEED, step, site, p).reshape(rows, H)).to(dev)
    return k.double() * drop_scale(p)


def within(got, ref, bound, what):
    """element-wise |got - ref| <= bound; the worst ratio goes to the parity report"""
    err = (got.double() - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    report("step_kernels", {"check": what, "err_over_bound": ratio})
    assert ratio <= 1.0, "%s: worst error is %.3g x its bound" % (what, ratio)


def bf_bound(ref, E):
    """bound for a bf16 store of an fp32 value within E of ref"""
    return UB * ref.abs() + (1 + UB) * E


# ---- float64 references -------------------------------------------------------------------------------------------
def ln_fwd_check(v, mean, rstd, y, g, b, what, keep=None, y_f32=None, stats_bound=None, ev=None, check=within):
    """v: the fp32 row values the kernel normalised (as fp64); mean / rstd / y: the kernel's outputs.
    Statistics against fp64 two-pass statistics; y against fp64 LayerNorm from the kernel's own statistics.
    stats_bound: (e_mu, e_rel) of a kernel whose statistics take another path (default: this file's one-warp row,
    H/32 + 6 deep chains, two-pass variance around the fp32 mean); ev: how far the kernel's own row values may lie
    from v (default: they are v); check: the within(got, ref, bound, what) that asserts and reports."""
    H = v.shape[1]
    mu64 = v.mean(1)
    var64 = ((v - mu64[:, None]) ** 2).mean(1)
    if stats_bound is None:
        depth = H / 32 + 6                  # per-lane sequential sum + 5 shuffle levels
        e_mu = depth * U * v.abs().mean(1)
        # two-pass variance around the fp32 mean: the mean's error enters squared; rsqrtf is within 2 ulp
        e_rel = depth * U + 4 * U + (e_mu ** 2) / (2 * (var64 + EPS))
    else:
        e_mu, e_rel = stats_bound
    check(mean, mu64, e_mu, what + " mean")
    rs64 = 1.0 / torch.sqrt(var64 + EPS)
    check(rstd, rs64, e_rel * rs64, what + " rstd")
    mu, rs = mean.double()[:, None], rstd.double()[:, None]
    ref = (v - mu) * rs * g.double() + b.double()
    E = 4 * U * (((v - mu) * rs * g.double()).abs() + b.double().abs())
    if ev is not None:
        E = E + ev * rs * g.double().abs()
    if keep is not None:
        ref, E = ref * keep, (E * keep + U * (ref * keep).abs())
    check(y, ref, bf_bound(ref, E), what + " y")
    if y_f32 is not None:
        check(y_f32, ref, E, what + " y_f32")


def ln_bwd_ref(dy, x, mean, rstd, g, ex_extra=0.0):
    """fp64 LayerNorm backward from the kernel's own fp32 statistics and bf16 input.  Returns dx, the bound of the
    kernel's fp32 dx, and xhat.  Row sums are chains of H/32 + 8 additions in either kernel form.
    ex_extra: a further bound on how far the kernel's xhat lies from (x - mean) * rstd, where x, mean and rstd are
    not exactly what the kernel reads."""
    H = x.shape[1]
    depth = H / 32 + 8
    dy, x, g = dy.double(), x.double(), g.double()
    mu, rs = mean.double()[:, None], rstd.double()[:, None]
    xh = (x - mu) * rs
    dxh = dy * g
    s1 = dxh.mean(1, keepdim=True)
    s2 = (dxh * xh).mean(1, keepdim=True)
    dx = rs * (dxh - s1 - xh * s2)
    ex = 2 * U * (x.abs() + mu.abs()) * rs + ex_extra          # the kernel's xhat
    e_s1 = depth * U * dxh.abs().mean(1, keepdim=True)
    e_s2 = depth * U * (dxh * xh).abs().mean(1, keepdim=True) + (dxh.abs() * ex).mean(1, keepdim=True)
    E = rs * (6 * U * (dxh.abs() + s1.abs() + (xh * s2).abs()) + e_s1 + (xh.abs() + ex) * e_s2 + ex * s2.abs())
    return dx, E, xh, ex


# ======================================================================================================================
# E. LayerNorm at the engine's row counts
# ======================================================================================================================
LN_ROWS = [1, 7, 4096, 4101, 16384]
LN_H = [256, 512, 768, 1024]


def ln_input(rows, H, dev, seed, constant_rows=True):
    gen = torch.Generator(device=dev).manual_seed(seed)
    x = rnd((rows, H), dev, 2.0, 0.3, gen)
    if rows > 1:
        x[1] = rnd((H,), dev, 0.05, 50.0, gen)                   # large common offset
    if constant_rows:
        x[0] = 3.0
        if rows > 2:
            x[2] = -1000.0
        if rows > 5:
            x[5] = rnd((H,), dev, 1e-3, -7.0, gen)               # bf16 spacing at 7 is 2^-5: (almost) constant
    return x


@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("H", LN_H)
def test_layernorm_fwd_engine_rows(cuda_dev, rows, H):
    dev = cuda_dev
    x = ln_input(rows, H, dev, 10 + rows + H)
    gen = torch.Generator(device=dev).manual_seed(H)
    g, b = rnd((H,), dev, 0.2, 1.0, gen), rnd((H,), dev, 0.1, 0.0, gen)
    y = torch.full((rows, H), float("nan"), dtype=bf, device=dev)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    L.call("b2_layernorm_fwd", x.data_ptr(), g.data_ptr(), b.data_ptr(), rows, H, EPS, y.data_ptr(), mean.data_ptr(),
           rstd.data_ptr(), stream())
    torch.cuda.synchronize()
    ln_fwd_check(x.double(), mean, rstd, y, g, b, "ln_fwd rows=%d H=%d" % (rows, H))
    const = [0] + ([2] if rows > 2 else [])
    for r in const:                  # exact mean of a constant row: x - mean == 0, the output is beta, bit for bit
        assert torch.equal(y[r], b), r


def ln_bwd_sums_check(acc, dy, xh, ex, dxd, rows, H, what, offset=0.0, bf_out=False):
    """the three column sums against fp64 sums (d_bias: of the kernel's own bf16 dx_drop)"""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    nb = min(nsm, (rows + 7) // 8)
    depth = -(-rows // (8 * nb)) + 8 + nb + 1 + (nb // 8 + 8 if bf_out else 0)
    dy = dy.double()
    terms = [(dy * xh, (dy.abs() * ex).sum(0) + 3 * U * (dy * xh).abs().sum(0)), (dy, 0.0),
             (dxd.double(), 0.0)]
    for k, (t, extra) in enumerate(terms):
        ref = t.sum(0) + offset
        E = depth * U * (t.abs().sum(0) + abs(offset)) + extra + U * ref.abs()
        within(acc[k], ref, bf_bound(ref, E) if bf_out else E, "%s sum %d" % (what, k))


@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("H", LN_H)
def test_layernorm_bwd_engine_rows(cuda_dev, rows, H):
    """b2_layernorm_bwd_accum (what the engine calls) and the grad_fp32 form of b2_layernorm_bwd: the same warp-pair
    kernel; from ~3 200 rows every warp pair walks several rows, so the cp.async ring and the two-parity row-sum
    exchange wrap"""
    dev = cuda_dev
    p, site = 0.1, 11
    x = ln_input(rows, H, dev, 20 + rows + H, constant_rows=False)
    gen = torch.Generator(device=dev).manual_seed(H + 1)
    g, b = rnd((H,), dev, 0.2, 1.0, gen), rnd((H,), dev, 0.1, 0.0, gen)
    y = torch.empty_like(x)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    L.call("b2_layernorm_fwd", x.data_ptr(), g.data_ptr(), b.data_ptr(), rows, H, EPS, y.data_ptr(), mean.data_ptr(),
           rstd.data_ptr(), stream())
    dy = torch.randn(rows, H, device=dev, generator=gen)
    rs = rng_state(dev)
    dx = torch.full((rows, H), float("nan"), device=dev)
    dxd = torch.full((rows, H), float("nan"), dtype=bf, device=dev)
    acc = torch.full((3, H), 0.5, device=dev)
    L.call("b2_layernorm_bwd_accum", dy.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), g.data_ptr(), rows,
           H, p, rs.data_ptr(), site, dx.data_ptr(), dxd.data_ptr(), acc.data_ptr(), stream())
    dx2, dxd2 = torch.empty_like(dx), torch.empty_like(dxd)
    outs = [torch.full((H,), SENT, dtype=bf, device=dev) for _ in range(3)]
    scratch = torch.empty(4 << 20, dtype=torch.uint8, device=dev)
    L.call("b2_layernorm_bwd", dy.data_ptr(), None, x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), g.data_ptr(), rows,
           H, p, rs.data_ptr(), site, 1, dx2.data_ptr(), dxd2.data_ptr(), *[o.data_ptr() for o in outs],
           scratch.data_ptr(), scratch.numel(), None, stream())
    torch.cuda.synchronize()
    assert torch.equal(dx, dx2) and torch.equal(dxd, dxd2)
    ref, E, xh, ex = ln_bwd_ref(dy, x, mean, rstd, g)
    what = "ln_bwd rows=%d H=%d" % (rows, H)
    within(dx, ref, E, what + " dx")
    keep = keep_mask(rows, H, site, p, dev) != 0
    # dx_drop is the kernel's own fp32 dx, masked and scaled in fp32, rounded once
    assert torch.equal(dxd, torch.where(keep, dx * drop_scale(p), torch.zeros_like(dx)).to(bf))
    ln_bwd_sums_check(acc, dy, xh, ex, dxd, rows, H, what + " accum", offset=0.5)
    ln_bwd_sums_check(torch.stack(outs), dy, xh, ex, dxd, rows, H, what + " bf16", bf_out=True)


@pytest.mark.parametrize("nsets,nparts,cols", [(1, 1, 37), (2, 7, 100), (3, 33, 1000), (3, 7, 33), (1, 33, 2304)])
def test_colsum_finish(cuda_dev, nsets, nparts, cols):
    dev = cuda_dev
    gen = torch.Generator(device=dev).manual_seed(nparts * cols)
    parts = torch.randn(nparts, nsets, cols, device=dev, generator=gen) * 3
    outs = [torch.full((cols + 8,), SENT, dtype=bf, device=dev) for _ in range(3)]
    null = 1 if nsets == 3 else None          # a NULL output: that set is skipped
    ptrs = [None if (k == null or k >= nsets) else outs[k].data_ptr() for k in range(3)]
    L.call("b2_colsum_finish", parts.data_ptr(), nparts, nsets, cols, *ptrs, stream())
    torch.cuda.synchronize()
    ref = parts.double().sum(0)
    E = (nparts + 9) * U * parts.double().abs().sum(0)
    for k in range(3):
        if k < nsets and k != null:
            within(outs[k][:cols], ref[k], bf_bound(ref[k], E[k]), "colsum_finish set %d" % k)
            assert (outs[k][cols:] == SENT).all()
        else:
            assert (outs[k] == SENT).all()


# ======================================================================================================================
# A. Embeddings
# ======================================================================================================================
VOCAB, MAX_POS, HOT = 21128, 512, 4242


def token_ids(n, gen):
    """ids mostly seen once, one hot id in > 128 tokens across many 128-token blocks, id vocab-1 twice, id 0 often"""
    ids = torch.randint(1, VOCAB, (n,), generator=gen)
    ids[torch.randperm(n, generator=gen)[: max(160, n // 12)]] = HOT
    ids[torch.randperm(n, generator=gen)[: n // 20]] = 0
    ids[n // 3] = ids[n - 2] = VOCAB - 1
    return ids


def embed_batch(packed, T, gen):
    """(input_ids, token_type_ids, position_ids or None, bins, seq) as host int64"""
    if not packed:
        B, S = 32, 128
        ids = token_ids(B * S, gen).view(B, S)
        tt = torch.randint(0, T, (B, S), generator=gen)
        return ids, tt, None, B, S
    # a length mix like the reference's rows (mean ~18) with a 1-token and a 128-token sequence
    lens = torch.cat([torch.randint(3, 34, (100,), generator=gen), torch.tensor([1, 128])])
    B = lens.numel()
    mask = (torch.arange(128)[None] < lens[:, None]).long()
    ids = token_ids(B * 128, gen).view(B, 128) * mask
    ids[0, 0] = ids[B - 1, 100] = VOCAB - 1
    tt = torch.randint(0, T, (B, 128), generator=gen) * mask
    pk = pack_batch(ids, tt, mask)
    return pk["input_ids"], pk["token_type_ids"], pk["position_ids"], pk["bins"], 128


def embed_fwd(tabs, ids, tt, pos_ids, B, S, H, T, p, dev):
    word, pos, typ, gam, bet = tabs
    M = B * S
    out = dict(y=torch.full((M, H), float("nan"), dtype=bf, device=dev),
               yf=torch.full((M, H), float("nan"), device=dev),
               pre=torch.full((M, H), float("nan"), dtype=bf, device=dev),
               mean=torch.empty(M, device=dev), rstd=torch.empty(M, device=dev),
               ids32=torch.full((M,), -7, dtype=torch.int32, device=dev),
               tt32=torch.full((M,), -7, dtype=torch.int32, device=dev),
               pos32=torch.full((M,), -7, dtype=torch.int32, device=dev))
    rs = rng_state(dev)
    o = out
    tail = (word.data_ptr(), pos.data_ptr(), typ.data_ptr(), gam.data_ptr(), bet.data_ptr(), H, VOCAB, T, EPS, p,
            rs.data_ptr(), 0, o["y"].data_ptr(), o["yf"].data_ptr(), o["pre"].data_ptr(), o["mean"].data_ptr(),
            o["rstd"].data_ptr(), o["ids32"].data_ptr(), o["tt32"].data_ptr())
    if pos_ids is None:
        L.call("b2_embed_fwd", ids.data_ptr(), tt.data_ptr(), B, S, *tail, stream())
    else:
        L.call("b2_embed_fwd_packed", ids.data_ptr(), tt.data_ptr(), pos_ids.data_ptr(), MAX_POS, B, S, *tail,
               o["pos32"].data_ptr(), stream())
    return out


def embed_bwd(fw, dy, dy32, gam, B, S, H, T, pad, p, scratch_bytes, owner, packed, dev):
    M = B * S
    g = dict(word=torch.full((VOCAB, H), SENT, dtype=bf, device=dev),
             pos=torch.full((MAX_POS, H), SENT, dtype=bf, device=dev),
             type=torch.full((T + 1, H), SENT, dtype=bf, device=dev),       # one row past the table: untouched
             gamma=torch.full((H,), SENT, dtype=bf, device=dev), beta=torch.full((H,), SENT, dtype=bf, device=dev),
             sdx=torch.full((M, H), float("nan"), dtype=bf, device=dev))
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
    rs = rng_state(dev)
    head = (dy.data_ptr(), 1 if dy32 else 0, fw["pre"].data_ptr(), fw["mean"].data_ptr(), fw["rstd"].data_ptr(),
            gam.data_ptr(), fw["ids32"].data_ptr(), fw["tt32"].data_ptr())
    tail = (B, S, H, VOCAB, T, pad, p, rs.data_ptr(), 0, g["word"].data_ptr(), g["pos"].data_ptr(),
            g["type"].data_ptr(), g["gamma"].data_ptr(), g["beta"].data_ptr(), g["sdx"].data_ptr(), scratch.data_ptr(),
            scratch_bytes, owner.data_ptr(), stream())
    if packed:
        L.call("b2_embed_bwd_packed", *head, fw["pos32"].data_ptr(), *tail)
    else:
        L.call("b2_embed_bwd", *head, *tail)
    torch.cuda.synchronize()
    return g


def index_sums(idx, vals, n):
    """fp64 sums of the rows of `vals` grouped by idx, their absolute sums and counts"""
    ref = torch.zeros(n, vals.shape[1], dtype=f64, device=vals.device).index_add_(0, idx, vals)
    mag = torch.zeros_like(ref).index_add_(0, idx, vals.abs())
    cnt = torch.bincount(idx, minlength=n).double()[:, None]
    return ref, mag, cnt


def check_embed_grads(g, fw, dy, keep, gam, S, H, T, pad, scratch_bytes, what, vocab=VOCAB, max_pos=MAX_POS,
                      unused=SENT, check=within):
    """stage 1: scratch_dx against fp64 LayerNorm backward (mask on the output); stage 2: the table gradients against
    fp64 sums of the kernel's own scratch_dx.  Rows outside the batch must hold `unused` (what was there before the
    backward); check: the within(got, ref, bound, what) that asserts and reports."""
    dev = dy.device
    M = dy.shape[0]
    dym = dy.double() * keep
    ref, E, xh, ex = ln_bwd_ref(dym, fw["pre"], fw["mean"], fw["rstd"], gam)
    check(g["sdx"], ref, bf_bound(ref, E), what + " scratch_dx")
    sdx = g["sdx"].double()
    ids, tt = fw["ids32"].long(), fw["tt32"].long()
    posi = fw["pos32"].long() if fw.get("packed") else torch.arange(M, device=dev) % S
    # word rows: one chain of additions per row (fp32 atomics in any order, or the owner's scan)
    valid = ids != pad
    uniq, inv = torch.unique(ids[valid], return_inverse=True)
    ref, mag, cnt = index_sums(inv, sdx[valid], uniq.numel())
    check(g["word"][uniq], ref, bf_bound(ref, cnt * U * mag), what + " d_word")
    untouched = torch.ones(vocab, dtype=torch.bool, device=dev)
    untouched[uniq] = False
    assert (g["word"][untouched] == unused).all(), what + ": a row outside the batch was written"
    if pad >= 0:
        assert (g["word"][pad] == unused).all(), what + ": the pad row was written"
    # position rows
    ref, mag, cnt = index_sums(posi, sdx, max_pos)
    check(g["pos"][:S], ref[:S], bf_bound(ref[:S], cnt[:S] * U * mag[:S]), what + " d_pos")
    assert (g["pos"][S:] == unused).all(), what + ": d_pos rows >= seq were written"
    # type rows: per-position chains then the partial reduction (fast path) or the filtered column sums (fallback)
    ref, mag, _ = index_sums(tt, sdx, T)
    depth = int(cnt.max()) + S + M // 8 + 48
    check(g["type"][:T], ref, bf_bound(ref, depth * U * mag), what + " d_type")
    if g["type"].shape[0] > T:
        assert (g["type"][T] == unused).all()
    # LayerNorm parameters (the generic backward's partial rows + colsum_finish)
    nb = min(296, scratch_bytes // (12 * H), (M + 7) // 8)
    depth = -(-M // (8 * nb)) + 8 + nb // 8 + 9
    t_g, t_b = dym * xh, dym
    ref = t_g.sum(0)
    E = (depth + 3) * U * t_g.abs().sum(0) + (dym.abs() * ex).sum(0)
    check(g["gamma"], ref, bf_bound(ref, E), what + " d_gamma")
    ref = t_b.sum(0)
    check(g["beta"], ref, bf_bound(ref, depth * U * t_b.abs().sum(0)), what + " d_beta")


EMBED_CASES = [  # H, packed, type_vocab, pad_token_id, p, fp32 dy
    (768, False, 2, 0, 0.1, True),        # config A as the engine runs it
    (256, False, 1, -1, 0.0, False),
    (512, True, 3, 0, 0.1, True),
    (1024, True, 2, -1, 0.0, True),
    (1024, False, 4, 0, 0.1, True),       # four token types: the filtered-colsum fallback
    (768, True, 1, 0, 0.0, False),
    (256, True, 2, -1, 0.1, False),
    (512, False, 3, -1, 0.0, True),
]


@pytest.mark.parametrize("H,packed,T,pad,p,dy32", EMBED_CASES)
def test_embed_fwd_bwd(cuda_dev, H, packed, T, pad, p, dy32):
    dev = cuda_dev
    gen = torch.Generator().manual_seed(H * 7 + T * 3 + int(packed))
    ids, tt, pos_ids, B, S = embed_batch(packed, T, gen)
    ids, tt = ids.to(dev), tt.to(dev)
    pos_ids = None if pos_ids is None else pos_ids.to(dev)
    M = B * S
    assert int((ids == HOT).sum()) > 128 and bool((ids == VOCAB - 1).any()) and bool((ids == 0).any())
    dgen = torch.Generator(device=dev).manual_seed(H)
    tabs = (rnd((VOCAB, H), dev, 0.5, 0, dgen), rnd((MAX_POS, H), dev, 0.5, 0, dgen), rnd((T, H), dev, 0.5, 0, dgen),
            rnd((H,), dev, 0.2, 1.0, dgen), rnd((H,), dev, 0.1, 0, dgen))
    word, pos, typ, gam, bet = tabs
    fw = embed_fwd(tabs, ids, tt, pos_ids, B, S, H, T, p, dev)
    fw["packed"] = packed
    torch.cuda.synchronize()
    what = "embed H=%d packed=%d T=%d" % (H, packed, T)
    # ids / types / positions are exact; pre_ln is bf16((word + pos) + type) summed in fp32
    posi = pos_ids.view(-1) if packed else torch.arange(M, device=dev) % S
    assert torch.equal(fw["ids32"].long(), ids.view(-1)) and torch.equal(fw["tt32"].long(), tt.view(-1))
    if packed:
        assert torch.equal(fw["pos32"].long(), posi)
    v = (word[ids.view(-1)].float() + pos[posi].float()) + typ[tt.view(-1)].float()
    assert torch.equal(fw["pre"], v.to(bf))
    keep = keep_mask(M, H, 0, p, dev) if p > 0 else None
    ln_fwd_check(v.double(), fw["mean"], fw["rstd"], fw["y"], gam, bet, what, keep=keep, y_f32=fw["yf"])
    assert torch.equal(fw["yf"].to(bf), fw["y"])

    dy = torch.randn(M, H, device=dev, generator=dgen)
    dy = dy if dy32 else dy.to(bf)
    keep = keep if keep is not None else torch.ones(M, H, dtype=f64, device=dev)
    owner = torch.empty(VOCAB, dtype=torch.int32, device=dev)
    L.call("b2_embed_owner_init", owner.data_ptr(), VOCAB, stream())
    fast = 4 * H * (M + S * T)        # exactly enough for the fp32 owner-row path
    g = embed_bwd(fw, dy, dy32, gam, B, S, H, T, pad, p, fast, owner, packed, dev)
    assert bool((owner == INT_MAX).all()), "owner table not re-armed"
    check_embed_grads(g, fw, dy, keep, gam, S, H, T, pad, fast, what + (" fast" if T <= 3 else " fallback"))
    if packed:
        with pytest.raises(RuntimeError, match="scratch too small"):
            embed_bwd(fw, dy, dy32, gam, B, S, H, T, pad, p, fast - 1, owner, packed, dev)
        return
    # one byte less: the owner-scan path, bit-reproducible from call to call
    g1 = embed_bwd(fw, dy, dy32, gam, B, S, H, T, pad, p, fast - 1, owner, packed, dev)
    assert bool((owner == INT_MAX).all()), "owner table not re-armed"
    check_embed_grads(g1, fw, dy, keep, gam, S, H, T, pad, fast - 1, what + " scan")
    g2 = embed_bwd(fw, dy, dy32, gam, B, S, H, T, pad, p, fast - 1, owner, packed, dev)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


# ======================================================================================================================
# B. Head and loss
# ======================================================================================================================
HEAD_FWD_CASES = [(1, 256, 1, 0.0), (5, 768, 2, 0.1), (13, 1024, 6, 0.0), (32, 768, 37, 0.1), (33, 1024, 6, 0.1),
                  (33, 256, 37, 0.0), (13, 256, 2, 0.1)]
HEAD_SITE = 1 + 3 * 12


def head_params(H, C, dev, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    return (rnd((H, H), dev, 0.03, 0, gen), rnd((H,), dev, 0.1, 0, gen), rnd((C, H), dev, 0.05, 0, gen),
            rnd((C,), dev, 0.1, 0, gen))


def packed_cls_rows():
    """pack_batch's cls rows for lengths whose first-fit layout puts a 1-token sequence on the last row of the last
    bin; in batch order the rows are unsorted"""
    lens = torch.tensor([50, 1, 64, 128, 27, 100, 50, 28, 64])
    mask = (torch.arange(128)[None] < lens[:, None]).long()
    pk = pack_batch(mask, None, mask)
    cls = pk["cls_index"]
    assert int(cls.max()) == pk["bins"] * 128 - 1 and not bool((cls[1:] >= cls[:-1]).all())
    return cls, pk["bins"] * 128


def head_fwd(hs, cls, B, S, H, params, C, p, dev):
    Wp, bp, Wc, bc = params
    rs = rng_state(dev)
    pooled = torch.full((B, H), float("nan"), dtype=bf, device=dev)
    logits = torch.full((B, C), float("nan"), device=dev)
    if cls is None:
        L.call("b2_head_fwd", hs.data_ptr(), B, S, H, Wp.data_ptr(), bp.data_ptr(), Wc.data_ptr(), bc.data_ptr(), C, p,
               rs.data_ptr(), HEAD_SITE, pooled.data_ptr(), logits.data_ptr(), stream())
    else:
        L.call("b2_head_fwd_packed", hs.data_ptr(), cls.data_ptr(), B, H, Wp.data_ptr(), bp.data_ptr(), Wc.data_ptr(),
               bc.data_ptr(), C, p, rs.data_ptr(), HEAD_SITE, pooled.data_ptr(), logits.data_ptr(), stream())
    torch.cuda.synchronize()
    return pooled, logits


def check_head_fwd(hs, rows, pooled, logits, params, p, what, keep=None, check=within):
    """pooled and logits of the sequence head from the kernel's own bf16 pooled; keep: the scaled fp64 [B, H] mask of
    the classifier dropout (None: this file's key at HEAD_SITE)"""
    Wp, bp, Wc, bc = (t.double() for t in params)
    B, H = pooled.shape
    h0 = hs[rows].double()
    depth = H / 32 + 6
    pre = h0 @ Wp.t() + bp
    ref = torch.tanh(pre)
    E = (1 - ref ** 2) * (depth * U * (h0.abs() @ Wp.abs().t() + bp.abs())) + 4 * U * ref.abs() + U
    check(pooled, ref, bf_bound(ref, E), what + " pooled")
    if keep is None and p > 0:
        keep = keep_mask(B, H, HEAD_SITE, p, hs.device)
    x = pooled.double() * keep if keep is not None else pooled.double()
    ref = x @ Wc.t() + bc
    E = (depth + 2) * U * (x.abs() @ Wc.abs().t() + bc.abs())
    check(logits, ref, E, what + " logits")


@pytest.mark.parametrize("B,H,C,p", HEAD_FWD_CASES)
def test_head_fwd(cuda_dev, B, H, C, p):
    dev = cuda_dev
    S = 128
    params = head_params(H, C, dev, B * H + C)
    hs = rnd((B * S, H), dev, 1.0, 0, torch.Generator(device=dev).manual_seed(B))
    pooled, logits = head_fwd(hs, None, B, S, H, params, C, p, dev)
    check_head_fwd(hs, torch.arange(B, device=dev) * S, pooled, logits, params, p, "head B=%d H=%d C=%d" % (B, H, C))


@pytest.mark.parametrize("H,C,p", [(768, 6, 0.1), (256, 37, 0.0)])
def test_head_fwd_packed(cuda_dev, H, C, p):
    dev = cuda_dev
    cls, tokens = packed_cls_rows()
    cls = cls.to(dev)
    B = cls.numel()
    params = head_params(H, C, dev, H + C)
    hs = rnd((tokens, H), dev, 1.0, 0, torch.Generator(device=dev).manual_seed(3))
    pooled, logits = head_fwd(hs, cls, B, 1, H, params, C, p, dev)
    check_head_fwd(hs, cls, pooled, logits, params, p, "head packed H=%d C=%d" % (H, C))


def head_bwd(dl, hs, pooled, cls, tokens, B, S, H, params, C, p, f32, side, dev):
    Wp, _, Wc, _ = params
    rs = rng_state(dev)
    grads = [torch.full((H, H), SENT, dtype=bf, device=dev), torch.full((H,), SENT, dtype=bf, device=dev),
             torch.full((C, H), SENT, dtype=bf, device=dev), torch.full((C,), SENT, dtype=bf, device=dev)]
    dh = torch.full((tokens, H), float("nan"), dtype=torch.float32 if f32 else bf, device=dev)
    scratch = torch.empty(2 * B, H, device=dev)
    L.call("b2_head_bwd_split", dl.data_ptr(), hs.data_ptr(), pooled.data_ptr(), L.ptr(cls), tokens, B, S, H,
           Wp.data_ptr(), Wc.data_ptr(), C, p, rs.data_ptr(), HEAD_SITE, *[t.data_ptr() for t in grads], dh.data_ptr(),
           1 if f32 else 0, scratch.data_ptr(), stream(), None if side is None else side.cuda_stream)
    torch.cuda.synchronize()
    return grads, dh


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("f32", [True, False])
def test_head_bwd_split(cuda_dev, packed, f32):
    dev = cuda_dev
    H, C, p = 768, 6, 0.1
    if packed:
        cls, tokens = packed_cls_rows()
        cls = cls.to(dev)
        B, S = cls.numel(), 1
        rows = cls
    else:
        B, S, cls = 33, 128, None
        tokens = B * S
        rows = torch.arange(B, device=dev) * S
    params = head_params(H, C, dev, 77)
    hs = rnd((tokens, H), dev, 1.0, 0, torch.Generator(device=dev).manual_seed(4))
    pooled, _ = head_fwd(hs, cls, B, S, H, params, C, p, dev)
    dl = torch.randn(B, C, device=dev, generator=torch.Generator(device=dev).manual_seed(5)) / B
    g1, dh1 = head_bwd(dl, hs, pooled, cls, tokens, B, S, H, params, C, p, f32, None, dev)
    side = torch.cuda.Stream(dev)
    g2, dh2 = head_bwd(dl, hs, pooled, cls, tokens, B, S, H, params, C, p, f32, side, dev)
    for a, b in zip(g1 + [dh1], g2 + [dh2]):
        assert torch.equal(a, b), "the weight-gradient stream changed a result"
    what = "head_bwd packed=%d f32=%d" % (packed, f32)
    check_head_bwd(dl, hs, rows, pooled, params, g1, dh1, f32, keep_mask(B, H, HEAD_SITE, p, dev), what)
    if not packed:
        with pytest.raises(RuntimeError, match="tokens / seq mismatch"):
            head_bwd(dl, hs, pooled, None, tokens - 1, B, S, H, params, C, p, f32, None, dev)


def check_head_bwd(dl, hs, rows, pooled, params, grads, dh, f32, m, what, check=within):
    """the four head parameter gradients and d_hidden (rows: the cls rows; every other row must be 0), in fp64 from
    the kernel's own pooled (the same statements autograd runs); m: the scaled fp64 [B, H] keep mask"""
    B, C, H = dl.shape[0], dl.shape[1], pooled.shape[1]
    other = torch.ones(dh.shape[0], dtype=torch.bool, device=dh.device)
    other[rows] = False
    assert bool((dh[other] == 0).all()), what + ": non-CLS rows of d_hidden are not zero"
    Wp, _, Wc, _ = (t.double() for t in params)
    P = pooled.double()
    h0, dl64 = hs[rows].double(), dl.double()
    dpd, apd = dl64 @ Wc, dl64.abs() @ Wc.abs()
    d_pre = dpd * m * (1 - P ** 2)
    e_pre = apd * m * ((C + 3) * U * (1 - P ** 2).abs() + 2 * U * (1 + P ** 2))
    a_pre = apd * m * (1 - P ** 2).abs()
    pm = P * m
    refs = [(d_pre.t() @ h0, (B + 2) * U * (a_pre.t() @ h0.abs()) + e_pre.t() @ h0.abs()),
            (d_pre.sum(0), B * U * a_pre.sum(0) + e_pre.sum(0)),
            (dl64.t() @ pm, (B + 2) * U * (dl64.abs().t() @ pm.abs())),
            (dl64.sum(0), B * U * dl64.abs().sum(0))]
    for k, (ref, E) in enumerate(refs):
        check(grads[k], ref, bf_bound(ref, E), "%s grad %d" % (what, k))
    ref = d_pre @ Wp
    E = (H / 8 + 9) * U * (a_pre @ Wp.abs()) + e_pre @ Wp.abs()
    check(dh[rows], ref, E if f32 else bf_bound(ref, E), what + " d_hidden")


@pytest.mark.parametrize("B,C", [(1, 1), (1, 100), (300, 7), (1000, 100), (1000, 2)])
@pytest.mark.parametrize("with_grad", [True, False])
def test_ce_fwd_bwd(cuda_dev, B, C, with_grad):
    """never a label outside [0, C) other than -100: the kernel traps on one by design"""
    dev = cuda_dev
    gen = torch.Generator(device=dev).manual_seed(B * C)
    z = (torch.rand(B, C, device=dev, generator=gen) * 2 - 1) * 80
    labels = torch.randint(0, C, (B,), device=dev, generator=gen)
    if B > 1:
        labels[torch.rand(B, device=dev, generator=gen) < 0.2] = -100
    loss = torch.full((), float("nan"), device=dev)
    dlog = torch.full((B, C), float("nan"), device=dev) if with_grad else None
    L.call("b2_ce_fwd_bwd", z.data_ptr(), labels.data_ptr(), B, C, loss.data_ptr(), L.ptr(dlog), stream())
    torch.cuda.synchronize()
    check_ce(z, labels, loss, dlog, "ce B=%d C=%d" % (B, C))


def check_ce(z, labels, loss, dlog, what, check=within):
    """the mean cross-entropy and (dlog not None) its logits gradient against float64 from the kernel's logits"""
    B, C = z.shape
    zz = z.double().requires_grad_(True)
    ref = F.cross_entropy(zz, labels)
    ref.backward()
    valid = labels != -100
    n = int(valid.sum())
    z64 = z.double()
    lse = torch.logsumexp(z64, 1)
    zy = z64.gather(1, labels.clamp_min(0)[:, None])[:, 0]
    # per sample: C expf (2 ulp) of exactly-rounded differences, the sum, logf
    e_lse = (C + 3) * U + U * (z64 - z64.max(1).values[:, None]).abs().max(1).values + 2 * U * lse.abs()
    lb = (lse - zy)
    e_loss = ((e_lse + U * zy.abs() + U * lb.abs())[valid].sum() + (-(-B // 256) + 9) * U * lb[valid].abs().sum()) / n
    check(loss.view(1), ref.detach().view(1), (e_loss + 2 * U * ref.detach().abs()).view(1), what + " loss")
    if dlog is not None:
        sm = torch.softmax(z64, 1)
        # expf underflows below 2^-126 (gradual, to 2^-149): an absolute floor of 2^-126 / n
        E = (sm * (U * (z64 - lse[:, None]).abs() + e_lse[:, None] + 2 * U) + 2.0 ** -126) / n + 4 * U * zz.grad.abs()
        check(dlog, zz.grad, E, what + " dlogits")
        assert bool((dlog[~valid] == 0).all()), what + ": ignored rows have a nonzero gradient"


# ======================================================================================================================
# C. Optimizer
# ======================================================================================================================
def hparams(lr=1e-2, wd=0.01, correct_bias=1, scale=None, found_inf=None):
    hp = L.AdamWHParams()
    hp.lr, hp.beta1, hp.beta2, hp.eps, hp.weight_decay, hp.correct_bias = lr, 0.9, 0.999, 1e-6, wd, correct_bias
    hp.grad_scale, hp.found_inf = L.ptr(scale), L.ptr(found_inf)
    return hp


class ReduceRun:
    """`world` local bf16 gradient buffers stand in for the peers (the kernel only sees pointers).  Shadow buffers of
    odd ranks other than `rank` are passed as NULL and must keep their sentinel."""

    def __init__(self, dev, world, n, seed=0):
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.dev, self.world, self.n, self.gen, self.rank = dev, world, n, gen, world - 1
        self.master = torch.randn(n, device=dev, generator=gen)
        self.m, self.v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
        self.decay = (torch.rand(n // 8, device=dev, generator=gen) < 0.5).to(torch.uint8)
        self.shadow = [torch.full((n,), SENT, dtype=bf, device=dev) for _ in range(world)]
        self.null = [r % 2 == 1 and r != self.rank for r in range(world)]
        self.step = torch.zeros(1, dtype=torch.int64, device=dev)
        self.rng = rng_state(dev, 0)

    def grads(self, mult=1.0):
        return [(torch.randn(self.n, device=self.dev, generator=self.gen) * 1e-2 * (1 + r) * mult).to(bf)
                for r in range(self.world)]

    def state(self):
        return [t.clone() for t in [self.master, self.m, self.v] + self.shadow]

    def call(self, grads, hp, begin=0, end=None, found_inf=None):
        end = self.n if end is None else end
        sh = [None if self.null[r] else self.shadow[r].data_ptr() for r in range(self.world)]
        L.call("b2_bucket_reduce_adamw", L.ptr_array([g.data_ptr() for g in grads]), L.ptr_array(sh), self.world,
               self.rank, self.master.data_ptr(),
               self.m.data_ptr(), self.v.data_ptr(), self.decay.data_ptr(), begin, end, hp, self.step.data_ptr(),
               stream())
        L.call("b2_step_advance", self.step.data_ptr(), self.rng.data_ptr(), L.ptr(found_inf), stream())


class AdamWRef:
    """oracle.adamw_ref.HFAdamW in float64 on the selected elements, plus a first-order bound of the kernel's fp32
    rounding carried along: the mean of `world` bf16 values (world additions, the (1/scale)/world product), two
    roundings per moment statement, and the update's own roundings plus what the moments' errors make of it."""

    def __init__(self, master, decay_el, sel, lr, wd, correct_bias, world, extra=0):
        self.sel = sel
        self.dec = decay_el[sel]
        w = master.double()[sel]
        self.p = {"x.weight": w[self.dec].clone(), "x.bias": w[~self.dec].clone()}
        self.opt = adamw_ref.HFAdamW(self.p, lr=lr, weight_decay=wd, correct_bias=bool(correct_bias))
        self.lr, self.wd, self.cg = lr, wd, (world + 3 + extra) * U
        z = torch.zeros_like(w)
        self.em, self.ev, self.ew = z.clone(), z.clone(), z.clone()

    def gather(self, name):
        out = torch.empty(self.dec.numel(), dtype=f64, device=self.dec.device)
        st = lambda k: self.opt.state[k][name] if name != "w" else self.p[k]
        out[self.dec], out[~self.dec] = st("x.weight"), st("x.bias")
        return out

    def step(self, g):
        g = g[self.sel]
        b1, b2 = self.opt.betas
        m0, v0, w0 = self.gather("exp_avg"), self.gather("exp_avg_sq"), self.gather("w")
        self.opt.step({"x.weight": g[self.dec], "x.bias": g[~self.dec]})
        m, v, w = self.gather("exp_avg"), self.gather("exp_avg_sq"), self.gather("w")
        t = self.opt.state["x.weight"]["step"]
        ss = self.lr * (math.sqrt(1 - b2 ** t) / (1 - b1 ** t) if self.opt.correct_bias else 1.0)
        self.em = b1 * self.em + 2 * U * (b1 * m0.abs() + (1 - b1) * g.abs()) + (1 - b1) * g.abs() * self.cg
        self.ev = b2 * self.ev + 3 * U * (b2 * v0 + (1 - b2) * g * g) + (1 - b2) * g * g * 2 * self.cg
        den = v.sqrt() + 1e-6
        upd = ss * m / den
        e_upd = 6 * U * upd.abs() + ss * self.em / den + upd.abs() * self.ev / (2 * v.clamp_min(1e-300)) * (v > 0)
        self.ew = self.ew * (1 + self.lr * self.wd) + U * w0.abs() + e_upd + 2 * U * w.abs() * self.dec
        return m, v, w


def check_reduce(run, ref, sel, what):
    m, v, w = ref.gather("exp_avg"), ref.gather("exp_avg_sq"), ref.gather("w")
    within(run.m[sel], m, ref.em, what + " exp_avg")
    within(run.v[sel], v, ref.ev, what + " exp_avg_sq")
    within(run.master[sel], w, ref.ew, what + " master")
    for r in range(run.world):
        if run.null[r]:
            assert bool((run.shadow[r] == SENT).all()), "%s: NULL shadow %d" % (what, r)
        else:
            assert torch.equal(run.shadow[r][sel], run.master[sel].to(bf)), "%s: shadow %d" % (what, r)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_reduce_adamw_world(cuda_dev, world):
    """the mean over `world` peer buffers feeding HF AdamW, three steps, decay and no-decay vectors"""
    dev = cuda_dev
    n = 8 * 9001
    run = ReduceRun(dev, world, n, seed=world)
    sel = torch.arange(n, device=dev)
    ref = AdamWRef(run.master, run.decay.bool().repeat_interleave(8), sel, 1e-2, 0.01, 1, world)
    for _ in range(3):
        grads = run.grads()
        run.call(grads, hparams())
        ref.step(sum(g.double() for g in grads) / world)
    torch.cuda.synchronize()
    assert int(run.step.item()) == 3 and int(run.rng[1].item()) == 3
    check_reduce(run, ref, sel, "reduce world=%d" % world)


REDUCE_EDGES = ["wrap", "slice", "no_bias_correction", "no_weight_decay", "scale_1000"]


@pytest.mark.parametrize("case", REDUCE_EDGES)
def test_reduce_adamw_edges(cuda_dev, case):
    dev = cuda_dev
    world = {"wrap": 2, "slice": 3, "no_bias_correction": 4, "no_weight_decay": 1, "scale_1000": 3}[case]
    # "wrap": more vectors than the capped grid (132 x 8 blocks of 256 threads) covers in one sweep, ragged tail
    n = (3 << 20) + 8 * 13 if case == "wrap" else 8 * 20011
    run = ReduceRun(dev, world, n, seed=len(case))
    begin, end = (8 * 1001, n - 8 * 77) if case == "slice" else (0, n)
    lr, wd, cb = 1e-2, (0.0 if case == "no_weight_decay" else 0.01), (0 if case == "no_bias_correction" else 1)
    if case == "no_weight_decay":
        run.decay.fill_(1)
    scale = torch.tensor([1000.0], device=dev) if case == "scale_1000" else None
    vec = torch.zeros(n // 8, dtype=torch.bool, device=dev)
    vec[begin // 8: end // 8] = True
    sel_mask = vec.repeat_interleave(8)
    sel = sel_mask.nonzero()[:, 0]
    before = run.state()
    ref = AdamWRef(run.master, run.decay.bool().repeat_interleave(8), sel, lr, wd, cb, world,
                   extra=2 if scale is not None else 0)
    for _ in range(3):
        grads = run.grads(1000.0 if scale is not None else 1.0)
        run.call(grads, hparams(lr, wd, cb, scale=scale), begin, end)
        g = sum(x.double() for x in grads) / world
        ref.step(g / 1000.0 if scale is not None else g)
    torch.cuda.synchronize()
    check_reduce(run, ref, sel, "reduce " + case)
    for a, b in zip(before, run.state()):         # everything outside the slice: bit for bit
        assert torch.equal(a[~sel_mask], b[~sel_mask]), case


def test_reduce_adamw_grad_scale_pow2_and_found_inf(cuda_dev):
    """a power-of-two GradScaler scale unscales exactly: bitwise the unscaled update; found_inf != 0 leaves master,
    moments and every shadow bitwise unchanged, and b2_step_advance keeps the step count but advances dropout"""
    dev = cuda_dev
    n, world = 8 * 5003, 3
    a, b = ReduceRun(dev, world, n, seed=9), ReduceRun(dev, world, n, seed=9)
    scale = torch.tensor([65536.0], device=dev)
    for _ in range(2):
        grads = a.grads()
        a.call(grads, hparams())
        b.call([(g.float() * 65536.0).to(bf) for g in grads], hparams(scale=scale), found_inf=None)
    torch.cuda.synchronize()
    for x, y in zip(a.state(), b.state()):
        assert torch.equal(x, y)
    inf = torch.tensor([1.0], device=dev)
    before = b.state()
    b.call([(g.float() * 65536.0).to(bf) for g in b.grads()], hparams(scale=scale, found_inf=inf), found_inf=inf)
    torch.cuda.synchronize()
    for x, y in zip(before, b.state()):
        assert torch.equal(x, y)
    assert int(b.step.item()) == 2 and int(b.rng[1].item()) == 3


def test_adamw_background_ragged_slice(cuda_dev):
    """b2_adamw_background on a slice that starts past 0 and is not a whole number of 4096-element blocks agrees
    with b2_bucket_reduce_adamw at world 1 to an ulp (the compiler may contract a different product into an FMA);
    outside the slice nothing changes"""
    dev = cuda_dev
    n = 8 * 7000
    begin, end = 8 * 123, 8 * 123 + 3 * 4096 + 8 * 5
    a, b = ReduceRun(dev, 1, n, seed=11), ReduceRun(dev, 1, n, seed=11)
    hp = hparams()
    step_size = torch.zeros(1, device=dev)
    before = a.state()
    for _ in range(3):
        g = a.grads()
        L.call("b2_adamw_prepare", hp, a.step.data_ptr(), step_size.data_ptr(), stream())
        L.call("b2_adamw_background", g[0].data_ptr(), a.shadow[0].data_ptr(), a.master.data_ptr(), a.m.data_ptr(),
               a.v.data_ptr(), a.decay.data_ptr(), begin, end, hp, step_size.data_ptr(), stream())
        L.call("b2_step_advance", a.step.data_ptr(), a.rng.data_ptr(), None, stream())
        b.call(g, hp, begin, end)
    torch.cuda.synchronize()
    for x, y in zip(a.state()[:3], b.state()[:3]):
        ulp = torch.maximum(x.abs(), y.abs()) * 2.0 ** -23
        within(x[begin:end], y[begin:end].double(), 2 * ulp[begin:end].double(), "adamw background vs reduce")
    assert (a.shadow[0][begin:end].float() - b.shadow[0][begin:end].float()).abs().le(
        a.master[begin:end].abs() * 2.0 ** -7).all()
    for x, y in zip(before, a.state()):
        assert torch.equal(torch.cat([x[:begin], x[end:]]), torch.cat([y[:begin], y[end:]]))


# ======================================================================================================================
# D. Bookkeeping
# ======================================================================================================================
def test_accum_finish_engine_segments(cuda_dev):
    """the engine's per-layer segment table ([3H qkv | I | 3H output-LN sets | 3H attention-output-LN sets] of the fp32
    accumulators -> bias / LayerNorm gradients in the flat bf16 space) for 2 layers at H = 768, called per layer as
    the engine does: all eight segments at seq 128, the seven without QKV otherwise"""
    dev = cuda_dev
    cfg = tiny_config(hidden_size=768, intermediate_size=3072, num_attention_heads=12)
    lay = _Layout(cfg)
    H, I, nl = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
    per = 9 * H + I
    segs = []
    for l in range(nl):
        pre = "bert.encoder.layer.%d." % l
        b2_ = l * per + 3 * H + I
        b1_ = b2_ + 3 * H
        segs += [[l * per, lay.off(pre + "attention.self.query.bias"), 3 * H],
                 [l * per + 3 * H, lay.off(pre + "intermediate.dense.bias"), I],
                 [b2_, lay.off(pre + "output.LayerNorm.weight"), H], [b2_ + H, lay.off(pre + "output.LayerNorm.bias"), H],
                 [b2_ + 2 * H, lay.off(pre + "output.dense.bias"), H],
                 [b1_, lay.off(pre + "attention.output.LayerNorm.weight"), H],
                 [b1_ + H, lay.off(pre + "attention.output.LayerNorm.bias"), H],
                 [b1_ + 2 * H, lay.off(pre + "attention.output.dense.bias"), H]]
    seg_t = torch.tensor(segs, dtype=torch.int64, device=dev)
    src = torch.randn(nl * per, device=dev, generator=torch.Generator(device=dev).manual_seed(1)) * 10
    src[::97] = 0.0
    src[1::89] = float(2.0 ** -130)           # fp32 subnormals
    dst = torch.full((lay.total,), SENT, dtype=bf, device=dev)
    src0, dst0 = src.clone(), dst.clone()
    for l, seq in ((0, 128), (1, 64)):
        s0 = 8 * l if seq == 128 else 8 * l + 1
        L.call("b2_accum_finish", src.data_ptr(), dst.data_ptr(), seg_t.data_ptr() + 24 * s0, 8 * (l + 1) - s0,
               max(3 * H, I), stream())
    torch.cuda.synchronize()
    in_src = torch.zeros(nl * per, dtype=torch.bool, device=dev)
    in_dst = torch.zeros(lay.total, dtype=torch.bool, device=dev)
    for k, (so, do, cnt) in enumerate(segs):
        if k == 8:                                 # layer 1's QKV segment was not part of its call
            continue
        in_src[so:so + cnt] = True
        in_dst[do:do + cnt] = True
        assert torch.equal(dst[do:do + cnt], src0[so:so + cnt].to(bf)), k
    assert bool((src[in_src] == 0).all()), "accumulators not re-armed"
    assert torch.equal(src[~in_src], src0[~in_src]) and torch.equal(dst[~in_dst], dst0[~in_dst])


def special_f32(n, dev):
    """n fp32 values with +-inf, nan, -0, subnormals, exact bf16 round-to-nearest-even ties, largest finite"""
    gen = torch.Generator(device=dev).manual_seed(n)
    x = torch.randn(n, device=dev, generator=gen) * 100
    bits = np.array([0x7F800000, 0xFF800000, 0x7FC00000, 0x80000000, 0x00000001, 0x807FFFFF, 0x3F808000,
                     0x3F818000, 0xBF808000, 0x7F7FFFFF, 0x00408000, 0x3F80FFFF], dtype=np.uint32)
    sp = torch.from_numpy(bits.view(np.float32)).to(dev)
    k = min(n, sp.numel())
    pos = torch.randperm(n, device=dev, generator=gen)[:k]
    x[pos] = sp[:k]
    if n > 0:
        x[-1] = sp[(n * 7) % sp.numel()]           # the last element goes through the scalar tail
    return x


@pytest.mark.parametrize("n", [1, 7, 8, 9, 4097, (1 << 20) + 3])
def test_casts(cuda_dev, n):
    """b2_cast_f32_to_bf16 / b2_cast_bf16_to_f32 bitwise against torch's casts (nan compared as nan); nothing past
    n is written"""
    dev = cuda_dev
    x = torch.zeros(n + 16, device=dev)
    x[:n] = special_f32(n, dev)
    out = torch.full((n + 16,), SENT, dtype=bf, device=dev)
    L.call("b2_cast_f32_to_bf16", x.data_ptr(), out.data_ptr(), n, stream())
    back = torch.full((n + 16,), SENT, device=dev)
    L.call("b2_cast_bf16_to_f32", out.data_ptr(), back.data_ptr(), n, stream())
    torch.cuda.synchronize()
    ref = x[:n].to(bf)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(out[:n]), nan)
    assert torch.equal(out[:n][~nan].view(torch.int16), ref[~nan].view(torch.int16))
    assert bool((out[n:] == SENT).all()) and bool((back[n:] == SENT).all())
    ref2 = out[:n].float()
    assert torch.equal(torch.isnan(back[:n]), torch.isnan(ref2))
    assert torch.equal(back[:n][~nan].view(torch.int32), ref2[~nan].view(torch.int32))
