"""Per-kernel parity through the C ABI against fp32 torch restatements of the same op (GPU)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from parity import attention_ref, attn_keep_mask, b2, padded_visibility, philox_keep_mask, rel_l2
from pytorch_distributed_nlp_b200 import _lib as L

pytestmark = pytest.mark.gpu
bf = torch.bfloat16


def S():
    return torch.cuda.current_stream().cuda_stream


def rnd(shape, dev, scale=1.0, shift=0.0):
    return (torch.randn(*shape, device=dev) * scale + shift).to(bf)


def rng_state(dev, seed=1234, step=5):
    return torch.tensor([seed, step], dtype=torch.int64, device=dev)


@pytest.mark.parametrize("H", [256, 768, 1024])
def test_layernorm_fwd_bwd(cuda_dev, H):
    dev = cuda_dev
    rows = 1000
    torch.manual_seed(0)
    x, g, b = rnd((rows, H), dev, 2.0, 0.3), rnd((H,), dev, 0.2, 1.0), rnd((H,), dev, 0.1)
    y = torch.empty_like(x)
    mean = torch.empty(rows, dtype=torch.float32, device=dev)
    rstd = torch.empty_like(mean)
    L.call("b2_layernorm_fwd", x.data_ptr(), g.data_ptr(), b.data_ptr(), rows, H, 1e-12, y.data_ptr(),
           mean.data_ptr(), rstd.data_ptr(), S())
    xr = x.float().requires_grad_(True)
    gr, br = g.float().requires_grad_(True), b.float().requires_grad_(True)
    yr = F.layer_norm(xr, (H,), gr, br, 1e-12)
    assert (y.float() - yr).abs().max().item() < 3e-2
    assert (mean - xr.mean(-1)).abs().max().item() < 1e-4

    dy = rnd((rows, H), dev)
    for p in (0.0, 0.1):
        dx, dxd = torch.empty_like(x), torch.empty_like(x)
        dg, db, dbias = (torch.empty(H, dtype=bf, device=dev) for _ in range(3))
        scratch = torch.empty(4 << 20, dtype=torch.uint8, device=dev)
        rs = rng_state(dev)
        L.call("b2_layernorm_bwd", dy.data_ptr(), None, x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), g.data_ptr(),
               rows, H, p, rs.data_ptr(), 11, 0, dx.data_ptr(), dxd.data_ptr(), dg.data_ptr(), db.data_ptr(),
               dbias.data_ptr(), scratch.data_ptr(), scratch.numel(), None, S())
        # fp32 gradient stream variant: fp32 dy in, fp32 dx out, bf16 dx_drop always written
        dy32, dx32, dxd32 = dy.float(), torch.empty(rows, H, device=dev), torch.empty_like(x)
        dg2, db2, dbias2 = (torch.empty(H, dtype=bf, device=dev) for _ in range(3))
        L.call("b2_layernorm_bwd", dy32.data_ptr(), None, x.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
               g.data_ptr(), rows, H, p, rs.data_ptr(), 11, 1, dx32.data_ptr(), dxd32.data_ptr(), dg2.data_ptr(),
               db2.data_ptr(), dbias2.data_ptr(), scratch.data_ptr(), scratch.numel(), None, S())
        # accumulate form (what the engine calls): same dx / dx_drop, column sums ADDED into fp32 [3][H]
        acc = torch.full((3, H), 0.5, dtype=torch.float32, device=dev)
        dx_a, dxd_a = torch.empty(rows, H, device=dev), torch.empty_like(x)
        L.call("b2_layernorm_bwd_accum", dy32.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
               g.data_ptr(), rows, H, p, rs.data_ptr(), 11, dx_a.data_ptr(), dxd_a.data_ptr(), acc.data_ptr(), S())
        torch.cuda.synchronize()
        assert torch.equal(dx_a, dx32) and torch.equal(dxd_a, dxd32)
        for k, ref in enumerate((dg2, db2, dbias2)):
            got = acc[k] - 0.5
            assert float((got - ref.float()).abs().max()) <= 1e-2 * float(ref.float().abs().max()) + 1e-3, k
        # deferred finish: partials only, then the reduction as a separate call
        import ctypes
        npart = ctypes.c_int32(0)
        dg3, db3, dbias3 = (torch.zeros(H, dtype=bf, device=dev) for _ in range(3))
        scratch3 = torch.empty(4 << 20, dtype=torch.uint8, device=dev)
        L.call("b2_layernorm_bwd", dy32.data_ptr(), None, x.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
               g.data_ptr(), rows, H, p, rs.data_ptr(), 11, 1, dx32.data_ptr(), dxd32.data_ptr(), dg3.data_ptr(),
               db3.data_ptr(), dbias3.data_ptr(), scratch3.data_ptr(), scratch3.numel(), ctypes.byref(npart), S())
        assert npart.value > 0 and float(dg3.float().abs().max()) == 0.0
        L.call("b2_colsum_finish", scratch3.data_ptr(), npart.value, 3, H, dg3.data_ptr(), db3.data_ptr(),
               dbias3.data_ptr(), S())
        torch.cuda.synchronize()
        assert torch.equal(dg3, dg2) and torch.equal(db3, db2) and torch.equal(dbias3, dbias2)
        torch.cuda.synchronize()
        assert rel_l2(dx32, dx.float()) < 5e-3 and rel_l2(dg2.float(), dg.float()) < 1e-2
        if p > 0:
            # same mask (identical zero pattern); values agree to bf16 rounding (the two kernels order the fp32
            # arithmetic differently)
            assert torch.equal(dxd32 == 0, dxd == 0)
            assert rel_l2(dxd32.float(), dxd.float()) < 5e-3
        else:
            assert torch.equal(dxd32, dx32.to(bf))
        for t in (xr, gr, br):
            t.grad = None
        yr = F.layer_norm(xr, (H,), gr, br, 1e-12)
        yr.backward(dy.float())
        assert rel_l2(dx.float(), xr.grad) < 1e-2
        assert rel_l2(dg.float(), gr.grad) < 1e-2
        assert rel_l2(db.float(), br.grad) < 1e-2
        ref_drop = xr.grad
        if p > 0:
            keep = torch.from_numpy(philox_keep_mask(rows * H, 1234, 5, 11, p).reshape(rows, H)).to(dev)
            ref_drop = xr.grad * keep / (1 - p)
            assert rel_l2(dxd.float(), ref_drop) < 1e-2
        assert rel_l2(dbias.float(), ref_drop.sum(0)) < 1e-2


def test_colsum(cuda_dev):
    dev = cuda_dev
    x = rnd((4096, 2304), dev)
    out = torch.empty(2304, dtype=bf, device=dev)
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    L.call("b2_colsum", x.data_ptr(), 4096, 2304, 2304, out.data_ptr(), scratch.data_ptr(), scratch.numel(), S())
    assert rel_l2(out.float(), x.float().sum(0)) < 1e-2
    with pytest.raises(RuntimeError, match="empty"):
        L.call("b2_colsum", x.data_ptr(), 0, 2304, 2304, out.data_ptr(), scratch.data_ptr(), scratch.numel(), S())


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_embed_fwd_bwd(cuda_dev, p):
    dev = cuda_dev
    B, Sq, H, V, T = 8, 128, 768, 2000, 2
    torch.manual_seed(1)
    word, pos, typ = rnd((V, H), dev, 0.5), rnd((512, H), dev, 0.5), rnd((T, H), dev, 0.5)
    gam, bet = rnd((H,), dev, 0.2, 1.0), rnd((H,), dev, 0.1)
    ids = torch.randint(0, V, (B, Sq), device=dev)
    ids[:, 40:] = ids[:, 40:] % 7          # heavy duplication + pad id 0
    tt = torch.randint(0, T, (B, Sq), device=dev)
    rs = rng_state(dev)
    M = B * Sq
    y, pre = torch.empty(M, H, dtype=bf, device=dev), torch.empty(M, H, dtype=bf, device=dev)
    yf = torch.empty(M, H, dtype=torch.float32, device=dev)
    mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
    ids32, tt32 = torch.empty(M, dtype=torch.int32, device=dev), torch.empty(M, dtype=torch.int32, device=dev)
    L.call("b2_embed_fwd", ids.data_ptr(), tt.data_ptr(), B, Sq, word.data_ptr(), pos.data_ptr(), typ.data_ptr(),
           gam.data_ptr(), bet.data_ptr(), H, V, T, 1e-12, p, rs.data_ptr(), 0, y.data_ptr(), yf.data_ptr(),
           pre.data_ptr(), mean.data_ptr(), rstd.data_ptr(), ids32.data_ptr(), tt32.data_ptr(), S())
    assert torch.equal(yf.to(bf), y)          # the fp32 copy (first residual of the fp32 stream) rounds to the bf16 output
    wr, pr, tr = (t.float().requires_grad_(True) for t in (word, pos, typ))
    gr, br = gam.float().requires_grad_(True), bet.float().requires_grad_(True)
    e = F.embedding(ids, wr, padding_idx=0) + pr[:Sq][None] + tr[tt]
    yr = F.layer_norm(e, (H,), gr, br, 1e-12)
    keep = None
    if p > 0:
        keep = torch.from_numpy(philox_keep_mask(M * H, 1234, 5, 0, p).reshape(B, Sq, H)).to(dev)
        yr = yr * keep / (1 - p)
    assert (y.float().view(B, Sq, H) - yr).abs().max().item() < 4e-2
    assert torch.equal(ids32.view(B, Sq).long(), ids)

    dy = rnd((M, H), dev)
    d_word = torch.zeros(V, H, dtype=bf, device=dev)
    d_pos = torch.zeros(512, H, dtype=bf, device=dev)
    d_typ, d_g, d_b = torch.zeros(T, H, dtype=bf, device=dev), torch.zeros(H, dtype=bf, device=dev), \
        torch.zeros(H, dtype=bf, device=dev)
    scratch_dx = torch.empty(M, H, dtype=bf, device=dev)
    owner = torch.empty(V, dtype=torch.int32, device=dev)
    L.call("b2_embed_owner_init", owner.data_ptr(), V, S())
    yr.backward(dy.float().view(B, Sq, H))
    # 4 MB of scratch: the fp32 owner-row path ([tokens + seq*types][H] fp32 = 3.9 MB here); 3 MB: the scan path
    for scratch_bytes in (4 << 20, 3 << 20):
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
        for _ in range(2):  # twice: the owner table must re-arm itself
            for t in (d_word, d_pos, d_typ, d_g, d_b):
                t.zero_()
            L.call("b2_embed_bwd", dy.data_ptr(), 0, pre.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gam.data_ptr(),
                   ids32.data_ptr(), tt32.data_ptr(), B, Sq, H, V, T, 0, p, rs.data_ptr(), 0, d_word.data_ptr(),
                   d_pos.data_ptr(), d_typ.data_ptr(), d_g.data_ptr(), d_b.data_ptr(), scratch_dx.data_ptr(),
                   scratch.data_ptr(), scratch.numel(), owner.data_ptr(), S())
        torch.cuda.synchronize()
        assert rel_l2(d_word.float(), wr.grad) < 1.5e-2
        assert float(d_word[0].float().abs().max()) == 0.0        # padding_idx row
        assert rel_l2(d_pos.float(), pr.grad) < 1.5e-2
        assert rel_l2(d_typ.float(), tr.grad) < 1.5e-2
        assert rel_l2(d_g.float(), gr.grad) < 1.5e-2
        assert rel_l2(d_b.float(), br.grad) < 1.5e-2


@pytest.mark.parametrize("Sq,masked,p,cache", [(128, False, 0.0, False), (128, True, 0.1, False), (128, True, 0.1, True),
                                               (128, False, 0.1, True), (256, True, 0.0, False),
                                               (512, True, 0.1, True), (256, True, 0.1, False),
                                               (512, False, 0.0, False)])
def test_attention_fwd_bwd(cuda_dev, Sq, masked, p, cache):
    """cache: hand both calls a keep-bit buffer (the forward's dropout decisions, re-read by the backward at seq 128;
    ignored at other lengths) -- results must not depend on it"""
    dev = cuda_dev
    B, nh = 3, 4
    H = nh * 64
    M = B * Sq
    torch.manual_seed(2)
    qkv = rnd((M, 3 * H), dev, 1.0)
    mask = None
    if masked:
        lens = torch.tensor([Sq, 9, Sq // 2 + 3], device=dev)
        mask = (torch.arange(Sq, device=dev)[None] < lens[:, None]).long()
    rs = rng_state(dev)
    ctx = torch.empty(M, H, dtype=bf, device=dev)
    lse = torch.empty(B * nh * Sq, dtype=torch.float32, device=dev)
    kb = torch.zeros(B * nh * Sq * (Sq // 64), dtype=torch.int64, device=dev) if cache else None
    L.call("b2_attention_fwd", qkv.data_ptr(), L.ptr(mask), B, Sq, nh, 64, p, rs.data_ptr(), 4, ctx.data_ptr(),
           lse.data_ptr(), L.ptr(kb), S())
    torch.cuda.synchronize()
    keep = attn_keep_mask(B, nh, Sq, 1234, 5, 4, p, dev)
    qr = qkv.double().requires_grad_(True)
    ref, lse_ref = attention_ref(qr, padded_visibility(mask, Sq), B, nh, keep, p)
    assert (ctx.float() - ref).abs().max().item() < 3e-2
    assert (lse.view(B, nh, Sq) - lse_ref).abs().max().item() < 2e-2

    dctx = rnd((M, H), dev)
    dqkv = torch.zeros(M, 3 * H, dtype=bf, device=dev)
    dq_acc = torch.empty(M, H, dtype=torch.float32, device=dev) if Sq > 128 else None
    dbias = torch.zeros(3 * H, dtype=torch.float32, device=dev) if Sq == 128 else None
    L.call("b2_attention_bwd", qkv.data_ptr(), L.ptr(mask), ctx.data_ptr(), dctx.data_ptr(), lse.data_ptr(), B, Sq,
           nh, 64, p, rs.data_ptr(), 4, dqkv.data_ptr(), L.ptr(dq_acc), L.ptr(dbias), L.ptr(kb), S())
    torch.cuda.synchronize()
    if cache and Sq == 128 and p > 0:   # the cached bits are exactly the Philox decisions
        bits = kb.view(B, nh, Sq, 2).cpu().numpy().astype("uint64")
        got = ((bits[..., None] >> np.arange(64, dtype="uint64")) & np.uint64(1)).reshape(B, nh, Sq, 128).astype(bool)
        assert np.array_equal(got, keep.cpu().numpy().astype(bool))
    if dbias is not None:   # fused QKV bias gradient == column sums of what was written
        assert rel_l2(dbias, dqkv.float().sum(0)) < 1e-4
    ref.backward(dctx.double())
    for i, nm in enumerate("qkv"):
        e = rel_l2(dqkv[:, i * H:(i + 1) * H].float(), qr.grad[:, i * H:(i + 1) * H])
        assert e < 3e-2, "d%s rel err %.3g" % (nm, e)


def test_attention_rejects_bad_shapes(cuda_dev):
    qkv = rnd((100, 768), cuda_dev)
    with pytest.raises(RuntimeError, match="multiple of 128"):
        L.call("b2_attention_fwd", qkv.data_ptr(), None, 1, 100, 4, 64, 0.0, None, 0, qkv.data_ptr(), None, None, S())
    with pytest.raises(RuntimeError, match="head_dim"):
        L.call("b2_attention_fwd", qkv.data_ptr(), None, 1, 128, 4, 32, 0.0, None, 0, qkv.data_ptr(), None, None, S())


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_head_and_ce(cuda_dev, p):
    dev = cuda_dev
    B, Sq, H, C = 32, 128, 768, 6
    torch.manual_seed(3)
    hs = rnd((B * Sq, H), dev)
    Wp, bp, Wc, bc = rnd((H, H), dev, 0.03), rnd((H,), dev, 0.1), rnd((C, H), dev, 0.05), rnd((C,), dev, 0.1)
    labels = torch.randint(0, C, (B,), device=dev)
    rs = rng_state(dev)
    pooled = torch.empty(B, H, dtype=bf, device=dev)
    logits = torch.empty(B, C, dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    dlog = torch.empty(B, C, dtype=torch.float32, device=dev)
    L.call("b2_head_fwd", hs.data_ptr(), B, Sq, H, Wp.data_ptr(), bp.data_ptr(), Wc.data_ptr(), bc.data_ptr(), C, p,
           rs.data_ptr(), 37, pooled.data_ptr(), logits.data_ptr(), S())
    L.call("b2_ce_fwd_bwd", logits.data_ptr(), labels.data_ptr(), B, C, loss.data_ptr(), dlog.data_ptr(), S())
    h0 = hs.view(B, Sq, H)[:, 0].float().requires_grad_(True)
    Wpr, bpr, Wcr, bcr = (t.float().requires_grad_(True) for t in (Wp, bp, Wc, bc))
    pr = torch.tanh(h0 @ Wpr.t() + bpr)
    if p > 0:
        keep = torch.from_numpy(philox_keep_mask(B * H, 1234, 5, 37, p).reshape(B, H)).to(dev)
        prd = pr * keep / (1 - p)
    else:
        prd = pr
    zr = prd @ Wcr.t() + bcr
    lr = F.cross_entropy(zr, labels)
    assert (logits - zr).abs().max().item() < 2e-2
    # CE kernel is exact fp32 on the logits it was given
    l2 = F.cross_entropy(logits, labels)
    assert abs(loss.item() - l2.item()) < 1e-5
    lg = logits.clone().requires_grad_(True)
    F.cross_entropy(lg, labels).backward()
    assert (dlog - lg.grad).abs().max().item() < 1e-6

    grads = {k: torch.empty_like(v) for k, v in dict(Wp=Wp, bp=bp, Wc=Wc, bc=bc).items()}
    d_hidden = torch.empty(B * Sq, H, dtype=bf, device=dev)
    scratch = torch.empty(2 * B, H, dtype=torch.float32, device=dev)
    L.call("b2_head_bwd", dlog.data_ptr(), hs.data_ptr(), pooled.data_ptr(), B, Sq, H, Wp.data_ptr(), Wc.data_ptr(),
           C, p, rs.data_ptr(), 37, grads["Wp"].data_ptr(), grads["bp"].data_ptr(), grads["Wc"].data_ptr(),
           grads["bc"].data_ptr(), d_hidden.data_ptr(), 0, scratch.data_ptr(), S())
    torch.cuda.synchronize()
    lr.backward()
    assert rel_l2(grads["Wc"].float(), Wcr.grad) < 2e-2
    assert rel_l2(grads["bc"].float(), bcr.grad) < 2e-2
    assert rel_l2(grads["Wp"].float(), Wpr.grad) < 2e-2
    assert rel_l2(grads["bp"].float(), bpr.grad) < 2e-2
    dh = d_hidden.view(B, Sq, H)
    assert rel_l2(dh[:, 0].float(), h0.grad) < 2e-2
    assert float(dh[:, 1:].float().abs().max()) == 0.0


def test_adamw_background_form_matches_hf_restatement(cuda_dev):
    """b2_adamw_background (the one-GPU form shaped to run beside the GEMM CTAs: 128 threads x 32 registers) +
    b2_adamw_prepare (bias-corrected step size on the device) vs oracle/adamw_ref.HFAdamW, and bit-identical to
    b2_bucket_reduce_adamw on the same inputs."""
    from oracle import adamw_ref
    dev = cuda_dev
    n = 8 * 5004        # (half of it is a whole number of 8-element decay-flag groups; 39 blocks + a ragged tail)
    torch.manual_seed(4)
    master = torch.randn(n, device=dev)
    ref_p = {"w.weight": master[: n // 2].clone().cpu(), "w.bias": master[n // 2:].clone().cpu()}
    opt = adamw_ref.HFAdamW(ref_p, lr=3e-5, weight_decay=0.01)
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    shadow = torch.empty(n, dtype=bf, device=dev)
    master2, m2, v2, shadow2 = master.clone(), m.clone(), v.clone(), shadow.clone()
    decay = torch.zeros(n // 8, dtype=torch.uint8, device=dev)
    decay[: n // 16] = 1
    step = torch.zeros(1, dtype=torch.int64, device=dev)
    step_size = torch.zeros(1, device=dev)
    rs = rng_state(dev, 1, 0)
    hp = L.AdamWHParams()
    hp.lr, hp.beta1, hp.beta2, hp.eps, hp.weight_decay, hp.correct_bias = 3e-5, 0.9, 0.999, 1e-6, 0.01, 1
    L.call("b2_adamw_prepare", hp, step.data_ptr(), step_size.data_ptr(), S())
    for it in range(4):
        g = (torch.randn(n, device=dev) * 0.01).to(bf)
        L.call("b2_adamw_background", g.data_ptr(), shadow.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(),
               decay.data_ptr(), 0, n, hp, step_size.data_ptr(), S())
        L.call("b2_bucket_reduce_adamw", L.ptr_array([g.data_ptr()]), L.ptr_array([shadow2.data_ptr()]), 1, 0,
               master2.data_ptr(), m2.data_ptr(), v2.data_ptr(), decay.data_ptr(), 0, n, hp, step.data_ptr(), S())
        L.call("b2_step_advance", step.data_ptr(), rs.data_ptr(), None, S())
        L.call("b2_adamw_prepare", hp, step.data_ptr(), step_size.data_ptr(), S())
        gc = g.float().cpu()
        opt.step({"w.weight": gc[: n // 2], "w.bias": gc[n // 2:]})
    torch.cuda.synchronize()
    ref = torch.cat([ref_p["w.weight"], ref_p["w.bias"]])
    d_ref = (master.cpu() - ref).abs().max().item()
    d_reg = (master - master2).abs().max().item()
    d_m, d_v = (m - m2).abs().max().item(), (v - v2).abs().max().item()
    # same statements as the regular kernel; the compiler may contract a different product of `m*b1 + g*(1-b1)` into
    # the FMA, so moments agree to an ulp, not necessarily bit for bit
    assert d_ref < 3e-7 and d_reg < 3e-7 and d_m < 1e-9 and d_v < 1e-11, (d_ref, d_reg, d_m, d_v)
    assert (shadow.float() - shadow2.float()).abs().max().item() <= 2.0 ** -6
    with pytest.raises(RuntimeError, match="8-element aligned"):
        L.call("b2_adamw_background", g.data_ptr(), shadow.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(),
               decay.data_ptr(), 4, n, hp, step_size.data_ptr(), S())


def test_ce_ignore_index_matches_torch(cuda_dev):
    """torch.nn.CrossEntropyLoss defaults (multi-gpu-distributed-cls.py:343): label -100 is ignored and the mean runs
    over the remaining samples; all-ignored -> nan."""
    dev = cuda_dev
    B, C = 32, 6
    torch.manual_seed(5)
    logits = torch.randn(B, C, device=dev)
    labels = torch.randint(0, C, (B,), device=dev)
    labels[::5] = -100
    loss = torch.empty((), dtype=torch.float32, device=dev)
    dlog = torch.empty(B, C, dtype=torch.float32, device=dev)
    L.call("b2_ce_fwd_bwd", logits.data_ptr(), labels.data_ptr(), B, C, loss.data_ptr(), dlog.data_ptr(), S())
    lg = logits.clone().requires_grad_(True)
    ref = F.cross_entropy(lg, labels)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5
    assert (dlog - lg.grad).abs().max().item() < 1e-6
    assert float(dlog[::5].abs().max()) == 0.0
    labels[:] = -100
    L.call("b2_ce_fwd_bwd", logits.data_ptr(), labels.data_ptr(), B, C, loss.data_ptr(), dlog.data_ptr(), S())
    assert torch.isnan(loss).item() and float(dlog.abs().max()) == 0.0


def test_adamw_matches_hf_restatement(cuda_dev):
    """Fused kernel vs oracle/adamw_ref.HFAdamW over several steps, decay and no-decay vectors, world == 1."""
    from oracle import adamw_ref
    dev = cuda_dev
    n = 8 * 5000
    torch.manual_seed(4)
    master = torch.randn(n, device=dev)
    ref_p = {"w.weight": master[: n // 2].clone().cpu(), "w.bias": master[n // 2:].clone().cpu()}
    opt = adamw_ref.HFAdamW(ref_p, lr=3e-5, weight_decay=0.01)
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    shadow = torch.empty(n, dtype=bf, device=dev)
    decay = torch.zeros(n // 8, dtype=torch.uint8, device=dev)
    decay[: n // 16] = 1
    step = torch.zeros(1, dtype=torch.int64, device=dev)
    rs = rng_state(dev, 1, 0)
    hp = L.AdamWHParams()
    hp.lr, hp.beta1, hp.beta2, hp.eps, hp.weight_decay, hp.correct_bias = 3e-5, 0.9, 0.999, 1e-6, 0.01, 1
    for it in range(4):
        g = (torch.randn(n, device=dev) * 0.01).to(bf)
        L.call("b2_bucket_reduce_adamw", L.ptr_array([g.data_ptr()]), L.ptr_array([shadow.data_ptr()]), 1, 0,
               master.data_ptr(), m.data_ptr(), v.data_ptr(), decay.data_ptr(), 0, n, hp, step.data_ptr(), S())
        L.call("b2_step_advance", step.data_ptr(), rs.data_ptr(), None, S())
        gc = g.float().cpu()
        opt.step({"w.weight": gc[: n // 2], "w.bias": gc[n // 2:]})
    torch.cuda.synchronize()
    ref = torch.cat([ref_p["w.weight"], ref_p["w.bias"]])
    assert (master.cpu() - ref).abs().max().item() < 2e-7
    assert int(step.item()) == 4 and int(rs[1].item()) == 4
    assert torch.equal(shadow.cpu(), master.to(bf).cpu())
    # torch.optim.AdamW is a different algorithm (eps inside the bias-corrected denominator): must NOT match that well
    tp = torch.nn.Parameter(torch.ones(8))
    to = torch.optim.AdamW([tp], lr=3e-5, eps=1e-6, weight_decay=0.01)
    hp2 = {"p": torch.ones(8)}
    ho = adamw_ref.HFAdamW({"p.weight": hp2["p"]}, lr=3e-5, weight_decay=0.01)
    for _ in range(3):
        gg = torch.full((8,), 1e-6)
        tp.grad = gg.clone()
        to.step()
        ho.step({"p.weight": gg})
    assert (tp.data - hp2["p"]).abs().max().item() > 1e-7
