"""Shared parity helpers for the tests and __graft_entry__.smoke().

* a numpy replica of the kernels' Philox4x32-10 dropout stream, so the oracle can replay the exact keep-masks the
  CUDA path drew (dropout-ON parity is then a plain numeric comparison, not a statistical one);
* tolerance table (BASELINE.md §4) and comparison utilities;
* tiny / full configurations.
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytorch_distributed_nlp_b200 as b2  # noqa: E402
from oracle import adamw_ref, bert_ref  # noqa: E402

# ---- stated tolerances (bf16 compute vs the fp32 oracle; BASELINE.md §4) -------------------------------------------
TOL_LOSS = 2e-3          # |loss - loss_ref|
TOL_LOGITS = 1e-2        # max |logit - logit_ref|
TOL_GRAD_REL = 2e-2      # per-tensor ||g - g_ref|| / ||g_ref||  (tensors with a non-negligible reference norm)
TOL_TRAJ = 1e-2          # per-step |loss - loss_ref| along a short trajectory
# Query / key projection gradients are the most rounding-sensitive tensors of the model: their gradient is
# P * (dP - delta) with dP - delta = dO . (V_j - O_i), and at random initialisation the value rows of a sequence are
# nearly collinear in the upper layers, so every bf16 rounding upstream is amplified ~10x.  With the residual stream of
# the forward kept in fp32 (csrc/gemm_ln.cu) they meet the general 2e-2 at the headline config A (measured worst 1.9e-2,
# stock torch bf16 autocast on the same batch: 1.4e-2; tests/test_trainer.py measures both).  Stated exception
# (BASELINE.md §4): the deeper / longer parity configs -- bert-large's 24 layers (config C, measured 3.4e-2) and the
# seq-512 attention path (config B shapes, 1.9e-2) -- are held to 4e-2 on these tensors only.
TOL_GRAD_REL_QK = 4e-2


def is_qk(name):
    return ".attention.self.query." in name or ".attention.self.key." in name


def grad_tol(name, qk_tol=TOL_GRAD_REL):
    return qk_tol if is_qk(name) else TOL_GRAD_REL


def report(tag, obj):
    """appends one JSON line to $B2_PARITY_REPORT (the GPU runs collect their measured parity tables there)"""
    import json
    path = os.environ.get("B2_PARITY_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps({"tag": tag, **obj}) + "\n")


def tiny_config(**kw):
    d = dict(vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512,
             max_position_embeddings=128, num_labels=6)
    d.update(kw)
    return b2.BertConfig(**d)


def full_config(**kw):
    return b2.chinese_bert_wwm_ext_config(num_labels=6, **kw)


# ---- Philox4x32-10 replica (csrc/common.cuh: philox4x32_10 / dropout_keep8) -------------------------------------------
def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Salmon et al., "Parallel random numbers: as easy as 1, 2, 3" (SC'11): counters are uint64 arrays holding 32-bit
    values, keys python ints.  tests/test_host.py checks it against the published known-answer vectors."""
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    W0, W1 = 0x9E3779B9, 0xBB67AE85
    mask32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = M0 * c0
        p1 = M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & mask32
        hi1, lo1 = p1 >> np.uint64(32), p1 & mask32
        n0 = hi1 ^ c1 ^ np.uint64(k0)
        n2 = hi0 ^ c3 ^ np.uint64(k1)
        c0, c1, c2, c3 = n0, lo1, n2, lo0
        k0 = (k0 + W0) & 0xFFFFFFFF
        k1 = (k1 + W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def philox_keep_mask(n_elements, seed, step, site, p):
    """Boolean keep mask for `n_elements` (multiple of 8) consecutive elements of dropout site `site`."""
    assert n_elements % 8 == 0
    if p <= 0:
        return np.ones(n_elements, dtype=bool)
    thresh = int(p * 65536.0 + 0.5)
    g = np.arange(n_elements // 8, dtype=np.uint64)
    mask32 = np.uint64(0xFFFFFFFF)
    c0, c1, c2, c3 = philox4x32_10(g & mask32, g >> np.uint64(32), np.full_like(g, site & 0xFFFFFFFF),
                                   np.full_like(g, step & 0xFFFFFFFF), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    lanes = np.stack([c0 & np.uint64(0xFFFF), c0 >> np.uint64(16), c1 & np.uint64(0xFFFF), c1 >> np.uint64(16),
                      c2 & np.uint64(0xFFFF), c2 >> np.uint64(16), c3 & np.uint64(0xFFFF), c3 >> np.uint64(16)],
                     axis=1)
    return (lanes >= np.uint64(thresh)).reshape(-1)


def oracle_masks(cfg, B, S, seed, step):
    """Keep masks for every dropout site of one training forward, keyed as oracle.bert_ref.forward expects."""
    H, nh, L = cfg.hidden_size, cfg.num_attention_heads, cfg.num_hidden_layers
    p_h, p_a = cfg.hidden_dropout_prob, cfg.attention_probs_dropout_prob
    t = lambda a, shape: torch.from_numpy(a.reshape(shape))
    m = {"emb": t(philox_keep_mask(B * S * H, seed, step, 0, p_h), (B, S, H)),
         "cls": t(philox_keep_mask(B * H, seed, step, 1 + 3 * L, p_h), (B, H))}
    for l in range(L):
        m[("attn", l)] = t(philox_keep_mask(B * nh * S * S, seed, step, 1 + 3 * l, p_a), (B, nh, S, S))
        m[("self_out", l)] = t(philox_keep_mask(B * S * H, seed, step, 2 + 3 * l, p_h), (B, S, H))
        m[("out", l)] = t(philox_keep_mask(B * S * H, seed, step, 3 + 3 * l, p_h), (B, S, H))
    return m


def attn_keep_mask(B, nh, S, seed, step, site, p, device="cpu"):
    """Attention-probability keep mask [B, nh, S, S] as the attention kernels draw it: element ((b*nh + h)*S + q)*S + k
    of dropout site `site` (packed bins use the same index, with b the bin).  None when p == 0."""
    if p <= 0:
        return None
    return torch.from_numpy(philox_keep_mask(B * nh * S * S, seed, step, site, p).reshape(B, nh, S, S)).to(device)


def padded_visibility(mask, S):
    """[B, S, S] bool: query q of sequence b sees key k iff mask[b, k] (mask None: every key)"""
    if mask is None:
        return None
    return (mask != 0)[:, None, :].expand(mask.shape[0], S, S)


def packed_visibility(segments):
    """[bins, 128, 128] bool from the packed segment words (lo | hi << 16): row q sees keys lo(q) <= k < hi(q)"""
    seg = segments.long()
    lo, hi = (seg & 0xffff)[..., None], (seg >> 16)[..., None]
    k = torch.arange(seg.shape[-1], device=seg.device)
    return (k >= lo) & (k < hi)


def attention_ref(qkv, vis, B, nh, keep=None, p=0.0):
    """HF BertSelfAttention (eager) in float64: softmax(q k^T / 8 + (~vis) * finfo(fp32).min) -> dropout -> @ v.
    qkv [B*S, 3*nh*64] (Q | K | V column blocks); vis [B, S, S] bool (vis[b, q, k]: query q may see key k) or None
    (every key visible); keep [B, nh, S, S] or None.  Make qkv a float64 leaf to take gradients by autograd.
    Returns ctx [B*S, nh*64] and the natural-log lse [B, nh, S] of the masked scores.  A row with no visible key has
    all-equal scores (finfo.min absorbs them), so its softmax is uniform, as in HF."""
    H = nh * 64
    S = qkv.shape[0] // B
    q, k, v = (qkv[:, i * H:(i + 1) * H].double().view(B, S, nh, 64).transpose(1, 2) for i in range(3))
    s = (q @ k.transpose(-1, -2)) * 0.125
    if vis is not None:
        s = s + (~vis)[:, None].double() * torch.finfo(torch.float32).min
    pr = torch.softmax(s, -1)
    lse = torch.logsumexp(s, -1)
    if keep is not None:
        pr = pr * keep / (1 - p)
    return (pr @ v).transpose(1, 2).reshape(B * S, H), lse


# ---- comparisons --------------------------------------------------------------------------------------------------------
def rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def grad_report(got, ref, floor_frac=1e-3):
    """Per-tensor relative L2 error.  Tensors whose reference norm is below `floor_frac` of the largest reference
    norm are compared in absolute terms against that scale (bf16 noise dominates a near-zero gradient)."""
    scale = max(float(v.double().norm()) for v in ref.values())
    worst, rows = 0.0, []
    for k, r in ref.items():
        g = got[k].detach().cpu().double()
        r = r.double()
        rn = float(r.norm())
        err = float((g - r).norm())
        rel = err / rn if rn > floor_frac * scale else err / (floor_frac * scale)
        rows.append((k, rel, rn))
        worst = max(worst, rel)
    return worst, rows


def assert_grads_within_tolerance(got, ref, floor_frac=1e-3, qk_tol=TOL_GRAD_REL):
    """every tensor within the stated tolerance TOL_GRAD_REL (query / key projections: `qk_tol`, see TOL_GRAD_REL_QK);
    returns (worst q/k, worst other)"""
    _, rows = grad_report(got, ref, floor_frac)
    bad = [(k, rel) for (k, rel, _rn) in rows if rel > grad_tol(k, qk_tol)]
    assert not bad, sorted(bad, key=lambda r: -r[1])[:5]
    qk = max([rel for (k, rel, _rn) in rows if is_qk(k)] or [0.0])
    other = max([rel for (k, rel, _rn) in rows if not is_qk(k)] or [0.0])
    return qk, other


def state_from_hf_init(cfg, seed=123):
    """Initial fp32 weights: HF ``_init_weights`` under set_seed(seed) (what from_pretrained leaves for a fresh head)."""
    from oracle import cpu_step
    hf = cpu_step.build_hf_model(cfg, seed=seed)
    return {k: v.detach().clone() for k, v in hf.named_parameters()}


def make_model(cfg, state, dev):
    model = b2.BertForSequenceClassification(cfg)
    model.load_state_dict(state, strict=True)
    model.to(dev)
    return model


def to_dev(batch, dev):
    return {k: v.to(dev) for k, v in batch.items()}


def run_smoke():
    """One tiny training step on cuda:0 (dropout ON, replayed in the oracle) checked against the oracle."""
    dev = torch.device("cuda", 0)
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, dev)
    model.train()
    seed = 4242
    model._engine.seed_dropout(seed, 0)
    batch = bert_ref.synthetic_batch(cfg, 4, 128, 1000, padded=True)
    out = model(**{k if k != "label" else "labels": v for k, v in to_dev(batch, dev).items()})
    loss = torch.nn.functional.cross_entropy(out[1], batch["label"].to(dev))
    loss.backward()
    torch.cuda.synchronize()
    masks = oracle_masks(cfg, 4, 128, seed, 0)
    ref_loss, ref_logits, ref_grads = bert_ref.loss_and_grads(state, cfg, batch, masks=masks)
    dl = abs(float(loss) - float(ref_loss))
    dz = float((out[1].detach().cpu() - ref_logits).abs().max())
    qk, other = assert_grads_within_tolerance(model.grad_dict(), ref_grads)
    print("smoke: |dloss|=%.2e max|dlogit|=%.2e worst grad rel-L2: q/k %.2e, others %.2e" % (dl, dz, qk, other))
    assert dl <= TOL_LOSS and dz <= TOL_LOGITS, "smoke parity failed"
    if torch.cuda.device_count() >= 2:
        run_smoke_ddp(2)


def run_smoke_ddp(world=2):
    """>= 2 GPUs visible: the peer-HBM gradient exchange + partitioned AdamW + loss_reduce / output_reduce of
    tests/ddp_worker.py (eager, GradScaler and CUDA-graph loops vs the oracle's DDP restatement) on `world` ranks."""
    import subprocess
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29571", os.path.join(ROOT, "tests", "ddp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    tail = (r.stdout[-2000:] + r.stderr[-2000:])
    assert r.returncode == 0 and "mode fused OK" in r.stdout, "smoke: %d-rank DDP parity failed:\n%s" % (world, tail)
    print("smoke: %d-rank peer-HBM DDP parity OK" % world)
