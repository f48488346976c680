"""The fused attention kernels (csrc/attention.cu: b2_attention_fwd / _bwd and their packed forms) element-wise against
HF's attention in float64, at bounds derived from the kernels' rounding sequence, and the dropout rates they reject.

Reference.  parity.attention_ref in float64 from the same bf16 operands, gradients by autograd, with the Philox
replica's keep mask (parity.attn_keep_mask) and the visibility of parity.padded_visibility / packed_visibility.  U =
2^-24 and UB = 2^-8 are the fp32 and bf16 unit roundoffs, gamma(n) = nU / (1 - nU).  The only assumption about
undocumented hardware is test_gemm_reference's: a wgmma accumulation over K is within C_ACC K U (|A| @ |B|) of the
exact product (C_ACC imported from there).  Everything else follows the rounding points of attention.cu:

  scores      s = Q K^T, K = 64: E_s = C_ACC 64 U (|Q| @ |K|^T).  c2 = 0.125 fp32(log2 e) is off by EPS_C2 relative.
  fwd exp     x = fma(s, c2, -m) (U |x|), pr = ex2.approx.ftz(x): 4U relative, test_gemm_reference's ex2 model, plus
              ln2 times the argument's error.  So pr is off by rho = ln2 (c2 E_s + EPS_C2 |s c2| + U |x|) + 4U
              relative.  The row maximum m cancels between P and l, except through the fma's rounding.
  row sum     l: 32 sequential adds per lane and key block, 2 quad shuffles: gamma(34 nkv + 2), nkv = seq / 128.
  P tile      bf16(fp32(pr sc)), sc = fp32(1 / (1 - p)), which differs from the reference's 1 / (1 - p) by D_SC
              relative: UB + U + D_SC.
  fwd output  o = P~ V, K = 128 per key block; ctx = bf16(o (1 / l)), IEEE division (no fast math): 2U.
  lse         (m + log2f(l)) ln2 with log2f at 1 ulp (2U |log2 l|), the add (U |lse2|) and fp32(ln2) (U + EPS_LN2).
  online      seq > 128 (attention_fwd_kernel): at each of the nkv - 1 later key blocks, o and l are rescaled by
              alpha = exp2f(m_prev - m_new), 2 ulp, of an fp32 difference of two maxima (U |2 m|), then one
              multiply-add: EA = (nkv - 1) (6U + 2 ln2 U max|s c2|) relative on every P and on l.  The bound does
              not assume the P tile was rounded at the final maximum: each key's P~ carries its own relative error.
  bwd exp     pr' = ex2(fma(s, c2, -lse2)) with lse2 = fp32(lse log2e) from the kernel's own lse, whose distance
              from the float64 lse2 is measured (|d_lse2|): rho' = ln2 (c2 E_s + EPS_C2 |s c2| + |d_lse2| + U |x|)
              + 4U.  Rows with no visible key take row_masked_x: P = 1/seq, rho' = 4U + ln2 2U log2(seq).
  dP, delta   dp = dO V^T, K = 64: E_dp = C_ACC 64 U (|dO| @ |V|^T).  delta = sum ctx dO over 64 fp32 adds:
              gamma(64) sum |ctx dO|, plus the kernel's own ctx error, measured: |sum (ctx - ctx64) dO|.  This is
              where the P-tile and ctx roundings enter dS.
  dS          bf16(fp32(pr' fp32(dp sc - delta)) 0.125): A = keep sc dp - delta within keep (sc E_dp + D_SC |dp|)
              + |d_delta| + gamma(64) sum |ctx dO| + 2U (|keep sc dp| + |delta|); E_dS32 = 0.125 P (E_A + (rho' + U)
              |A|); the tile: E_dS = UB |dS| + (1 + UB) E_dS32.
  gradients   dV = P~'^T dO and dK = dS^T Q: one accumulator over all seq query rows (C_ACC seq U).  dQ = dS K,
              K = 128 per key block, then at seq > 128 nkv fp32 atomics in no fixed order and dq_convert's bf16
              rounding: (C_ACC 128 + nkv) U.  E_dQ = E_dS @ |K| + (C_ACC 128 + nkv) U (|dS| + E_dS) @ |K|, etc.
  QKV bias    (seq 128) dbias += column sums of the stored bf16 d_qkv, from a nonzero fp32 C0: 4 in-warp adds and
              one atomic per warp per item, in no fixed order: gamma(4 + 8 batch) (|C0| + sum |d_qkv|).
Each stored output gets bf_bound(ref, E) = UB |ref| + (1 + UB) E.  Every first-order E is multiplied by SLACK = 1.02
for the products of small terms left out, and gets an absolute 2^-126 per P or dS element (ex2.approx.ftz flushes
results below it).  The bound is a running-error bound computed in float64 next to the reference, so rows where dS
cancels (nearly one-hot rows, one-token segments under dropout) are covered by the same rule as every other row.
lse is checked on rows with a visible key; the others must keep lse < -1e38, which the backward takes as "no visible
key".

The packed x4-dropout case.  test_attention.py used to leave it out: there the dQ / dK of one-token segments came out
up to ~50x the float64 emulation's rounding residue.  It passes this bound, and the kernel does what the model above
describes; the kernel and the emulation differ in how they round ctx.  A one-token row's only visible key is itself,
so its true dS is 0 and what any bf16 implementation returns is rounding residue: the P tile holds bf16(sc) =
1.109375 against sc = 1.1111112, and ctx = bf16(1.109375 v / l).  1.109375 v is exact in 15 bits, so about one element
in 64 is an exact bf16 tie.  The float64 emulation has l = 1 and rounds the tie to even.  The kernel has l = ex2(x)
with x = fma(s, c2, -m) the nonzero rounding remainder of s c2, so its 1 / l moves the value off the tie, either way.
One such flip moves delta, and so dS, by as much as the whole residue.  Kernel and emulation residues are then the
same size but not on the same elements, and a rule of 3x the emulation's error per (segment, head) block cannot hold
for blocks of one row.  This bound takes delta's error from the kernel's own ctx, so a flipped tie is inside it by
construction.  Measured on that case (H100): the one-token rows' max |dQ - ref| is 0.41 for the kernel, the float64
emulation and kernel_emulation alike, while the kernel differs from the emulations by up to 0.18.  On the CPU, all 402
of the one-token rows' ctx elements where the float64 and fp32 emulations disagree are such ties (of 1096 ties).

Shapes and edges: seq 128, 256, 384 (three key and query blocks: three online rescales, three dQ atomics per element)
and 512, with test_attention.padded_masks (prefix lengths at every 32-key word / 64-key half / 128-key block edge,
non-prefix masks, a row with no visible key, at 512 the fully masked leading key blocks) and packed_layout (one-token
segments, unused rows); p in {0, 0.1} and operand scale x1 and x4 on both; engine sizes at p = 0.1: config A (B 32,
12 heads, seq 128) at the persistent backward's default grid and at B2_DEBUG_ATTN_CTAS = 1 and 7, config B (B 16, 12
heads, seq 512) and bert-large (B 16, 16 heads, seq 128).  The float64 work runs in chunks of whole sequences of at
most CHUNK elements per [b, h, q, k] tensor, so a test holds well under 2 GB on the card.

The checker catches subtle defects.  kernel_emulation restates the kernels' rounding sequence in torch fp32 / bf16
(on the CPU, no GPU needed): the clean emulation passes every check, at seq 128, 384, 512 and a packed batch, and
each planted defect fails at least one element: one visible key dropped from one row, one masked key admitted, one
keep bit flipped in the backward only, one row's lse off by 1e-3, the +-1 edge of one packed segment, one key
block's dQ contribution missing at seq 512, dS without the 0.125.

Rejected arguments: a dropout_p outside [0, 1) or NaN, at all four entry points.  A negative or NaN p used to run
with no mask and convert p * 65536 to uint32 (undefined for a negative value); p >= 1 dropped every key.  These run
in a child process that sees no device, as test_gemm_reference's alignment checks do.

Measured on an H100 80GB HBM3 (700 W power limit), worst error / bound per check family:
  padded sweep      ctx 0.795, lse 0.012, dQ 0.969, dK 0.962, dV 0.817, dbias 0.012
  packed            ctx 0.802, lse 0.0087, dQ 0.965, dK 0.966, dV 0.835, dbias 0.013
  config A          ctx 0.738, lse 0.0093, dQ 0.964, dK 0.521, dV 0.58, dbias 0.0063 (default grid and 1 and 7 CTAs)
  config B          ctx 0.784, lse 0.012, dQ 0.967, dK 0.411, dV 0.345
  bert-large        ctx 0.762, lse 0.0090, dQ 0.967, dK 0.584, dV 0.52, dbias 0.0070
  every row with no visible key kept lse < -1e38.
dQ and dK come near 1 in the rows where dS cancels: there the largest term of the bound is the measured ctx error
inside delta, which the error itself nearly equals.  lse and dbias sit far inside their bounds, which are dominated by
the C_ACC score model and by gamma(4 + 8 batch)'s worst-case order; the lse bound still catches an error of 1e-3 at
x1 scores.  The clean emulation on the CPU reaches ctx 0.73, dQ 0.967, dK 0.964, dV 0.848; each planted defect fails
its most sensitive check by a factor of 12.8 (the lse offset) or more, most by far over 100.
Runtime, from one `pytest -m gpu tests/test_attention_reference.py --durations=0` on that card: 25 tests in 13.4 s as
pytest counts it.  The slowest are the first (3.5 s, mostly CUDA start-up) and config B (2.9 s: its 50M-element Philox
keep mask is drawn on the CPU).
With B2_PARITY_REPORT set, every check appends its ratio there (tag "attention_reference").
"""
import contextlib
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from parity import attention_ref, attn_keep_mask, packed_visibility, padded_visibility, report
from pytorch_distributed_nlp_b200 import _lib as L
from test_attention import SEED, SITE, STEP, attn_bwd, attn_fwd, packed_layout, padded_masks
from test_gemm_reference import C_ACC, U, UB, drop_scale, gamma

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAG = "attention_reference"
bf, f32, f64 = torch.bfloat16, torch.float32, torch.float64
LN2 = math.log(2.0)
LOG2E_32 = float(np.float32(math.log2(math.e)))       # kLog2e
LN2_32 = float(np.float32(LN2))                       # kLn2
C2 = 0.125 * LOG2E_32                                 # p.scale * kLog2e, exact in fp32
EPS_C2 = abs(LOG2E_32 / math.log2(math.e) - 1.0)
EPS_LN2 = abs(LN2_32 / LN2 - 1.0)
MASK_BIAS = float(torch.finfo(f32).min)               # kMaskBias
EX2 = 4 * U                                           # ex2.approx relative error (test_gemm_reference)
TINY = 2.0 ** -126                                    # ex2.approx.ftz flushes results below this to 0
SLACK = 1.02
CHUNK = 1 << 22                                       # elements per [b, h, q, k] float64 tensor


# ---- the checker ----------------------------------------------------------------------------------------------------
class Verdict:
    """worst error / bound per check family, and the failing elements by (sequence, head, row, column)"""

    def __init__(self, case):
        self.case, self.worst, self.bad = case, {}, []

    def _note(self, family, worst):
        old = self.worst.get(family, 0.0)
        self.worst[family] = old if old != old else (worst if worst != worst or worst > old else old)

    def within(self, family, got, ref, bound, b0=0, where=None):
        """element-wise |got - ref| <= bound over [b, h, row, col] (or [b, h, row] for lse); `where` limits the check
        to some elements.  Anything that is not <= 1, NaN included, fails."""
        ratio = (got.double() - ref).abs() / bound.clamp_min(1e-300)
        if where is not None:
            ratio = torch.where(where, ratio, torch.zeros_like(ratio))
        worst = float(ratio.max()) if ratio.numel() else 0.0
        self._note(family, worst)
        bad = ~(ratio <= 1.0)
        if bool(bad.any()):
            nan = torch.isnan(ratio)
            flat = int(nan.flatten().nonzero()[0]) if bool(nan.any()) else int(ratio.argmax())
            idx = tuple(int(i) for i in np.unravel_index(flat, tuple(ratio.shape)))
            at = dict(zip(("sequence", "head", "row", "col"), (idx[0] + b0,) + idx[1:]))
            self.bad.append("%s: error %.3g x its bound at %s (got %r, ref %r, %d elements over, %d NaN)" % (
                family, worst, at, float(got[idx]), float(ref[idx]), int(bad.sum()), int(nan.sum())))

    def require(self, family, bad, what):
        """a condition that must hold element-wise; `bad` marks the elements that break it"""
        n = int(bad.sum())
        self._note(family, 0.0 if n == 0 else float("inf"))
        if n:
            self.bad.append("%s: %d elements %s, first at %s" % (family, n, what, tuple(bad.nonzero()[0].tolist())))

    def finish(self):
        for family, worst in sorted(self.worst.items()):
            report(TAG, {"case": self.case, "family": family, "err_over_bound": worst})
        print("%s: %s" % (self.case, "  ".join("%s %.3g" % kv for kv in sorted(self.worst.items()))))
        return self

    def assert_ok(self):
        assert not self.bad, "%s:\n  %s" % (self.case, "\n  ".join(self.bad))


def heads(t, B, S, nh):
    """[B*S, nh*64] -> [B, nh, S, 64] float64"""
    return t.double().view(B, S, nh, 64).transpose(1, 2)


def check_outputs(case, qkv, dctx, vis, B, S, nh, p, keep, ctx, lse, dqkv, dbias=None, c0=None, slack=SLACK,
                  grad_bounds=None):
    """every output of one forward + backward against float64 at the bounds of the module docstring; `slack`
    scales every first-order error term E (not the final bf16 rounding); grad_bounds, if given ([B*S, 3*nh*64]
    float64), receives the bounds of dQ | dK | dV in d_qkv's layout"""
    dev, H, nkv = qkv.device, nh * 64, S // 128
    sc32, sc64 = drop_scale(p), 1.0 / (1.0 - p)
    d_sc = abs(sc32 / sc64 - 1.0)
    v = Verdict(case)
    bc = max(1, CHUNK // (nh * S * S))
    for b0 in range(0, B, bc):
        b1 = min(B, b0 + bc)
        n = b1 - b0
        rows = slice(b0 * S, b1 * S)
        vis_c = vis[b0:b1] if vis is not None else None
        keep_c = keep[b0:b1] if keep is not None else None
        # the reference: HF attention in float64, gradients by autograd
        qr = qkv[rows].double().requires_grad_(True)
        ref, lse64 = attention_ref(qr, vis_c, n, nh, keep_c, p)
        lse64 = lse64.detach()
        ref.backward(dctx[rows].double())
        ref = heads(ref.detach(), n, S, nh)
        gq, gk, gv = (heads(qr.grad[:, i * H:(i + 1) * H], n, S, nh) for i in range(3))
        del qr
        # magnitudes for the bound, from the same operands
        q, k, vv = (heads(qkv[rows, i * H:(i + 1) * H], n, S, nh) for i in range(3))
        do = heads(dctx[rows], n, S, nh)
        vis4 = vis_c[:, None] if vis_c is not None else torch.ones(n, 1, S, S, dtype=torch.bool, device=dev)
        none = ~vis4.any(-1, keepdim=True)                      # rows with no visible key
        seen = vis4 & ~none
        kf = keep_c.double() if keep_c is not None else torch.ones(1, dtype=f64, device=dev)
        s = q @ k.transpose(-1, -2)
        E_s = C_ACC * 64 * U * (q.abs() @ k.abs().transpose(-1, -2))
        s2 = s * C2                                             # log2 domain
        sm = torch.where(seen, s * 0.125, -math.inf)
        lse_t = torch.logsumexp(sm, -1, keepdim=True)
        P = torch.where(seen, torch.exp(sm - torch.where(none, 0.0, lse_t)), 0.0)
        P = torch.where(none, 1.0 / S, P)
        del sm
        # forward
        m2 = torch.where(seen, s2, -math.inf).amax(-1, keepdim=True)
        mx = torch.where(seen, s2.abs(), 0.0).amax(-1, keepdim=True)
        x = torch.where(seen, s2 - torch.where(none, 0.0, m2), 0.0)
        rho = torch.where(seen, LN2 * (C2 * E_s + EPS_C2 * s2.abs() + U * x.abs()) + EX2, torch.where(none, EX2, 0.0))
        ea = (nkv - 1) * (6 * U + 2 * LN2 * U * mx)
        w = P * kf * sc64
        lam = (P * rho).sum(-1, keepdim=True) + gamma(34 * nkv + 2) + ea
        c64 = ref
        E_ctx = ((w * (rho + d_sc + U + UB + ea) + TINY) @ vv.abs() + (C_ACC * 128 + 2 * nkv) * U * (w @ vv.abs())
                 + (lam + 2 * U) * c64.abs())
        ck = heads(ctx[rows], n, S, nh)
        v.within("ctx", ck, c64, UB * c64.abs() + (1 + UB) * slack * E_ctx, b0)
        # lse: rows with a visible key within their bound; the others below -1e38
        lk = lse[b0:b1].double()
        lt = lse_t[..., 0]
        vis_row = ~none[..., 0].expand(n, nh, S)
        lt0 = torch.where(vis_row, lt, 0.0)
        E_lse = lam[..., 0] + LN2 * (2 * U * math.log2(S) + U * (lt0 * math.log2(math.e)).abs()) + (U + EPS_LN2) * lt0.abs()
        v.within("lse", lk, torch.where(vis_row, lse64, 0.0), slack * E_lse, b0, where=vis_row)
        v.require("lse of rows with no visible key", ~vis_row & ~(lk < -1e38), "not below -1e38")
        del x, rho, E_ctx
        # backward, from the kernel's own lse and ctx
        lse2 = (lse[b0:b1].float() * LOG2E_32).double()[..., None]
        d2 = torch.where(vis_row[..., None], lse2 - lse_t * math.log2(math.e), 0.0)
        xb = torch.where(seen, s2 - torch.where(none, 0.0, lse2), 0.0)
        rho_b = torch.where(seen, LN2 * (C2 * E_s + EPS_C2 * s2.abs() + d2.abs() + U * xb.abs()) + EX2,
                            torch.where(none, EX2 + LN2 * 2 * U * math.log2(S), 0.0))
        del xb, s2, E_s, s
        E_dv = ((w * (rho_b + d_sc + U + UB) + TINY).transpose(-1, -2) @ do.abs()
                + C_ACC * S * U * (w.transpose(-1, -2) @ do.abs()))
        keep_bound = lambda i, bound: grad_bounds[rows, i * H:(i + 1) * H].copy_(
            bound.transpose(1, 2).reshape(n * S, H)) if grad_bounds is not None else None
        bound = UB * gv.abs() + (1 + UB) * slack * E_dv
        v.within("dV", heads(dqkv[rows, 2 * H:], n, S, nh), gv, bound, b0)
        keep_bound(2, bound)
        del w, E_dv
        dp = do @ vv.transpose(-1, -2)
        E_dp = C_ACC * 64 * U * (do.abs() @ vv.abs().transpose(-1, -2))
        delta = (c64 * do).sum(-1, keepdim=True)
        d_delta = ((ck - c64) * do).sum(-1, keepdim=True).abs() + gamma(64) * (ck.abs() * do.abs()).sum(-1, keepdim=True)
        A = kf * sc64 * dp - delta
        E_A = kf * (sc32 * E_dp + d_sc * sc64 * dp.abs()) + d_delta + 2 * U * (kf * sc32 * dp.abs() + delta.abs())
        del dp, E_dp
        dS = 0.125 * P * A
        E_ds = UB * dS.abs() + (1 + UB) * 0.125 * P * (E_A + (rho_b + U) * A.abs()) + TINY
        del A, E_A, rho_b, P
        DS = dS.abs() + E_ds
        E_dk = E_ds.transpose(-1, -2) @ q.abs() + C_ACC * S * U * (DS.transpose(-1, -2) @ q.abs())
        bound = UB * gk.abs() + (1 + UB) * slack * E_dk
        v.within("dK", heads(dqkv[rows, H:2 * H], n, S, nh), gk, bound, b0)
        keep_bound(1, bound)
        del E_dk
        E_dq = E_ds @ k.abs() + (C_ACC * 128 + (nkv if nkv > 1 else 0)) * U * (DS @ k.abs())
        bound = UB * gq.abs() + (1 + UB) * slack * E_dq
        v.within("dQ", heads(dqkv[rows, :H], n, S, nh), gq, bound, b0)
        keep_bound(0, bound)
        del E_ds, DS, E_dq, dS
    if dbias is not None:
        d = dqkv.double()
        c = c0.double()
        E = slack * gamma(4 + 8 * B) * (c.abs() + d.abs().sum(0))
        v.within("dbias", dbias.view(1, 3, nh, 64), (c + d.sum(0)).view(1, 3, nh, 64), E.view(1, 3, nh, 64))
    return v.finish()


# ---- the kernels' rounding sequence in torch (any device, no GPU needed) --------------------------------------------
def kernel_emulation(qkv, dctx, vis, B, S, nh, p, keep, c0=None, defect=None):
    """fp32 arithmetic with bf16 roundings where attention_fwd(128)_kernel / attention_bwd(128)_kernel round: the key
    blocks of 128 with the online rescale, the P tile, ctx, lse, the backward's P and dS tiles, dQ summed over key
    blocks, the outputs.  `vis` is the visibility the emulated kernel applies.  defect = (kind, where) plants one
    mistake: "flip_keep" (b, h, q, k) in the backward only, "lse" (b, h, q) + 1e-3 on the stored lse, "dq_block"
    (b, h, query block, key block) left out of dQ, "no_scale" (dS without the 0.125).  Returns ctx, lse, dqkv, dbias."""
    kind, at = defect if defect is not None else (None, None)
    dev, H = qkv.device, nh * 64
    hf = lambda t: t.float().view(B, S, nh, 64).transpose(1, 2)
    q, k, v = (hf(qkv[:, i * H:(i + 1) * H]) for i in range(3))
    do = hf(dctx)
    vis4 = (vis[:, None] if vis is not None else torch.ones(B, 1, S, S, dtype=torch.bool, device=dev)).expand(
        B, nh, S, S)
    kf = keep if keep is not None else torch.ones(B, nh, S, S, dtype=torch.bool, device=dev)
    sc = drop_scale(p)
    fma = lambda a, b, c: (a.double() * b + c.double()).float()      # one rounding: a * b is exact in float64
    s = q @ k.transpose(-1, -2)
    m = torch.full((B, nh, S, 1), -math.inf, device=dev)
    l = torch.zeros(B, nh, S, 1, device=dev)
    o = torch.zeros(B, nh, S, 64, device=dev)
    for j in range(S // 128):
        cols = slice(128 * j, 128 * j + 128)
        sj, vj = s[..., cols], vis4[..., cols]
        mb = torch.clamp_min(torch.where(vj, sj, -math.inf).amax(-1, keepdim=True) * C2, MASK_BIAS)
        m_new = torch.maximum(m, mb)
        alpha = torch.exp2(m - m_new)
        x = torch.where(vj, fma(sj, C2, -m_new), MASK_BIAS - m_new)
        pr = torch.exp2(x)
        l = l * alpha + pr.sum(-1, keepdim=True)
        pt = torch.where(kf[..., cols], (pr * sc).to(bf).float(), 0.0)
        o = o * alpha + pt @ v[..., cols, :]
        m = m_new
    ctx = (o * (1.0 / l)).to(bf)
    lse = (m + torch.log2(l)) * LN2_32
    if kind == "lse":
        lse[at] += 1e-3
    # backward
    kb = kf.clone()
    if kind == "flip_keep":
        kb[at] = ~kb[at]
    lse2 = lse * LOG2E_32
    xm = torch.where(lse2 < 0.5 * MASK_BIAS, -float(np.log2(np.float32(S), dtype=np.float32)), MASK_BIAS - lse2)
    pr = torch.exp2(torch.where(vis4, fma(s, C2, -lse2), xm))
    dp = do @ v.transpose(-1, -2)
    delta = (ctx.float() * do).sum(-1, keepdim=True)
    pd = torch.where(kb, (pr * sc).to(bf).float(), 0.0)
    dpv = torch.where(kb, dp * sc, 0.0)
    ds = pr * (dpv - delta)
    ds = (ds if kind == "no_scale" else ds * 0.125).to(bf).float()
    dv = pd.transpose(-1, -2) @ do
    dk = ds.transpose(-1, -2) @ q
    dq = torch.zeros(B, nh, S, 64, device=dev)
    for j in range(S // 128):
        part = ds[..., 128 * j:128 * j + 128] @ k[..., 128 * j:128 * j + 128, :]
        if kind == "dq_block" and at[3] == j:
            part[at[0], at[1], 128 * at[2]:128 * at[2] + 128] = 0.0
        dq = dq + part
    flat = lambda t: t.transpose(1, 2).reshape(B * S, H).to(bf)
    dqkv = torch.cat([flat(dq), flat(dk), flat(dv)], 1)
    dbias = c0 + dqkv.float().sum(0) if c0 is not None else None
    return flat(ctx.float()), lse[..., 0], dqkv, dbias


# ---- GPU: the kernels ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def attn_ctas(cap):
    """B2_DEBUG_ATTN_CTAS = cap for the persistent seq-128 backward (None: the default grid)"""
    old = os.environ.pop("B2_DEBUG_ATTN_CTAS", None)
    try:
        if cap is not None:
            os.environ["B2_DEBUG_ATTN_CTAS"] = str(cap)
        yield
    finally:
        os.environ.pop("B2_DEBUG_ATTN_CTAS", None)
        if old is not None:
            os.environ["B2_DEBUG_ATTN_CTAS"] = old


def run_and_check(case, dev, B, S, nh, p, scale, mask=None, seg=None, cap=None, seed=0):
    torch.manual_seed(seed)
    H = nh * 64
    qkv = (torch.randn(B * S, 3 * H, device=dev) * scale).to(bf)
    dctx = torch.randn(B * S, H, device=dev).to(bf)
    kb = torch.zeros(B * nh * S * (S // 64), dtype=torch.int64, device=dev) if S == 128 else None
    c0 = torch.randn(3 * H, device=dev) if S == 128 else None
    db = c0.clone() if c0 is not None else None
    with attn_ctas(cap):
        ctx, lse = attn_fwd(qkv, B, S, nh, p, mask, seg, kb)
        dqkv = attn_bwd(qkv, ctx, dctx, lse, B, S, nh, p, mask, seg, kb, db)
        torch.cuda.synchronize()
    vis = packed_visibility(seg) if seg is not None else padded_visibility(mask, S)
    keep = attn_keep_mask(B, nh, S, SEED, STEP, SITE, p, dev)
    check_outputs(case, qkv, dctx, vis, B, S, nh, p, keep, ctx, lse, dqkv, db, c0).assert_ok()


SWEEP = [(S, p, sc) for S in (128, 256, 384, 512) for p in (0.0, 0.1) for sc in (1, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("S,p,scale", SWEEP, ids=lambda x: str(x))
def test_padded_vs_float64(cuda_dev, S, p, scale):
    mask = padded_masks(S, seed=S).to(cuda_dev)
    run_and_check("padded S=%d p=%g x%d" % (S, p, scale), cuda_dev, mask.shape[0], S, 4, p, scale, mask=mask,
                  seed=S + int(10 * p) + scale)


@pytest.mark.gpu
@pytest.mark.parametrize("p,scale", [(0.0, 1), (0.1, 1), (0.0, 4), (0.1, 4)])
def test_packed_vs_float64(cuda_dev, p, scale):
    seg = packed_layout().to(cuda_dev)
    run_and_check("packed p=%g x%d" % (p, scale), cuda_dev, seg.shape[0], 128, 4, p, scale, seg=seg,
                  seed=11 + int(10 * p) + scale)


ENGINE = [("config_a", 32, 12, 128, None), ("config_a", 32, 12, 128, 1), ("config_a", 32, 12, 128, 7),
          ("config_b", 16, 12, 512, None), ("bert_large", 16, 16, 128, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINE, ids=lambda e: "%s-ctas%s" % (e[0], e[4]))
def test_engine_sizes_vs_float64(cuda_dev, engine):
    """the training step's shapes at p = 0.1; config A also with the persistent backward's grid capped"""
    name, B, nh, S, cap = engine
    rows = padded_masks(S, B, seed=B + S)
    pick = torch.randperm(rows.shape[0], generator=torch.Generator().manual_seed(S))[:B]
    run_and_check("%s ctas=%s" % (name, cap), cuda_dev, B, S, nh, 0.1, 1, mask=rows[pick].to(cuda_dev), cap=cap,
                  seed=B * nh)


# ---- CPU: the checker against the emulated kernels -------------------------------------------------------------------
def cpu_case(S, p, scale, packed=False, nh=2, seed=0):
    torch.manual_seed(seed)
    if packed:
        seg = packed_layout()
        B, vis, mask = seg.shape[0], packed_visibility(seg), None
    else:
        seg, mask = None, padded_masks(S, seed=S)
        B, vis = mask.shape[0], padded_visibility(mask, S)
    H = nh * 64
    qkv = (torch.randn(B * S, 3 * H) * scale).to(bf)
    dctx = torch.randn(B * S, H).to(bf)
    keep = attn_keep_mask(B, nh, S, SEED, STEP, SITE, p)
    c0 = torch.randn(3 * H) if S == 128 else None
    return dict(qkv=qkv, dctx=dctx, vis=vis, B=B, S=S, nh=nh, p=p, keep=keep, c0=c0, seg=seg, mask=mask)


def emulate_and_check(case, c, vis=None, defect=None, slack=SLACK):
    ctx, lse, dqkv, dbias = kernel_emulation(c["qkv"], c["dctx"], c["vis"] if vis is None else vis, c["B"], c["S"],
                                             c["nh"], c["p"], c["keep"], c["c0"], defect)
    return check_outputs(case, c["qkv"], c["dctx"], c["vis"], c["B"], c["S"], c["nh"], c["p"], c["keep"], ctx, lse,
                         dqkv, dbias, c["c0"], slack)


CLEAN = [(128, 0.1, 1, False), (128, 0.0, 4, False), (384, 0.1, 4, False), (512, 0.1, 1, False),
         (128, 0.1, 4, True), (128, 0.0, 1, True)]


@pytest.mark.parametrize("S,p,scale,packed", CLEAN, ids=lambda x: str(x))
def test_clean_emulation_passes(S, p, scale, packed):
    c = cpu_case(S, p, scale, packed, seed=S + scale)
    what = "emulation %s S=%d p=%g x%d" % ("packed" if packed else "padded", S, p, scale)
    emulate_and_check(what, c).assert_ok()


def strongest_key(c, b, h, row):
    """the visible, kept key of a row with the largest score"""
    H = c["nh"] * 64
    q = c["qkv"][b * c["S"] + row, h * 64:(h + 1) * 64].double()
    k = c["qkv"][b * c["S"]:(b + 1) * c["S"], H + h * 64:H + (h + 1) * 64].double()
    ok = c["vis"][b, row] & (c["keep"][b, h, row] if c["keep"] is not None else True)
    return int(torch.where(ok, k @ q, -math.inf).argmax())


def planted(kind):
    """(case, vis for the emulated kernel or None, defect) for one planted defect"""
    if kind == "dq_block_missing":
        c = cpu_case(512, 0.1, 1, seed=5)
        b = int((c["mask"].sum(1) == 512).nonzero()[0])       # a row that sees every key
        return c, None, ("dq_block", (b, 1, 2, 1))
    if kind in ("segment_edge_plus1", "segment_edge_minus1"):
        c = cpu_case(128, 0.1, 1, packed=True, seed=6)
        seg = c["seg"].clone()
        b = seg.shape[0] - 3                       # contiguous([1, 31, 1, 33, 62]): row 1 starts a 31-token segment
        lo, hi = int(seg[b, 1]) & 0xffff, int(seg[b, 1]) >> 16
        seg[b, 1] = lo | ((hi + (1 if kind.endswith("plus1") else -1)) << 16)
        return c, packed_visibility(seg), None
    c = cpu_case(128, 0.1, 1, seed=7)
    vis = c["vis"].clone()
    b0 = int((c["mask"].sum(1) == 128).nonzero()[0])          # a row that sees every key
    if kind == "visible_key_dropped":
        vis[b0, 5, strongest_key(c, b0, 0, 5)] = False
        return c, vis, None
    if kind == "masked_key_admitted":
        b = int((c["mask"].sum(1) == 33).nonzero()[0])         # prefix of 33: key 33 is masked
        vis[b, 40, 33] = True
        return c, vis, None
    if kind == "keep_bit_flipped_in_backward":
        return c, None, ("flip_keep", (b0, 1, 9, strongest_key(c, b0, 1, 9)))
    if kind == "lse_off_by_1e-3":
        return c, None, ("lse", (b0, 0, 17))
    if kind == "ds_without_scale":
        return c, None, ("no_scale", None)
    raise KeyError(kind)


DEFECTS = ["visible_key_dropped", "masked_key_admitted", "keep_bit_flipped_in_backward", "lse_off_by_1e-3",
           "segment_edge_plus1", "segment_edge_minus1", "dq_block_missing", "ds_without_scale"]


@pytest.mark.parametrize("kind", DEFECTS)
def test_planted_defect_is_caught(kind):
    c, vis, defect = planted(kind)
    v = emulate_and_check("planted " + kind, c, vis, defect)
    assert v.bad, "planted defect %s passed every check: %s" % (kind, v.worst)
    report(TAG, {"case": "planted " + kind, "caught_by": v.bad})
    print("caught %s: %s" % (kind, v.bad[0]))


# ---- dropout rates the entry points reject: no GPU needed --------------------------------------------------------------
# Made-up addresses, never dereferenced, in a child process that sees no device: a build without the check fails on
# "no device" (or launches) instead of naming dropout_p.
_P_CHILD = r"""
import ctypes, importlib.util, json, sys
spec = importlib.util.spec_from_file_location("b2_lib_child", sys.argv[1])
L = importlib.util.module_from_spec(spec)
spec.loader.exec_module(L)
lib = L.load()
a = [(1 << 24) + i * 0x100000 for i in range(10)]   # qkv, mask/seg, ctx, d_ctx, lse, rng, keep_bits, d_qkv, dbias
out = {}
for entry, p in json.loads(sys.argv[2]):
    if entry == "fwd":
        st = lib.b2_attention_fwd(a[0], a[1], 2, 128, 4, 64, p, a[5], 4, a[2], a[4], a[6], None)
    elif entry == "fwd_packed":
        st = lib.b2_attention_fwd_packed(a[0], a[1], 2, 4, 64, p, a[5], 4, a[2], a[4], a[6], None)
    elif entry == "bwd":
        st = lib.b2_attention_bwd(a[0], a[1], a[2], a[3], a[4], 2, 128, 4, 64, p, a[5], 4, a[7], None, a[8], a[6], None)
    else:
        st = lib.b2_attention_bwd_packed(a[0], a[1], a[2], a[3], a[4], 2, 4, 64, p, a[5], 4, a[7], a[8], a[6], None)
    out["%s %r" % (entry, p)] = [int(st), L.last_error()]
print(json.dumps(out))
"""
ENTRIES = ["fwd", "fwd_packed", "bwd", "bwd_packed"]
BAD_P = [-0.1, float("nan"), 1.0, 1.5, float("inf")]
GOOD_P = [0.0, 0.1, 0.9]


@pytest.fixture(scope="module")
def p_results():
    env = dict(os.environ)
    env["CUDA_VISIBLE_DEVICES"] = ""
    lib_py = os.path.join(ROOT, "pytorch-distributed-nlp_b200", "_lib.py")
    calls = [(e, p) for e in ENTRIES for p in BAD_P + GOOD_P]
    r = subprocess.run([sys.executable, "-c", _P_CHILD, lib_py, json.dumps(calls)], env=env, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("p", BAD_P, ids=repr)
@pytest.mark.parametrize("entry", ENTRIES)
def test_dropout_p_out_of_range_is_rejected(p_results, entry, p):
    st, err = p_results["%s %r" % (entry, p)]
    assert st != 0 and "dropout_p out of range" in err, err


@pytest.mark.parametrize("p", GOOD_P, ids=repr)
@pytest.mark.parametrize("entry", ENTRIES)
def test_dropout_p_in_range_passes_the_check(p_results, entry, p):
    """the same calls with p in [0, 1) get past the argument checks (and then fail for want of a device)"""
    st, err = p_results["%s %r" % (entry, p)]
    assert st != 0 and "dropout_p" not in err and "null" not in err and "seq=" not in err, err
