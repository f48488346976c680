"""The wgmma GEMM (b2_gemm_bf16, b2_gemm_bf16_grouped) element-wise against its own fp32 accumulator and float64, in
every form the training step issues, and the argument combinations it rejects.

Forms covered (modeling._Engine): forward QKV NT/BIAS, FFN1 NT/BIAS_GELU, the unfused NT/BIAS_DROPOUT_RESIDUAL of the
tiny configs; backward the four TN/NONE weight gradients (grouped, and their per-problem split-K fallback),
NN/GELU_BWD + colsum, NN/ACCUM_F32 at auto split, NN/NONE.  Shapes: H in {256, 768, 1024}, I = 4H (tiny: 512),
M = 4096 tokens, weight gradients over up to 16384 tokens; edges M in {1, 127, 129, 200, 4101}, K in {8, 72, 136}
(tails inside one 64-deep k-block), N in {64, 192, 320} with BN 128 and N = 768 with BN 256, the Q and V columns of a
packed QKV as a strided A, forced splits 2, 3, 4, 7, 8 (K = 2304 with 7 splits leaves the last slice no k-block),
auto configuration with and without a workspace, grouped tables of 1-4 ragged problems, an N = 192 member (issued
problem by problem) and 5 problems.

References run in float64 on the GPU from the same bf16 operands (A64, B64).  U = 2^-24 is the fp32 unit roundoff,
UB = 2^-8 the bf16 one (half an ulp, relative); S = |A64| @ |B64|.  Every check asserts error <= bound element-wise,
or bitwise equality, and sends its worst error / bound to parity.report.  The checks come in two layers so that only
one bound rests on how the tensor cores round.

Layer A: the accumulator against float64.  EPI_RESIDUAL_F32 onto an all-zero fp32 residual with one split stores
acc + 0 = acc, the raw fp32 accumulator.  NVIDIA does not document how wgmma rounds its fp32 accumulation, and
published measurements of earlier tensor cores report truncation on alignment rather than round-to-nearest, so the
bound assumes only this model: products of bf16 are exact in fp32; each 16-deep wgmma k-step adds its 16 products
into the accumulator, the 17 terms aligned to the largest, each term losing at most one fp32 ulp of that largest
term (2^-23 |largest| <= 2^-23 S).  Over ceil(K/16) k-steps that is at most (K/16) * 17 * 2^-23 * S = 2.125 K U S
(the padded terms of a K tail are exact zeros), so

    |acc - A64 @ B64| <= E_acc = c K U S,  c = 4.

This is the one assumption about undocumented hardware in this file.  At K <= 1024 with unit-variance operands,
E_acc is about 0.16 sigma_A sigma_B against 0.64 for a typical |a_k b_k|, so one product missing from every element
fails it; at larger K it still catches a missing k-block (64 products), not a single product.  Layer B stays exact
or rounding-tight at every K.

Layer B: every epilogue against its restatement from the kernel's own accumulator.  Same operands, same BN and one
split give the bit-identical accumulator (the mainloop does not depend on the epilogue), so:
  exact    EPI_NONE == bf16(acc); EPI_BIAS == bf16(fp32(acc + bias)); EPI_RESIDUAL == bf16(fp32(acc + aux));
           EPI_ACCUM_F32 with one split onto R == fp32(R + acc) (a red.add of one term rounds to nearest);
           EPI_RESIDUAL_F32 with aux R == fp32(acc + R); aux_out of EPI_BIAS_GELU == bf16(fp32(acc + bias));
           the grouped launch == b2_gemm_bf16 with BN 256 and one split (same mainloop, same EPI_NONE epilogue).
  bounded  (bf_bound(ref, E) = UB |ref| + (1 + UB) E: a bf16 store of an fp32 value within E of ref)
           BIAS_DROPOUT_RESIDUAL, p = 0 and 0.1: ref = keep * t * scale + r with t = fp32(acc + bias) exact, the
             Philox mask keyed by m * N + n, scale = fp32 1/(1-p); E = 2U (|t scale| + |r|) covers the product and
             the sum rounded apart or contracted into one FMA.
           BIAS_GELU output: gelu64 of the kernel's own bf16 aux_out u.  gelu_hq's erf is A&S 7.1.26 (|erf error|
             <= 1.5e-7, so 7.5e-8 on hq = erfc(|u|/sqrt2)/2); ex2.approx of a twice-rounded argument is within
             (u^2 + 4) U relative; rcp.approx, the five polynomial FMAs and their cancellation get a deliberately
             generous 256 U relative on hq.  E = |u| (7.5e-8 + (u^2 + 256) U hq64) + 2U |gelu64|.  Every such term
             is below 2^-16 relative, far under the bf16 rounding that decides the check.
           GELU_BWD: ref = acc * gelu'64(x) from the same ingredients for cdf and x * pdf, plus the product rounding.
           colsum_out (starting from a nonzero C0, so it must be +=): the fp64 column sums of the stored bf16 D;
             each column is a chain of 32 in-warp additions and ceil(M/32) atomics in no fixed order:
             E = gamma(32 + ceil(M/32)) (|C0| + sum |D|), gamma(n) = nU / (1 - nU).
           Split-K EPI_NONE with a workspace: per-slice accumulators within the layer A model (their k-ranges add up
             to K) plus the reduce pass's splits additions: E = (c K + splits) U S, then one bf16 rounding.
           EPI_ACCUM_F32 with 2-8 splits: E = c K U S + splits U (|R| + S), order unspecified.
  untouched  D, aux_out and the fp32 outputs live in buffers with ld > N and guard rows past M, filled with a
           sentinel: nothing outside [M) x [N) changes (the workspace past splits * M * N and colsum past N too), and
           the dropout mask is checked at ld > N, so a mask keyed on ld instead of N fails.

A bounded check fails on any element whose error / bound is not <= 1, so a NaN or inf in an output fails it (the
helpers' own CPU tests at the end show this).

Rejected arguments, which the kernels would otherwise drop without a word: colsum_out with a split, bias or
colsum_out with the fp32-output epilogues, bias with NONE / RESIDUAL / GELU_BWD, dropout_p > 0 outside
BIAS_DROPOUT_RESIDUAL, aux_out outside BIAS_GELU, and misaligned bias / aux_in / aux_out.  The grouped entry point
rejects a table before any problem of it runs.  The alignment checks run in a child process that sees no device, so
a build without them fails on "no device" instead of launching on a misaligned pointer; they need no GPU.  Still
accepted, because the step and the tools pass them: rng_state at p = 0, a workspace on a problem that does not
split, any force_kernel, a debug_timing pointer.

Measured worst error / bound on an H100 80GB HBM3 (700 W power limit), per check family: layer A accumulator 0.060
over 71 shapes (the hardware's accumulation sits far inside the model's bound); every exact check 0 mismatches (100
checks); BIAS_DROPOUT_RESIDUAL D 0.996, GELU_BWD D 0.996, BIAS_GELU D 0.971 (the half-ulp bf16 rounding itself
dominates); colsum_out 0.030; split-K EPI_NONE 0.47; ACCUM_F32 with 2-8 splits and at auto split 0.0018; EPI_NONE at
auto configuration 0.79; grouped tables and their fallback 0.82; the D of the colsum problem kept unsplit 0.27.
Runtime, from one `pytest -m gpu tests/test_gemm_reference.py --durations=0` on that card: 262 tests in 6.7 s as
pytest counts it, 17.9 s of wall time with interpreter and CUDA start-up.  The slowest test is the first (1.5 s,
mostly CUDA and cuBLAS initialisation), then the p = 0.1 dropout forms (up to 0.6 s each: their Philox mask is
computed on the CPU); the float64 products, up to 1024 x 1024 x 16384, take milliseconds on the GPU.
With B2_PARITY_REPORT set, every check appends its ratio there (tag "gemm_reference").
"""
import json
import math
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

from parity import philox_keep_mask, report
from pytorch_distributed_nlp_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
bf, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24       # fp32 unit roundoff
UB = 2.0 ** -8       # bf16 unit roundoff
C_ACC = 4.0          # layer A: |acc - A64 @ B64| <= C_ACC * K * U * S
SEED, STEP = 4321, 7
SENT = -3.0          # sentinel: exactly representable in bf16 and fp32
KM, MN = L.MAJOR_K, L.MAJOR_MN
LAYOUTS = {"NT": (KM, KM), "NN": (KM, MN), "TN": (MN, MN)}
SQRT1_2 = 1.0 / math.sqrt(2.0)
AS_HQ = 7.5e-8       # A&S 7.1.26: |erf error| <= 1.5e-7, halved in hq


def stream():
    return torch.cuda.current_stream().cuda_stream


def gamma(n):
    return n * U / (1 - n * U)


def drop_scale(p):
    """the kernel's 1/(1-p), computed in fp32"""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p))) if p > 0 else 1.0


def within(got, ref, bound, family, what, tag="gemm_reference"):
    """element-wise |got - ref| <= bound; the worst ratio goes to the parity report under `tag`.  Anything that is not
    <= 1 fails, so a NaN (or inf) in the output fails too."""
    err = (got.double() - ref).abs()
    ratio = err / bound.clamp_min(1e-300)
    worst = float(ratio.max()) if err.numel() else 0.0      # NaN if any element is NaN
    report(tag, {"family": family, "check": what, "err_over_bound": worst})
    bad = ~(ratio <= 1.0)
    if bool(bad.any()):
        nan = torch.isnan(ratio)
        flat = int(nan.flatten().nonzero()[0]) if bool(nan.any()) else int(ratio.argmax())
        idx = tuple(int(i) for i in np.unravel_index(flat, tuple(ratio.shape)))
        raise AssertionError("%s: worst error is %.3g x its bound at %s (got %r, ref %r, %d elements over, %d NaN)" % (
            what, worst, idx, float(got[idx]), float(ref[idx]), int(bad.sum()), int(nan.sum())))


def same(got, ref, family, what, tag="gemm_reference"):
    """bitwise, up to the sign of zero"""
    bad = got != ref
    n = int(bad.sum())
    report(tag, {"family": family, "check": what, "mismatches": n})
    if n:
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d elements differ, first at %s (got %r, ref %r)" % (
            what, n, idx, float(got[idx]), float(ref[idx])))


def bf_bound(ref, E):
    """bound for a bf16 store of an fp32 value within E of ref"""
    return UB * ref.abs() + (1 + UB) * E


def guarded(rows, cols, dtype, dev, pad=8, extra_rows=3):
    """[rows + extra_rows, cols + pad] of SENT: an output lives in its [:rows, :cols] corner, ld = cols + pad"""
    return torch.full((rows + extra_rows, cols + pad), SENT, dtype=dtype, device=dev), cols + pad


def untouched(buf, rows, cols, what):
    outside = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    outside[:rows, :cols] = False
    n = int((buf[outside] != SENT).sum())
    assert n == 0, "%s: %d elements outside [%d) x [%d) were written" % (what, n, rows, cols)


def padded_input(rows, cols, dtype, dev, gen, scale=1.0, pad=8):
    """an input [rows, cols] inside a wider buffer (ld = cols + pad)"""
    buf = (torch.randn(rows, cols + pad, device=dev, generator=gen) * scale).to(dtype)
    return buf[:, :cols], cols + pad


_RNG = {}


def rng_state(dev):
    if dev not in _RNG:
        _RNG[dev] = torch.tensor([SEED, STEP], dtype=torch.int64, device=dev)
    return _RNG[dev]


class Ops:
    """bf16 operands of D[M, N] = A[M, K] @ B[K, N] stored in one of the three layouts, and their fp64 values.
    a_cols = (offset, width): A is the columns [offset, offset + K) of a packed [M, width] activation (K-major A)."""

    def __init__(self, layout, M, N, K, dev, seed, a_cols=None):
        self.layout, self.M, self.N, self.K, self.dev = layout, M, N, K, dev
        self.am, self.bm = LAYOUTS[layout]
        gen = torch.Generator(device=dev).manual_seed(seed)
        if a_cols is not None:
            assert self.am == KM
            off, width = a_cols
            big = torch.randn(M, width, device=dev, generator=gen).to(bf)
            A = big[:, off:off + K]
            self.A_store, self.lda = A, width
        else:
            A = torch.randn(M, K, device=dev, generator=gen).to(bf)
            if self.am == KM:
                self.A_store, self.lda = A, K
            else:
                assert M % 8 == 0
                self.A_store, self.lda = A.t().contiguous(), M
        B = (torch.randn(K, N, device=dev, generator=gen) / math.sqrt(K)).to(bf)
        self.B_store, self.ldb = (B.t().contiguous(), K) if self.bm == KM else (B, N)
        self.a64, self.b64 = A.double(), B.double()
        self._exact = None
        self.gen = gen

    def exact(self):
        """(A64 @ B64, S = |A64| @ |B64|)"""
        if self._exact is None:
            self._exact = (self.a64 @ self.b64, self.a64.abs() @ self.b64.abs())
        return self._exact


def gemm_args(ops, D, ldd, epi=L.EPI_NONE, bn=0, splits=1, bias=None, aux_in=None, ld_aux_in=0, aux_out=None,
              ld_aux_out=0, p=0.0, site=0, rng=True, ws=None, colsum=None, kernel=0, timing=None):
    a = L.GemmArgs()
    a.M, a.N, a.K = ops.M, ops.N, ops.K
    a.A, a.lda, a.a_major = ops.A_store.data_ptr(), ops.lda, ops.am
    a.B, a.ldb, a.b_major = ops.B_store.data_ptr(), ops.ldb, ops.bm
    a.D, a.ldd, a.epilogue = D.data_ptr(), ldd, epi
    a.bias = L.ptr(bias)
    a.aux_in, a.ld_aux_in = L.ptr(aux_in), ld_aux_in
    a.aux_out, a.ld_aux_out = L.ptr(aux_out), ld_aux_out
    # the step always hands the GEMM its dropout stream, whatever the epilogue
    a.dropout_p, a.rng_state, a.rng_site = p, (rng_state(ops.dev).data_ptr() if rng else None), site
    a.workspace, a.workspace_bytes = L.ptr(ws), (ws.numel() * ws.element_size() if ws is not None else 0)
    a.force_bn, a.force_splits, a.force_kernel = bn, splits, kernel
    a.debug_timing = L.ptr(timing)
    a.colsum_out = L.ptr(colsum)
    return a


def gemm(ops, D, ldd, **kw):
    L.call("b2_gemm_bf16", gemm_args(ops, D, ldd, **kw), stream())
    torch.cuda.synchronize()


def accumulator(ops, bn):
    """the kernel's raw fp32 accumulator: EPI_RESIDUAL_F32 onto an all-zero fp32 residual, one split"""
    M, N = ops.M, ops.N
    buf, ld = guarded(M, N, f32, ops.dev)
    zero = torch.zeros(M, N, dtype=f32, device=ops.dev)
    gemm(ops, buf, ld, epi=L.EPI_RESIDUAL_F32, bn=bn, splits=1, aux_in=zero, ld_aux_in=N)
    untouched(buf, M, N, "accumulator (RESIDUAL_F32) output")
    return buf[:M, :N].clone()


def case_id(c):
    layout, bn, M, N, K = c[:5]
    s = "%s-bn%d-%dx%dx%d" % (layout, bn, M, N, K)
    if len(c) > 5 and c[5] is not None:
        s += "-cols%d+%d" % c[5]
    return s


# ======================================================================================================================
# Layer A: the accumulator against float64
# ======================================================================================================================
ENGINE_SHAPES = [
    ("NT", 4096, 2304, 768),     # QKV projection, H 768
    ("NT", 4096, 3072, 768),     # FFN1, H 768
    ("NT", 4096, 768, 3072),     # FFN2 (unfused dense + dropout + residual), H 768
    ("NT", 4096, 1024, 4096),    # FFN2, H 1024
    ("NT", 4096, 512, 256),      # tiny FFN1
    ("NT", 4096, 768, 256),      # tiny QKV
    ("NN", 4096, 3072, 768),     # dU = dY2 W2 (GELU_BWD)
    ("NN", 4096, 768, 3072),     # dX1 += dU W1 (ACCUM_F32)
    ("NN", 4096, 1024, 1024),    # dctx = dZ1 Wo, H 1024
    ("NN", 4096, 256, 768),      # tiny dX += dQKV Wqkv
    ("TN", 768, 3072, 4096),     # FFN2 weight gradient
    ("TN", 3072, 768, 4096),     # FFN1 weight gradient
    ("TN", 2304, 768, 4096),     # QKV weight gradient
    ("TN", 1024, 1024, 16384),   # attention-output weight gradient, H 1024, 16384 tokens
    ("TN", 256, 512, 4096),      # tiny FFN2 weight gradient
]
ACC_CASES = [(lay, bn, M, N, K, None) for (lay, M, N, K) in ENGINE_SHAPES for bn in (128, 256)]
ACC_CASES += [("NT", bn, M, 768, 768, None) for M in (1, 127, 129, 200, 4101) for bn in (128, 256)]
ACC_CASES += [("NN", 256, M, 768, 1024, None) for M in (1, 200, 4101)]
ACC_CASES += [("TN", bn, 328, 768, 1024, None) for bn in (128, 256)]
ACC_CASES += [(lay, 128, 512, 768, K, None) for lay in ("NT", "NN", "TN") for K in (8, 72, 136)]
ACC_CASES += [("NT", 256, 512, 768, K, None) for K in (8, 72, 136)]
ACC_CASES += [(lay, 128, 328 if lay == "TN" else 300, N, 200, None) for lay in ("NT", "NN", "TN")
              for N in (64, 192, 320)]
ACC_CASES += [("NT", bn, 512, 768, 768, cols) for cols in ((0, 2304), (1536, 2304)) for bn in (128, 256)]
ACC_CASES += [("NN", 128, 512, 768, 768, (0, 2304))]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ACC_CASES, ids=case_id)
def test_accumulator_vs_float64(cuda_dev, case):
    layout, bn, M, N, K, cols = case
    ops = Ops(layout, M, N, K, cuda_dev, seed=zlib.crc32(case_id(case).encode()), a_cols=cols)
    acc = accumulator(ops, bn)
    ref, S = ops.exact()
    within(acc, ref, C_ACC * K * U * S, "A accumulator", "accumulator " + case_id(case))


# ======================================================================================================================
# Layer B: every epilogue against its restatement from the kernel's own accumulator
# ======================================================================================================================
def gelu64(x):
    return 0.5 * x * torch.erfc(-x * SQRT1_2)


def hq64(x):
    return 0.5 * torch.erfc(x.abs() * SQRT1_2)


def gelu_err(x):
    """bound on |gelu_erf(x) - gelu64(x)| for the kernel's fp32 gelu_erf"""
    return x.abs() * (AS_HQ + (x * x + 256) * U * hq64(x)) + 2 * U * gelu64(x).abs()


def gelu_grad64(x):
    return 0.5 * torch.erfc(-x * SQRT1_2) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def gelu_grad_err(x):
    """bound on |gelu_erf_grad(x) - gelu_grad64(x)|: cdf from hq (plus the 1 - hq rounding), x * pdf from the same
    exp, one FMA"""
    xpdf = (x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)).abs()
    return AS_HQ + (x * x + 256) * U * hq64(x) + U + xpdf * (x * x + 8) * U + U * gelu_grad64(x).abs()


def form_none(ops, bn, acc):
    M, N = ops.M, ops.N
    D, ld = guarded(M, N, bf, ops.dev)
    gemm(ops, D, ld, epi=L.EPI_NONE, bn=bn)
    same(D[:M, :N], acc.to(bf), "B exact", "NONE D")
    untouched(D, M, N, "NONE D")


def form_bias(ops, bn, acc):
    M, N = ops.M, ops.N
    bias = torch.randn(N, device=ops.dev, generator=ops.gen).to(bf)
    D, ld = guarded(M, N, bf, ops.dev)
    gemm(ops, D, ld, epi=L.EPI_BIAS, bn=bn, bias=bias)
    same(D[:M, :N], (acc + bias.float()).to(bf), "B exact", "BIAS D")
    untouched(D, M, N, "BIAS D")


def form_residual(ops, bn, acc):
    M, N = ops.M, ops.N
    R, ldr = padded_input(M, N, bf, ops.dev, ops.gen)
    D, ld = guarded(M, N, bf, ops.dev)
    gemm(ops, D, ld, epi=L.EPI_RESIDUAL, bn=bn, aux_in=R, ld_aux_in=ldr)
    same(D[:M, :N], (acc + R.float()).to(bf), "B exact", "RESIDUAL D")
    untouched(D, M, N, "RESIDUAL D")


def form_bias_gelu(ops, bn, acc):
    M, N = ops.M, ops.N
    bias = torch.randn(N, device=ops.dev, generator=ops.gen).to(bf)
    D, ld = guarded(M, N, bf, ops.dev)
    Ub, ldu = guarded(M, N, bf, ops.dev, pad=16)
    gemm(ops, D, ld, epi=L.EPI_BIAS_GELU, bn=bn, bias=bias, aux_out=Ub, ld_aux_out=ldu)
    u = Ub[:M, :N]
    same(u, (acc + bias.float()).to(bf), "B exact", "BIAS_GELU aux_out")
    untouched(Ub, M, N, "BIAS_GELU aux_out")
    x = u.double()
    ref = gelu64(x)
    within(D[:M, :N], ref, bf_bound(ref, gelu_err(x)), "B BIAS_GELU D", "BIAS_GELU D")
    untouched(D, M, N, "BIAS_GELU D")


def form_bias_dropout_residual(p):
    def run(ops, bn, acc):
        M, N = ops.M, ops.N
        site = 5
        bias = torch.randn(N, device=ops.dev, generator=ops.gen).to(bf)
        R, ldr = padded_input(M, N, bf, ops.dev, ops.gen)
        D, ld = guarded(M, N, bf, ops.dev)
        gemm(ops, D, ld, epi=L.EPI_BIAS_DROPOUT_RESIDUAL, bn=bn, bias=bias, aux_in=R, ld_aux_in=ldr, p=p, site=site)
        t = (acc + bias.float()).double()                       # the kernel's fp32 acc + bias, exactly
        keep = torch.from_numpy(philox_keep_mask(M * N, SEED, STEP, site, p).reshape(M, N)).to(ops.dev)
        ts = t * keep.double() * drop_scale(p)
        r = R.double()
        ref = ts + r
        within(D[:M, :N], ref, bf_bound(ref, 2 * U * (ts.abs() + r.abs())), "B BIAS_DROPOUT_RESIDUAL D",
               "BIAS_DROPOUT_RESIDUAL p=%g D" % p)
        untouched(D, M, N, "BIAS_DROPOUT_RESIDUAL D")
    return run


def form_gelu_bwd_colsum(ops, bn, acc):
    M, N = ops.M, ops.N
    Ui, ldu = padded_input(M, N, bf, ops.dev, ops.gen, scale=2.0)
    c0 = torch.randn(N, device=ops.dev, generator=ops.gen)
    cs = torch.full((N + 8,), SENT, dtype=f32, device=ops.dev)
    cs[:N] = c0
    D, ld = guarded(M, N, bf, ops.dev)
    gemm(ops, D, ld, epi=L.EPI_GELU_BWD, bn=bn, aux_in=Ui, ld_aux_in=ldu, colsum=cs)
    x, a = Ui.double(), acc.double()
    g = gelu_grad64(x)
    ref = a * g
    within(D[:M, :N], ref, bf_bound(ref, a.abs() * gelu_grad_err(x) + U * ref.abs()), "B GELU_BWD D", "GELU_BWD D")
    untouched(D, M, N, "GELU_BWD D")
    d = D[:M, :N].double()
    ref_cs = c0.double() + d.sum(0)
    e_cs = gamma(32 + -(-M // 32)) * (c0.double().abs() + d.abs().sum(0))
    within(cs[:N], ref_cs, e_cs, "B colsum", "GELU_BWD colsum_out")
    assert bool((cs[N:] == SENT).all()), "colsum_out written past N"


def form_accum_f32(ops, bn, acc):
    M, N = ops.M, ops.N
    D, ld = guarded(M, N, f32, ops.dev)
    R = torch.randn(M, N, device=ops.dev, generator=ops.gen)
    D[:M, :N] = R
    gemm(ops, D, ld, epi=L.EPI_ACCUM_F32, bn=bn, splits=1)
    same(D[:M, :N], R + acc, "B exact", "ACCUM_F32 one split D")
    untouched(D, M, N, "ACCUM_F32 D")


def form_residual_f32(ops, bn, acc):
    M, N = ops.M, ops.N
    R, ldr = padded_input(M, N, f32, ops.dev, ops.gen)
    D, ld = guarded(M, N, f32, ops.dev)
    gemm(ops, D, ld, epi=L.EPI_RESIDUAL_F32, bn=bn, aux_in=R, ld_aux_in=ldr)
    same(D[:M, :N], acc + R, "B exact", "RESIDUAL_F32 D")
    untouched(D, M, N, "RESIDUAL_F32 D")


FORMS = {
    "none": form_none, "bias": form_bias, "residual": form_residual, "bias_gelu": form_bias_gelu,
    "bias_dropout_residual_p0": form_bias_dropout_residual(0.0),
    "bias_dropout_residual_p0.1": form_bias_dropout_residual(0.1),
    "gelu_bwd_colsum": form_gelu_bwd_colsum, "accum_f32": form_accum_f32, "residual_f32": form_residual_f32,
}
EPI_CASES = [
    ("NT", 256, 4096, 768, 768, None), ("NT", 128, 4096, 3072, 1024, None), ("NT", 256, 4096, 512, 256, None),
    ("NN", 256, 4096, 768, 3072, None), ("NN", 128, 4096, 1024, 4096, None), ("TN", 256, 1024, 4096, 4096, None),
    ("NT", 128, 1, 64, 8, None), ("NT", 128, 127, 192, 72, None), ("NN", 128, 129, 320, 136, None),
    ("NT", 256, 200, 768, 136, None), ("NN", 256, 4101, 768, 768, None), ("TN", 128, 328, 192, 1024, None),
    ("NT", 128, 512, 768, 768, (0, 2304)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", EPI_CASES, ids=case_id)
@pytest.mark.parametrize("form", list(FORMS))
def test_epilogue_vs_own_accumulator(cuda_dev, form, case):
    layout, bn, M, N, K, cols = case
    ops = Ops(layout, M, N, K, cuda_dev, seed=zlib.crc32((form + case_id(case)).encode()), a_cols=cols)
    FORMS[form](ops, bn, accumulator(ops, bn))


# ======================================================================================================================
# split-K and the automatic configuration: against float64
# ======================================================================================================================
def workspace(nbytes, dev):
    """fp32 scratch of nbytes plus a sentinel tail that must stay untouched"""
    return torch.full((nbytes // 4 + 64,), SENT, dtype=f32, device=dev)


def check_fp64_bf16(D, ops, adds, family, what):
    """a bf16 D within (c K + adds) U S of A64 @ B64, then one bf16 rounding"""
    ref, S = ops.exact()
    within(D, ref, bf_bound(ref, (C_ACC * ops.K + adds) * U * S), family, what)


SPLIT_NONE_CASES = [("TN", 256, 768, 768, 2304, None), ("TN", 128, 328, 192, 2304, None),
                    ("NN", 128, 300, 768, 2304, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SPLIT_NONE_CASES, ids=case_id)
@pytest.mark.parametrize("splits", [2, 3, 4, 7, 8])
def test_split_k_partials_and_reduce(cuda_dev, case, splits):
    """EPI_NONE with a workspace, forced splits: fp32 partials per slice, then the reduce pass"""
    layout, bn, M, N, K, _ = case
    ops = Ops(layout, M, N, K, cuda_dev, seed=11 * splits + M)
    ws = workspace(splits * M * N * 4, cuda_dev)
    D, ld = guarded(M, N, bf, cuda_dev)
    before = L.launch_count()
    gemm(ops, D, ld, epi=L.EPI_NONE, bn=bn, splits=splits, ws=ws)
    assert L.launch_count() - before == 2, "split-K is one GEMM launch and one reduce launch"
    check_fp64_bf16(D[:M, :N], ops, splits, "split-K NONE", "split-K %d NONE %s" % (splits, case_id(case)))
    untouched(D, M, N, "split-K D")
    assert bool((ws[splits * M * N:] == SENT).all()), "workspace written past splits * M * N"


ACCUM_SPLIT_CASES = [("NN", 256, 4096, 768, 2304, None), ("NN", 128, 300, 768, 2304, None)]


def check_accum(D, R, ops, adds, what):
    ref, S = ops.exact()
    r = R.double()
    within(D, r + ref, C_ACC * ops.K * U * S + adds * U * (r.abs() + S), "ACCUM_F32 split", what)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ACCUM_SPLIT_CASES, ids=case_id)
@pytest.mark.parametrize("splits", [2, 3, 4, 7, 8])
def test_accum_f32_split_k(cuda_dev, case, splits):
    """EPI_ACCUM_F32 slices adding into D in place, in no fixed order"""
    layout, bn, M, N, K, _ = case
    ops = Ops(layout, M, N, K, cuda_dev, seed=13 * splits + M)
    D, ld = guarded(M, N, f32, cuda_dev)
    R = torch.randn(M, N, device=cuda_dev, generator=ops.gen)
    D[:M, :N] = R
    gemm(ops, D, ld, epi=L.EPI_ACCUM_F32, bn=bn, splits=splits)
    check_accum(D[:M, :N], R, ops, splits, "ACCUM_F32 %d splits %s" % (splits, case_id(case)))
    untouched(D, M, N, "ACCUM_F32 D")


AUTO_CASES = [  # layout, M, N, K, epilogue, with a workspace
    ("TN", 768, 3072, 4096, L.EPI_NONE, True),      # weight gradient issued on its own (the grouped fallback)
    ("TN", 2304, 768, 16384, L.EPI_NONE, True),
    ("TN", 768, 768, 4096, L.EPI_NONE, False),
    ("NN", 4096, 768, 768, L.EPI_NONE, False),      # dctx
    ("NN", 4096, 768, 768, L.EPI_NONE, True),
    ("NN", 4096, 768, 3072, L.EPI_ACCUM_F32, False),  # dX1 += dU W1
    ("NN", 4096, 768, 2304, L.EPI_ACCUM_F32, False),  # dX += dQKV Wqkv
    ("NN", 4096, 1024, 4096, L.EPI_ACCUM_F32, False),
    ("NN", 4096, 256, 512, L.EPI_ACCUM_F32, False),   # tiny
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", AUTO_CASES, ids=lambda c: "%s-%dx%dx%d-epi%d-%s" % (
    c[0], c[1], c[2], c[3], c[4], "ws" if c[5] else "nows"))
def test_auto_configuration(cuda_dev, case):
    """the tile width and split count the library picks itself (up to 8 splits)"""
    layout, M, N, K, epi, with_ws = case
    ops = Ops(layout, M, N, K, cuda_dev, seed=M + N + K)
    ws = workspace(8 * M * N * 4, cuda_dev) if with_ws else None
    if epi == L.EPI_NONE:
        D, ld = guarded(M, N, bf, cuda_dev)
        gemm(ops, D, ld, epi=epi, bn=0, splits=0, ws=ws)
        check_fp64_bf16(D[:M, :N], ops, 8, "auto", "auto NONE %dx%dx%d" % (M, N, K))
    else:
        D, ld = guarded(M, N, f32, cuda_dev)
        R = torch.randn(M, N, device=cuda_dev, generator=ops.gen)
        D[:M, :N] = R
        gemm(ops, D, ld, epi=epi, bn=0, splits=0, ws=ws)
        check_accum(D[:M, :N], R, ops, 8, "auto ACCUM_F32 %dx%dx%d" % (M, N, K))
    untouched(D, M, N, "auto D")
    if ws is not None:
        assert bool((ws[8 * M * N:] == SENT).all())


@pytest.mark.gpu
def test_colsum_output_is_never_split(cuda_dev):
    """an EPI_NONE problem with a workspace that the automatic configuration splits: with colsum_out it must run whole
    tiles (the split-K partials path takes no column sums) and still add every row's column sum"""
    M, N, K = 768, 768, 4096
    ops = Ops("TN", M, N, K, cuda_dev, seed=3)
    ws = workspace(8 * M * N * 4, cuda_dev)
    D, ld = guarded(M, N, bf, cuda_dev)
    before = L.launch_count()
    gemm(ops, D, ld, epi=L.EPI_NONE, bn=0, splits=0, ws=ws)
    assert L.launch_count() - before == 2, "this shape is expected to split without colsum_out"
    c0 = torch.randn(N, device=cuda_dev, generator=ops.gen)
    cs = torch.full((N + 8,), SENT, dtype=f32, device=cuda_dev)
    cs[:N] = c0
    D, ld = guarded(M, N, bf, cuda_dev)
    before = L.launch_count()
    gemm(ops, D, ld, epi=L.EPI_NONE, bn=0, splits=0, ws=ws, colsum=cs)
    launches = L.launch_count() - before
    check_fp64_bf16(D[:M, :N], ops, 0, "colsum unsplit", "NONE + colsum D")
    d = D[:M, :N].double()
    within(cs[:N], c0.double() + d.sum(0), gamma(32 + -(-M // 32)) * (c0.double().abs() + d.abs().sum(0)),
           "B colsum", "NONE + colsum_out with a workspace")
    assert bool((cs[N:] == SENT).all())
    assert launches == 1, "a problem with colsum_out was split"


# ======================================================================================================================
# grouped weight gradients
# ======================================================================================================================
GROUPS = [  # (id, [(M_i, N_i)], K = tokens)
    ("bert-base-layer-16384", [(768, 3072), (3072, 768), (768, 768), (2304, 768)], 16384),
    ("one", [(328, 768)], 4096),
    ("two-ragged", [(456, 256), (1024, 1024)], 4096),
    ("three-ragged-ktail", [(328, 512), (768, 256), (72, 768)], 520),
    ("tiny-layer", [(256, 512), (512, 256), (256, 256), (768, 256)], 4096),
    ("n192-member", [(768, 768), (768, 192)], 4096),
    ("five", [(256, 256), (512, 256), (256, 512), (328, 768), (768, 256)], 1024),
]


@pytest.mark.gpu
@pytest.mark.parametrize("group", GROUPS, ids=lambda g: g[0])
def test_grouped_weight_gradients(cuda_dev, group):
    """b2_gemm_bf16_grouped with the step's arguments (workspace and rng_state set): one launch == each problem
    through b2_gemm_bf16 at BN 256 and one split, bitwise; a table it cannot group is issued problem by problem
    (auto configuration, may split); every output within its float64 bound"""
    name, shapes, K = group
    groupable = len(shapes) <= 4 and all(n % 256 == 0 for _, n in shapes)
    ops = [Ops("TN", m, n, K, cuda_dev, seed=100 + i) for i, (m, n) in enumerate(shapes)]
    ws = workspace(8 * max(m * n for m, n in shapes) * 4, cuda_dev)
    outs = [guarded(o.M, o.N, bf, cuda_dev) for o in ops]
    arr = (L.GemmArgs * len(ops))(*[gemm_args(o, D, ld, bn=0, splits=0, ws=ws) for o, (D, ld) in zip(ops, outs)])
    before = L.launch_count()
    L.call("b2_gemm_bf16_grouped", arr, len(ops), stream())
    torch.cuda.synchronize()
    if groupable:
        assert L.launch_count() - before == 1
    for i, (o, (D, ld)) in enumerate(zip(ops, outs)):
        untouched(D, o.M, o.N, "grouped D[%d]" % i)
        check_fp64_bf16(D[:o.M, :o.N], o, 0 if groupable else 8, "grouped", "%s problem %d" % (name, i))
        if groupable:
            D1, ld1 = guarded(o.M, o.N, bf, cuda_dev)
            gemm(o, D1, ld1, bn=256, splits=1)
            same(D[:o.M, :o.N], D1[:o.M, :o.N], "B exact", "%s problem %d grouped == single" % (name, i))


# ======================================================================================================================
# arguments: accepted ones change nothing, dropped ones are rejected
# ======================================================================================================================
def full_call(ops, epi, dev, gen):
    """a complete, valid set of extra arguments for `epi` (real, aligned device buffers)"""
    M, N = ops.M, ops.N
    kw = {"epi": epi}
    if epi in (L.EPI_BIAS, L.EPI_BIAS_GELU, L.EPI_BIAS_DROPOUT_RESIDUAL):
        kw["bias"] = torch.randn(N, device=dev, generator=gen).to(bf)
    if epi in (L.EPI_BIAS_DROPOUT_RESIDUAL, L.EPI_RESIDUAL, L.EPI_GELU_BWD):
        kw["aux_in"], kw["ld_aux_in"] = torch.randn(M, N, device=dev, generator=gen).to(bf), N
    if epi == L.EPI_RESIDUAL_F32:
        kw["aux_in"], kw["ld_aux_in"] = torch.randn(M, N, device=dev, generator=gen), N
    if epi == L.EPI_BIAS_GELU:
        kw["aux_out"], kw["ld_aux_out"] = torch.zeros(M, N, dtype=bf, device=dev), N
    return kw


F32_OUT = (L.EPI_RESIDUAL_F32, L.EPI_ACCUM_F32)
ALL_EPIS = {"NONE": L.EPI_NONE, "BIAS": L.EPI_BIAS, "BIAS_GELU": L.EPI_BIAS_GELU,
            "BIAS_DROPOUT_RESIDUAL": L.EPI_BIAS_DROPOUT_RESIDUAL, "RESIDUAL": L.EPI_RESIDUAL,
            "GELU_BWD": L.EPI_GELU_BWD, "RESIDUAL_F32": L.EPI_RESIDUAL_F32, "ACCUM_F32": L.EPI_ACCUM_F32}


@pytest.mark.gpu
@pytest.mark.parametrize("epi_name", list(ALL_EPIS))
def test_accepted_arguments_change_nothing(cuda_dev, epi_name):
    """rng_state at p = 0, a workspace on a problem that does not split, force_kernel and a debug_timing pointer are
    what the step, bench.py and the tools pass: accepted, and the result is the same bits"""
    epi = ALL_EPIS[epi_name]
    ops = Ops("NN", 256, 512, 512, cuda_dev, seed=21)
    kw = full_call(ops, epi, cuda_dev, ops.gen)
    dt = f32 if epi in F32_OUT else bf
    outs = []
    for extra in ({"rng": False}, {"rng": True, "ws": workspace(1 << 20, cuda_dev), "kernel": 2,
                                   "timing": torch.zeros(64, dtype=torch.int64, device=cuda_dev)}):
        D = torch.zeros(ops.M, ops.N, dtype=dt, device=cuda_dev)
        gemm(ops, D, ops.N, bn=128, splits=1, **kw, **extra)
        outs.append(D)
    same(outs[1], outs[0], "B exact", "%s with the accepted extra arguments" % epi_name)


def _reject_cases():
    cases = [("colsum_out-with-forced-split", "NONE", "colsum_out", {"colsum": True, "splits": 2, "ws": True})]
    for e in ("RESIDUAL_F32", "ACCUM_F32"):
        cases.append(("bias-with-" + e, e, "bias", {"bias": True}))
        cases.append(("colsum_out-with-" + e, e, "colsum_out", {"colsum": True}))
    for e in ("NONE", "RESIDUAL", "GELU_BWD"):
        cases.append(("bias-with-" + e, e, "bias", {"bias": True}))
    for e in ALL_EPIS:
        if e != "BIAS_DROPOUT_RESIDUAL":
            cases.append(("dropout_p-with-" + e, e, "dropout_p", {"p": 0.1}))
        if e != "BIAS_GELU":
            cases.append(("aux_out-with-" + e, e, "aux_out", {"aux_out": True}))
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("case", _reject_cases(), ids=lambda c: c[0])
def test_dropped_arguments_are_rejected(cuda_dev, case):
    """an argument the epilogue would not read is an error naming it, and nothing runs; without it the call works"""
    _name, epi_name, word, extra = case
    epi = ALL_EPIS[epi_name]
    M, N, K = 128, 256, 128
    ops = Ops("NN", M, N, K, cuda_dev, seed=31)
    kw = full_call(ops, epi, cuda_dev, ops.gen)
    dt = f32 if epi in F32_OUT else bf
    bad = dict(kw)
    if extra.get("bias"):
        bad["bias"] = torch.randn(N, device=cuda_dev).to(bf)
    if extra.get("colsum"):
        bad["colsum"] = torch.zeros(N, dtype=f32, device=cuda_dev)
    if extra.get("aux_out"):
        bad["aux_out"], bad["ld_aux_out"] = torch.zeros(M, N, dtype=bf, device=cuda_dev), N
    if extra.get("ws"):
        bad["ws"] = workspace(extra["splits"] * M * N * 4, cuda_dev)
    bad["splits"] = extra.get("splits", 1)
    bad["p"] = extra.get("p", 0.0)
    D, ld = guarded(M, N, dt, cuda_dev)
    with pytest.raises(RuntimeError) as ei:
        gemm(ops, D, ld, **bad)
    assert word in str(ei.value) and word in L.last_error(), str(ei.value)
    untouched(D, 0, 0, "output of a rejected call")
    gemm(ops, D, ld, splits=1, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("word", ["dropout_p", "bias"])
def test_grouped_rejects_the_table_before_running_any_of_it(cuda_dev, word):
    K = 1024
    ops = [Ops("TN", 256, 256, K, cuda_dev, seed=41 + i) for i in range(2)]
    outs = [guarded(o.M, o.N, bf, cuda_dev) for o in ops]
    args = [gemm_args(o, D, ld, bn=0, splits=0) for o, (D, ld) in zip(ops, outs)]
    bias = torch.randn(256, device=cuda_dev).to(bf)
    if word == "dropout_p":
        args[1].dropout_p = 0.1
    else:
        args[1].bias = bias.data_ptr()
    arr = (L.GemmArgs * 2)(*args)
    with pytest.raises(RuntimeError, match=word):
        L.call("b2_gemm_bf16_grouped", arr, 2, stream())
    torch.cuda.synchronize()
    for i, (D, _ld) in enumerate(outs):
        untouched(D, 0, 0, "grouped problem %d of a rejected table" % i)


# ---- pointer alignment: no GPU needed --------------------------------------------------------------------------------
# bias, aux_in and aux_out move in 16-byte vectors.  These calls run in a child process that sees no device
# (CUDA_VISIBLE_DEVICES empty) with made-up addresses that are never dereferenced: a build that does not check the
# alignment fails there on "no device" rather than launching a kernel on a misaligned pointer.
_ALIGN_CHILD = r"""
import ctypes, importlib.util, json, sys
spec = importlib.util.spec_from_file_location("b2_lib_child", sys.argv[1])
L = importlib.util.module_from_spec(spec)
spec.loader.exec_module(L)
base = 1 << 24
out = {}
for name, epi, field, offset in json.loads(sys.argv[2]):
    a = L.GemmArgs()
    a.M, a.N, a.K = 128, 256, 128
    a.A, a.lda, a.a_major = base, 128, L.MAJOR_K
    a.B, a.ldb, a.b_major = base + 0x100000, 256, L.MAJOR_MN
    a.D, a.ldd, a.epilogue = base + 0x200000, 256, epi
    if epi in (L.EPI_BIAS, L.EPI_BIAS_GELU, L.EPI_BIAS_DROPOUT_RESIDUAL):
        a.bias = base + 0x300000
    if epi in (L.EPI_BIAS_DROPOUT_RESIDUAL, L.EPI_RESIDUAL, L.EPI_GELU_BWD, L.EPI_RESIDUAL_F32):
        a.aux_in, a.ld_aux_in = base + 0x400000, 256
    if epi == L.EPI_BIAS_GELU:
        a.aux_out, a.ld_aux_out = base + 0x500000, 256
    if field:
        setattr(a, field, getattr(a, field) + offset)
    st = L.load().b2_gemm_bf16(ctypes.byref(a), None)
    out[name] = [int(st), L.last_error()]
print(json.dumps(out))
"""
ALIGN_CASES = [  # (id, epilogue, pointer, byte offset)
    ("bias+2-BIAS", L.EPI_BIAS, "bias", 2),
    ("bias+8-BIAS_GELU", L.EPI_BIAS_GELU, "bias", 8),
    ("bias+4-BIAS_DROPOUT_RESIDUAL", L.EPI_BIAS_DROPOUT_RESIDUAL, "bias", 4),
    ("aux_in+8-BIAS_DROPOUT_RESIDUAL", L.EPI_BIAS_DROPOUT_RESIDUAL, "aux_in", 8),
    ("aux_in+2-RESIDUAL", L.EPI_RESIDUAL, "aux_in", 2),
    ("aux_in+8-GELU_BWD", L.EPI_GELU_BWD, "aux_in", 8),
    ("aux_in+4-RESIDUAL_F32", L.EPI_RESIDUAL_F32, "aux_in", 4),
    ("aux_out+8-BIAS_GELU", L.EPI_BIAS_GELU, "aux_out", 8),
    ("aux_out+2-BIAS_GELU", L.EPI_BIAS_GELU, "aux_out", 2),
]
ALIGN_CONTROLS = [("aligned-%s" % e, epi, None, 0) for e, epi in ALL_EPIS.items()]


@pytest.fixture(scope="module")
def align_results():
    env = dict(os.environ)
    env["CUDA_VISIBLE_DEVICES"] = ""
    lib_py = os.path.join(ROOT, "pytorch-distributed-nlp_b200", "_lib.py")
    r = subprocess.run([sys.executable, "-c", _ALIGN_CHILD, lib_py, json.dumps(ALIGN_CASES + ALIGN_CONTROLS)],
                       env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", ALIGN_CASES, ids=lambda c: c[0])
def test_misaligned_pointer_is_rejected(align_results, case):
    name, _epi, field, _off = case
    st, err = align_results[name]
    assert st != 0 and "%s must be 16-byte aligned" % field in err, err


def test_aligned_pointers_pass_the_checks(align_results):
    """the same calls with aligned pointers get past every argument check (and then fail for want of a device), so
    the rejections above are the alignment's doing"""
    for name, *_ in ALIGN_CONTROLS:
        st, err = align_results[name]
        assert st != 0 and "aligned" not in err and "b2_gemm_bf16:" not in err, (name, err)


# ---- the comparison helpers themselves: no GPU needed ----------------------------------------------------------------
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf"), 1.5])
def test_within_fails_on_nan_inf_and_excess(bad):
    ref = torch.tensor([1.0, 2.0, 3.0], dtype=f64)
    bound = torch.full((3,), 1e-3, dtype=f64)
    within(torch.tensor([1.0, 2.0, 3.0], dtype=bf), ref, bound, "helper", "within passes when equal")
    got = torch.tensor([1.0, bad, 3.0], dtype=bf)
    with pytest.raises(AssertionError, match="at \\(1,\\)"):
        within(got, ref, bound, "helper", "within with %r" % bad)
    with pytest.raises(AssertionError):
        within(torch.tensor([1.0, 2.0, 3.0], dtype=bf), torch.tensor([1.0, bad, 3.0], dtype=f64), bound, "helper",
               "within with %r in the reference" % bad)


def test_same_fails_on_nan():
    ref = torch.tensor([1.0, 2.0], dtype=f32)
    same(ref.clone(), ref, "helper", "same passes when equal")
    with pytest.raises(AssertionError, match="1 elements differ"):
        same(torch.tensor([1.0, float("nan")], dtype=f32), ref, "helper", "same with NaN")
