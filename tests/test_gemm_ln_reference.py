"""The fused dense + bias + dropout + residual + LayerNorm kernel (b2_gemm_ln_fwd, csrc/gemm_ln.cu) element-wise
against float64 and against the unfused path, and the arguments it rejects.

Shapes: the engine's (config A M 4096 x N 768, K 768 / 3072; config B M 8192 x 768; config C M 2048 x 1024, K 1024 /
4096; a packed batch of 37 bins, M 4736), edges M in {1, 127, 128, 129, 200, 1000, 4101} at both cluster sizes
(N 768: 3 CTAs, N 1024: 4), K in {8, 72, 136} (tails inside one 64-deep k-block), and M 8192 at both N, where the row
blocks outnumber the clusters the device holds at once (asserted).  Dropout p in {0, 0.1} under two (site, step,
seed) keys.  Every output lives in a sentinel-filled buffer with guard rows and its own pad (ldd = N + 8,
ldy = N + 24, ldyf = N + 12; the fp32 residual is read at ld_aux_in = N + 20, A at K + 16, W at K + 8); mean and
rstd have guard entries past M.  Nothing outside [M) x [N) may change.  A second call with y_f32 = NULL must give
the same bits.

Notation: U = 2^-24, UB = 2^-8 (fp32 / bf16 unit roundoff); BN = 256 columns per CTA, CL = N / 256 CTAs per row.
Every check asserts bitwise equality or error <= bound element-wise (a NaN fails either), and sends its worst
error / bound (or mismatch count) to parity.report under the tag "gemm_ln_reference".

(a) Exact operands.  A and W integer in [-2, 2], bias and residual multiples of 1/8 (the residual of every 7th row
    offset by 1024).  Every partial sum of the accumulator is an integer below 4 K <= 2^14, exact in fp32 whatever
    the tensor cores' order or alignment, and z = acc + bias + residual is exact too.  So D == bf16(z) bitwise, and
    the statistics, y_f32 and y are checked against float64 LayerNorm of the exact z.  This layer makes no
    assumption about the hardware; it catches a dropped or repeated k-block, a wrong row or column tile and a wrong
    bias, gamma or beta column.
(b) Random operands.  The fused mainloop issues b2_gemm_bf16's NT sequence at BN 256 and one split (64-deep
    k-blocks, wgmma m64n256k16, the same descriptors), so its accumulator is that of test_gemm_reference.accumulator.
    At p = 0, D == bf16(fp32(fp32(acc + bias) + res)) bitwise and z is known exactly; at p = 0.1 the Philox mask
    (keyed m * N + n) gives ref = keep * t * scale + res with t = fp32(acc + bias), within Ez = 2U (|t scale| + |res|)
    (product and sum rounded apart or contracted), then one bf16 rounding.  Statistics and y as in (a), around the
    restated z, with Ez carried through.
(c) Fused == unfused.  The same operands with a bf16-representable residual through b2_gemm_bf16's
    BIAS_DROPOUT_RESIDUAL at BN 256 and one split give the same D, bit for bit, at p = 0 and 0.1: the two paths the
    engine chooses between (_Engine.fused_ln) share mask keying, site and epilogue arithmetic.
(d) Row edges, at both cluster sizes: rows with a common offset (residual 1000 + 0.05 noise, A's row scaled by 1/32),
    where E[z^2] - mean^2 in fp32 would lose every digit; constant rows of few-bit values 3, -1000 and 0.5 (A's row
    zero, residual c - bias, exact in fp32, so z is exactly c): mean == c and y == y_f32 == beta bit for bit -- at N
    768 the merged mean is multiplied by fp32(1/3) = (1 + 2^-25) / 3, which still rounds back to c for these values;
    a nearly constant row (-7 + 1e-3 noise) held to its bound.  Constant rows of full-precision fp32 values lie
    outside this analysis (the bound on the variance, e_mu^2 / var and the linear term below, is unbounded when
    var = 0 and the mean is not exact), so nothing is asserted on them.
(e) The saved state feeds the backward: b2_layernorm_bwd_accum on the fused kernel's D (bf16 z), mean and rstd, as
    the engine pairs them, against the float64 LayerNorm backward at the exact z of (a) with exact statistics.

Bounds of the statistics (per row; z the exact values, A_c = mean |z| over CTA tile c, mu_c / M2_c the tile's mean
and sum of squared deviations, d_c = mu_c - mu):
  partial mean   8 sequential lane adds + 5 shuffle levels, then * 1/256 (exact): |e_c| <= E_c = 13 U A_c
  merged mean    CL - 1 additions, and for CL = 3 the multiply by fp32(1/3) (2 more roundings):
                 e_mu = mean_c E_c + (CL - 1 [+ 2]) U mean_c(|mu_c| + E_c)
  partial M2     d = fl(z - mean_c) (2U on d^2) + 8 FMAs + 5 shuffle levels, around the inexact partial mean:
                 M2_c (1 +- 15U) + 256 E_c^2
  merge          Chan's M2 = sum M2_c + BN d_c^2, d_c computed from the two inexact means: |dd_c| <= E_c + e_mu +
                 U |d_c|, so BN (2 |d_c| dd_c + dd_c^2); CL + 1 roundings over the non-negative terms
  rstd           m2 / N and + eps (2U relative), rsqrtf within 2 ulp (4U): e_rel = r / (2 (1 - r)) + 4U (1 + r)
                 with r the relative error of var + eps; no claim (infinite bound) once r >= 1/2
  with Ez        (p = 0.1) e_mu += mean Ez, var += 2 mean(|z - mu| Ez) + mean Ez^2
All of it times 1.001 for the second-order terms left out.  y and y_f32 against (z - mean) rstd gamma + beta from
the kernel's own mean and rstd (checked above): 4 roundings, 4U (|xhat gamma| + |beta|) (+ Ez rstd |gamma|), then
bf_bound for y; y == bf16(y_f32) bitwise.
Backward (e): test_step_kernels.ln_bwd_ref at the exact z and exact statistics, with the kernel's xhat further off by
  UB |z| rstd (D is bf16(z)) + (e_mu + |xhat| e_rel / rstd) rstd (its statistics), and the whole dx by e_rel.

Measured on an H100 80GB HBM3 (700 W power limit), worst error / bound per check family, over every shape and key:
  (a) exact operands    mean 0.078, rstd 0.19, y_f32 0.63, y 0.996 (the half-ulp bf16 rounding itself); D bitwise
  (b) random operands   mean 0.033, rstd 0.19, y_f32 0.67, y 0.996; D at p = 0.1 0.996; D at p = 0 bitwise
  (c) fused == unfused  0 mismatches at p = 0 and 0.1
  (d) row edges         mean 0.089, rstd 0.13, y_f32 0.68, y 0.996; the constant rows bit for bit
  (e) backward dx       0.75.  The bf16 rounding of z moves the backward's xhat by up to UB |z| rstd = 0.68 on the
                        offset rows at K 8 (1024 against a spread of about 7), 0.20-0.28 at K 72-136, below 0.1
                        elsewhere: with z saved as bf16 the backward of a strongly offset row is that coarse.
  every exact check     0 mismatches (420 checks)
The accumulator of (b) is bitwise that of b2_gemm_bf16 (every p = 0 D matched).  The device held 39 clusters of 3 CTAs
at once, so M 8192 ran 64 row blocks over them.  Runtime, from one `pytest -m gpu tests/test_gemm_ln_reference.py`
on that card: 106 tests in 4.4 s as pytest counts it, 12.4 s of wall time with interpreter and CUDA start-up.
With B2_PARITY_REPORT set, every check appends its ratio there (tag "gemm_ln_reference").
"""
import json
import os
import subprocess
import sys
import zlib

import pytest
import torch

import test_gemm_reference as gr
from parity import philox_keep_mask
from pytorch_distributed_nlp_b200 import _lib as L
from test_gemm_reference import KM, SEED, SENT, STEP, U, UB, accumulator, bf_bound, drop_scale, guarded, untouched
from test_step_kernels import EPS, ln_bwd_ref, ln_fwd_check

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAG = "gemm_ln_reference"
bf, f32 = torch.bfloat16, torch.float32
BN = 256
SLACK = 1.001
PADS = {"D": 8, "Y": 24, "YF": 12, "RES": 20, "A": 16, "W": 8}
# (seed, step, site): the step's first key, and a second with a seed above 2^32 and a step that wraps 32 bits
KEYS = [(SEED, STEP, 5), (0x1234_5678_9ABC, 2 ** 32 + 9, 35)]


def stream():
    return torch.cuda.current_stream().cuda_stream


def within(got, ref, bound, family, what):
    gr.within(got, ref, bound, family, what, tag=TAG)


def same(got, ref, family, what):
    gr.same(got, ref, family, what, tag=TAG)


def checker(family):
    """the check= of test_step_kernels.ln_fwd_check, reporting under this file's tag"""
    return lambda got, ref, bound, what: within(got, ref, bound, family, what)


_MASKS = {}
_RNG = {}


def keep_mask(M, N, key, p, dev):
    """fp64 [M, N]: 1 where the Philox stream of `key` keeps element m * N + n, else 0"""
    k = (M, N, key, p)
    if k not in _MASKS:
        seed, step, site = KEYS[key]
        _MASKS[k] = torch.from_numpy(philox_keep_mask(M * N, seed, step, site, p).reshape(M, N)).to(dev).double()
    return _MASKS[k]


def rng_for(key, dev):
    if key not in _RNG:
        seed, step, _site = KEYS[key]
        _RNG[key] = torch.tensor([seed, step], dtype=torch.int64, device=dev)
    return _RNG[key]


class LnOps:
    """the fused kernel's operands: A [M, K] at lda = K + 16, W [N, K] at ldb = K + 8 (NT, both K-major), bias,
    gamma, beta, and the fp32 residual at ld_aux_in = N + 20.  Duck-types test_gemm_reference.Ops for accumulator().
    exact: A and W integers in [-2, 2], bias and residual multiples of 1/8, every 7th row's residual offset by 1024."""

    def __init__(self, M, N, K, dev, seed, exact):
        self.layout, self.M, self.N, self.K, self.dev = "NT", M, N, K, dev
        self.am = self.bm = KM
        self.exact = exact
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.gen = gen
        if exact:
            A = torch.randint(-2, 3, (M, K + PADS["A"]), device=dev, generator=gen).to(bf)
            W = torch.randint(-2, 3, (N, K + PADS["W"]), device=dev, generator=gen).to(bf)
            self.bias = (torch.randint(-32, 33, (N,), device=dev, generator=gen) / 8.0).to(bf)
            R = torch.randint(-64, 65, (M, N + PADS["RES"]), device=dev, generator=gen) / 8.0
            R[3::7] += 1024.0
        else:
            A = torch.randn(M, K + PADS["A"], device=dev, generator=gen).to(bf)
            W = (torch.randn(N, K + PADS["W"], device=dev, generator=gen) / K ** 0.5).to(bf)
            self.bias = torch.randn(N, device=dev, generator=gen).to(bf)
            R = torch.randn(M, N + PADS["RES"], device=dev, generator=gen)
        self.A_store, self.lda = A[:, :K], K + PADS["A"]
        self.B_store, self.ldb = W[:, :K], K + PADS["W"]
        self.R_buf, self.ldr = R.float(), N + PADS["RES"]
        self.gamma = (1 + 0.25 * torch.randn(N, device=dev, generator=gen)).to(bf)
        self.beta = (0.5 * torch.randn(N, device=dev, generator=gen)).to(bf)

    @property
    def res(self):
        return self.R_buf[:, :self.N]

    def z_exact(self):
        """(a): the exact fp64 z = A W^T + bias + res (every term and partial sum exact)"""
        return self.A_store.double() @ self.B_store.double().t() + self.bias.double() + self.res.double()


def ln_args(ops, D, ldd, p=0.0, key=0, **extra):
    a = gr.gemm_args(ops, D, ldd, epi=L.EPI_BIAS_DROPOUT_RESIDUAL, bias=ops.bias, aux_in=ops.R_buf,
                     ld_aux_in=ops.ldr, p=p, site=KEYS[key][2], **extra)
    a.rng_state = rng_for(key, ops.dev).data_ptr()
    return a


class Out:
    """sentinel-filled outputs of one fused call"""

    def __init__(self, M, N, dev, with_yf=True):
        self.M, self.N = M, N
        self.D, self.ldd = guarded(M, N, bf, dev, pad=PADS["D"])
        self.Y, self.ldy = guarded(M, N, bf, dev, pad=PADS["Y"])
        self.YF, self.ldyf = guarded(M, N, f32, dev, pad=PADS["YF"]) if with_yf else (None, 0)
        self.mean = torch.full((M + 5,), SENT, dtype=f32, device=dev)
        self.rstd = torch.full((M + 5,), SENT, dtype=f32, device=dev)

    def untouched(self, what):
        M, N = self.M, self.N
        untouched(self.D, M, N, what + " D")
        untouched(self.Y, M, N, what + " y")
        if self.YF is not None:
            untouched(self.YF, M, N, what + " y_f32")
        for name, v in (("mean", self.mean), ("rstd", self.rstd)):
            assert bool((v[M:] == SENT).all()), "%s %s written past M" % (what, name)

    d = property(lambda s: s.D[:s.M, :s.N])
    y = property(lambda s: s.Y[:s.M, :s.N])
    yf = property(lambda s: s.YF[:s.M, :s.N])
    mu = property(lambda s: s.mean[:s.M])
    rs = property(lambda s: s.rstd[:s.M])


def fused(ops, p=0.0, key=0, with_yf=True, **extra):
    o = Out(ops.M, ops.N, ops.dev, with_yf)
    a = ln_args(ops, o.D, o.ldd, p, key, **extra)
    L.call("b2_gemm_ln_fwd", a, ops.gamma.data_ptr(), ops.beta.data_ptr(), EPS, o.Y.data_ptr(), o.ldy,
           L.ptr(o.YF), o.ldyf, o.mean.data_ptr(), o.rstd.data_ptr(), stream())
    torch.cuda.synchronize()
    o.untouched("fused p=%g" % p)
    return o


def stats_bound(z, ez=None):
    """(e_mu, e_rel, var) of the fused kernel's statistics of the rows z (fp64 [M, N]); ez: how far the kernel's
    own z may lie from z.  Derived in the module docstring."""
    M, N = z.shape
    CL = N // BN
    t = z.view(M, CL, BN)
    Ac = t.abs().mean(2) if ez is None else (t.abs() + ez.view(M, CL, BN)).mean(2)
    mu_c = t.mean(2)
    mu = mu_c.mean(1)
    d = (mu_c - mu[:, None]).abs()
    M2c = ((t - mu_c[..., None]) ** 2).sum(2)
    var = (M2c.sum(1) + BN * (d ** 2).sum(1)) / N
    Ec = 13 * U * Ac
    e_mu = Ec.mean(1) + (CL - 1 + (2 if CL == 3 else 0)) * U * (mu_c.abs() + Ec).mean(1)
    dd = Ec + e_mu[:, None] + U * (d + Ec + e_mu[:, None])
    T = M2c + BN * Ec ** 2
    e_m2 = (BN * Ec ** 2 + 15 * U * T + BN * (2 * d * dd + dd ** 2)).sum(1)
    e_m2 = e_m2 + (CL + 1) * U * (T * (1 + 15 * U) + BN * (d + dd) ** 2).sum(1)
    e_var = e_m2 / N
    if ez is not None:
        e_mu = e_mu + ez.mean(1)
        e_var = e_var + 2 * ((z - mu[:, None]).abs() * ez).mean(1) + (ez ** 2).mean(1)
    e_mu, e_var = SLACK * e_mu, SLACK * e_var
    r = (e_var + 2 * U * (var + e_var + EPS)) / (var + EPS)
    e_rel = r / (2 * (1 - r)) + 4 * U * (1 + r)
    e_rel = torch.where(r < 0.5, SLACK * e_rel, torch.full_like(r, float("inf")))
    return e_mu, e_rel


def check_ln(ops, o, z, family, what, ez=None):
    """statistics, y_f32 and y of one fused call against float64 LayerNorm of z"""
    e_mu, e_rel = stats_bound(z, ez)
    ln_fwd_check(z, o.mu, o.rs, o.y, ops.gamma, ops.beta, what, y_f32=o.yf, stats_bound=(e_mu, e_rel), ev=ez,
                 check=checker(family))
    same(o.y, o.yf.to(bf), "exact", what + " y == bf16(y_f32)")
    return e_mu, e_rel


# ======================================================================================================================
# shapes
# ======================================================================================================================
ENGINE = [(4096, 768, 768), (4096, 768, 3072),        # config A: attention output, FFN output
          (8192, 768, 768), (8192, 768, 3072),        # config B
          (2048, 1024, 1024), (2048, 1024, 4096),     # config C
          (37 * 128, 768, 768)]                       # packed bins
EDGE_M = [(M, N, N) for N in (768, 1024) for M in (1, 127, 128, 129, 200, 1000, 4101)]
EDGE_K = [(512, N, K) for N in (768, 1024) for K in (8, 72, 136)] + [(200, 1024, 136)]
SHAPES = ENGINE + EDGE_M + EDGE_K


def sid(s):
    return "%dx%dx%d" % s


def need_cluster(N):
    if L.load().b2_gemm_ln_max_clusters(N) <= 0:
        pytest.fail("the device cannot hold a %d-CTA cluster of the fused kernel" % (N // BN))


# ======================================================================================================================
# (a) exact operands, and (e) the backward fed by the saved state
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=sid)
def test_exact_operands(cuda_dev, shape):
    M, N, K = shape
    need_cluster(N)
    ops = LnOps(M, N, K, cuda_dev, zlib.crc32(b"a" + sid(shape).encode()), exact=True)
    o = fused(ops)
    z = ops.z_exact()
    what = "(a) %s" % sid(shape)
    same(o.d, z.float().to(bf), "exact", what + " D == bf16(z)")
    e_mu, e_rel = check_ln(ops, o, z, "(a) exact operands", what)
    check_backward(ops, o, z, e_mu, e_rel, "(e) %s" % sid(shape))


def check_backward(ops, o, z, e_mu, e_rel, what):
    """(e): b2_layernorm_bwd_accum on the fused kernel's D, mean and rstd vs the fp64 backward at the exact z"""
    M, N = z.shape
    dev = ops.dev
    dy = torch.randn(M, N, device=dev, generator=ops.gen)
    x = o.d.contiguous()
    dx = torch.full((M, N), float("nan"), device=dev)
    dxd = torch.empty(M, N, dtype=bf, device=dev)
    acc = torch.zeros(3, N, device=dev)
    L.call("b2_layernorm_bwd_accum", dy.data_ptr(), x.data_ptr(), o.mean.data_ptr(), o.rstd.data_ptr(),
           ops.gamma.data_ptr(), M, N, 0.0, gr.rng_state(dev).data_ptr(), 0, dx.data_ptr(), dxd.data_ptr(),
           acc.data_ptr(), stream())
    torch.cuda.synchronize()
    mu64 = z.mean(1, keepdim=True)
    rs64 = 1.0 / torch.sqrt(((z - mu64) ** 2).mean(1, keepdim=True) + EPS)
    er = e_rel[:, None]
    xh = ((z - mu64) * rs64).abs()
    # the kernel's xhat: x = bf16(z) is UB |z| off, its mean e_mu, its rstd e_rel
    ex_extra = (UB * z.abs() + e_mu[:, None]) * rs64 * (1 + er) + xh * er
    ref, E, _xh, _ex = ln_bwd_ref(dy, z, mu64[:, 0], rs64[:, 0], ops.gamma, ex_extra=ex_extra)
    within(dx, ref, E * (1 + er) + er * ref.abs(), "(e) backward from the saved state", what + " dx")
    gr.report(TAG, {"family": "(e) xhat perturbation from bf16 z", "check": what,
                    "max_UB_z_rstd": float((UB * z.abs() * rs64).max())})


# ======================================================================================================================
# (b) random operands against the kernel's own accumulator
# ======================================================================================================================
B_CASES = [(s, 0.0, 0) for s in SHAPES] + [(s, 0.1, 0) for s in SHAPES] + [(s, 0.1, 1) for s in ENGINE]


@pytest.mark.gpu
@pytest.mark.parametrize("case", B_CASES, ids=lambda c: "%s-p%g-key%d" % (sid(c[0]), c[1], c[2]))
def test_random_operands(cuda_dev, case):
    shape, p, key = case
    M, N, K = shape
    need_cluster(N)
    ops = LnOps(M, N, K, cuda_dev, zlib.crc32(b"b" + sid(shape).encode()), exact=False)
    acc = accumulator(ops, 256)
    o = fused(ops, p, key)
    what = "(b) %s p=%g key%d" % (sid(shape), p, key)
    check_restated(ops, o, acc, p, key, what)
    # the same call without y_f32: every other output the same bits
    o2 = fused(ops, p, key, with_yf=False)
    for name in ("d", "y", "mu", "rs"):
        same(getattr(o2, name), getattr(o, name), "exact", what + " %s without y_f32" % name)


def check_restated(ops, o, acc, p, key, what, family="(b) random operands"):
    """D, statistics and y of a fused call against z restated from the kernel's own accumulator"""
    M, N = ops.M, ops.N
    t = acc + ops.bias.float()                                    # fp32, as the kernel rounds it
    if p == 0:
        z = (t + ops.res).double()                                # exact: the kernel's own z
        same(o.d, z.float().to(bf), "exact", what + " D")
        return check_ln(ops, o, z, family, what)
    ts = t.double() * keep_mask(M, N, key, p, ops.dev) * drop_scale(p)
    r = ops.res.double()
    z = ts + r
    ez = 2 * U * (ts.abs() + r.abs())
    within(o.d, z, bf_bound(z, ez), family + " D", what + " D")
    return check_ln(ops, o, z, family, what, ez=ez)


# ======================================================================================================================
# (c) fused == unfused
# ======================================================================================================================
C_SHAPES = [(4096, 768, 768), (4096, 768, 3072), (2048, 1024, 1024), (129, 768, 136), (1000, 1024, 72)]


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("shape", C_SHAPES, ids=sid)
def test_fused_equals_unfused(cuda_dev, shape, p):
    M, N, K = shape
    need_cluster(N)
    ops = LnOps(M, N, K, cuda_dev, zlib.crc32(b"c" + sid(shape).encode()), exact=False)
    ops.R_buf = ops.R_buf.to(bf).float()                          # a residual both paths hold exactly
    res_bf, ld_bf = guarded(M, N, bf, cuda_dev, pad=PADS["Y"])      # bf16 rows want ld % 8 == 0
    res_bf[:M, :N] = ops.res.to(bf)
    o = fused(ops, p, 0)
    D, ld = guarded(M, N, bf, cuda_dev, pad=PADS["D"])
    a = gr.gemm_args(ops, D, ld, epi=L.EPI_BIAS_DROPOUT_RESIDUAL, bn=256, splits=1, bias=ops.bias, aux_in=res_bf,
                     ld_aux_in=ld_bf, p=p, site=KEYS[0][2])
    a.rng_state = rng_for(0, cuda_dev).data_ptr()
    L.call("b2_gemm_bf16", a, stream())
    torch.cuda.synchronize()
    untouched(D, M, N, "unfused D")
    same(o.d, D[:M, :N], "(c) fused == unfused", "(c) %s p=%g D fused == unfused" % (sid(shape), p))


# ======================================================================================================================
# (d) row edges
# ======================================================================================================================
CONSTANT_ROWS = {0: 3.0, 2: -1000.0, 4: 0.5, 131: 3.0, 258: -1000.0, 299: 0.5}
OFFSET_ROWS = (1, 6, 130, 255)
NEAR_CONSTANT_ROWS = (5, 257)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [768, 1024])
def test_row_edges(cuda_dev, N):
    M, K = 300, N
    need_cluster(N)
    dev = cuda_dev
    ops = LnOps(M, N, K, dev, 17 + N, exact=False)
    ops.bias = (torch.round(ops.bias.float() * 64) / 64).to(bf)   # on the 2^-6 grid: c - bias is exact in fp32
    A = ops.A_store
    bias = ops.bias.float()
    for r in OFFSET_ROWS:
        A[r] = (A[r].float() / 32).to(bf)
        ops.res[r] = 1000.0 + 0.05 * torch.randn(N, device=dev, generator=ops.gen)
    for r in NEAR_CONSTANT_ROWS:
        A[r] = 0
        ops.res[r] = -7.0 + 1e-3 * torch.randn(N, device=dev, generator=ops.gen) - bias
    for r, c in CONSTANT_ROWS.items():
        A[r] = 0
        ops.res[r] = c - bias                                     # exact in fp32, and so is bias + (c - bias)
    acc = accumulator(ops, 256)
    o = fused(ops)
    what = "(d) N=%d" % N
    check_restated(ops, o, acc, 0.0, 0, what, family="(d) row edges")
    rows = list(CONSTANT_ROWS)
    c = torch.tensor([CONSTANT_ROWS[r] for r in rows], dtype=f32, device=dev)
    same(o.mu[rows], c, "exact", what + " mean of constant rows")
    same(o.d[rows], c[:, None].expand(-1, N).to(bf), "exact", what + " D of constant rows")
    same(o.yf[rows], ops.beta.float().expand(len(rows), -1), "exact", what + " y_f32 of constant rows == beta")
    same(o.y[rows], ops.beta.expand(len(rows), -1), "exact", what + " y of constant rows == beta")


# ======================================================================================================================
# more row blocks than clusters fit at once
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("N", [768, 1024])
def test_more_row_blocks_than_clusters(cuda_dev, N):
    M, K = 8192, N
    need_cluster(N)
    clusters = L.load().b2_gemm_ln_max_clusters(N)
    assert -(-M // 128) > clusters, "M %d does not exceed the %d co-resident clusters" % (M, clusters)
    ops = LnOps(M, N, K, cuda_dev, 23 + N, exact=True)
    o = fused(ops)
    z = ops.z_exact()
    what = "(a) %s, %d row blocks over %d clusters" % (sid((M, N, K)), M // 128, clusters)
    same(o.d, z.float().to(bf), "exact", what + " D == bf16(z)")
    check_ln(ops, o, z, "(a) exact operands", what)


# ======================================================================================================================
# arguments
# ======================================================================================================================
@pytest.mark.gpu
def test_accepted_arguments_change_nothing(cuda_dev):
    """force_kernel, a debug_timing pointer, force_bn 256 and force_splits 1 are accepted and change no bit"""
    ops = LnOps(300, 768, 768, cuda_dev, 29, exact=False)
    o = fused(ops, 0.1, 0)
    o2 = fused(ops, 0.1, 0, bn=256, splits=1, kernel=2, timing=torch.zeros(64, dtype=torch.int64, device=cuda_dev))
    for name in ("d", "y", "yf", "mu", "rs"):
        same(getattr(o2, name), getattr(o, name), "exact", "accepted arguments: %s" % name)


# The rejections run in a child process that sees no device, with made-up addresses that are never dereferenced: a
# build without a check fails there on the missing device instead of launching on the bad argument.
_CHILD = r"""
import ctypes, importlib.util, json, sys
spec = importlib.util.spec_from_file_location("b2_lib_child", sys.argv[1])
L = importlib.util.module_from_spec(spec)
spec.loader.exec_module(L)
base = 1 << 24
out = {}
for name, entry, epi, a_major, b_major, fields, extra in json.loads(sys.argv[2]):
    a = L.GemmArgs()
    a.M, a.N, a.K = 256, 768, 512
    a.A, a.a_major = base, a_major
    a.lda = 512 if a_major == L.MAJOR_K else 256
    a.B, a.b_major = base + 0x100000, b_major
    a.ldb = 512 if b_major == L.MAJOR_K else 768
    a.D, a.ldd, a.epilogue = base + 0x200000, 768, epi
    if epi in (L.EPI_BIAS, L.EPI_BIAS_GELU, L.EPI_BIAS_DROPOUT_RESIDUAL):
        a.bias = base + 0x300000
    if epi in (L.EPI_BIAS_DROPOUT_RESIDUAL, L.EPI_RESIDUAL, L.EPI_GELU_BWD, L.EPI_RESIDUAL_F32):
        a.aux_in, a.ld_aux_in = base + 0x400000, 768
    if epi == L.EPI_BIAS_GELU:
        a.aux_out, a.ld_aux_out = base + 0x500000, 768
    ln = {"y": base + 0x600000, "ldy": 768, "y_f32": base + 0x700000, "ldyf": 768}
    for k, v in fields.items():
        setattr(a, k, v if not isinstance(v, str) else base + int(v, 16))
    ln.update(extra)
    if entry == "ln":
        st = L.load().b2_gemm_ln_fwd(ctypes.byref(a), base + 0x800000, base + 0x810000, 1e-12, ln["y"], ln["ldy"],
                                     ln["y_f32"], ln["ldyf"], base + 0x820000, base + 0x830000, None)
    else:
        st = L.load().b2_gemm_bf16(ctypes.byref(a), None)
    out[name] = [int(st), L.last_error()]
print(json.dumps(out))
"""
E_BDR = L.EPI_BIAS_DROPOUT_RESIDUAL
LN_REJECT = [  # (id, entry, epilogue, a_major, b_major, GemmArgs fields, fused-only arguments, word in the error)
    ("ln-colsum_out", "ln", E_BDR, KM, KM, {"colsum_out": "900000"}, {}, "colsum_out"),
    ("ln-aux_out", "ln", E_BDR, KM, KM, {"aux_out": "500000", "ld_aux_out": 768}, {}, "aux_out"),
    ("ln-force_splits-2", "ln", E_BDR, KM, KM, {"force_splits": 2}, {}, "force_splits"),
    ("ln-force_bn-128", "ln", E_BDR, KM, KM, {"force_bn": 128}, {}, "force_bn"),
    ("ln-workspace", "ln", E_BDR, KM, KM, {"workspace": "a00000", "workspace_bytes": 1 << 20}, {}, "workspace"),
    ("ln-lda", "ln", E_BDR, KM, KM, {"lda": 504}, {}, "lda="),
    ("ln-ldb", "ln", E_BDR, KM, KM, {"ldb": 0}, {}, "ldb="),
    ("ln-ldd-0", "ln", E_BDR, KM, KM, {"ldd": 0}, {}, "ldd="),
    ("ln-ldd", "ln", E_BDR, KM, KM, {"ldd": 760}, {}, "ldd="),
    ("ln-ld_aux_in", "ln", E_BDR, KM, KM, {"ld_aux_in": 764}, {}, "ld_aux_in="),
    ("ln-ldy", "ln", E_BDR, KM, KM, {}, {"ldy": 0}, "ldy="),
    ("ln-ldyf-0", "ln", E_BDR, KM, KM, {}, {"ldyf": 0}, "ldyf="),
    ("ln-ldyf", "ln", E_BDR, KM, KM, {}, {"ldyf": 764}, "ldyf="),
]
GEMM_REJECT = [
    ("gemm-lda-K", "gemm", L.EPI_NONE, KM, L.MAJOR_MN, {"lda": 504}, {}, "lda="),
    ("gemm-lda-MN", "gemm", L.EPI_NONE, L.MAJOR_MN, L.MAJOR_MN, {"lda": 248}, {}, "lda="),
    ("gemm-ldb-K", "gemm", L.EPI_NONE, KM, KM, {"ldb": 0}, {}, "ldb="),
    ("gemm-ldb-MN", "gemm", L.EPI_NONE, KM, L.MAJOR_MN, {"ldb": 512}, {}, "ldb="),
    ("gemm-ldd-0", "gemm", L.EPI_BIAS, KM, KM, {"ldd": 0}, {}, "ldd="),
    ("gemm-ldd", "gemm", L.EPI_NONE, KM, KM, {"ldd": 760}, {}, "ldd="),
    ("gemm-ld_aux_in-BIAS_DROPOUT_RESIDUAL", "gemm", E_BDR, KM, KM, {"ld_aux_in": 0}, {}, "ld_aux_in="),
    ("gemm-ld_aux_in-RESIDUAL_F32", "gemm", L.EPI_RESIDUAL_F32, KM, L.MAJOR_MN, {"ld_aux_in": 760}, {}, "ld_aux_in="),
    ("gemm-ld_aux_in-GELU_BWD", "gemm", L.EPI_GELU_BWD, KM, L.MAJOR_MN, {"ld_aux_in": 256}, {}, "ld_aux_in="),
    ("gemm-ld_aux_out-BIAS_GELU", "gemm", L.EPI_BIAS_GELU, KM, KM, {"ld_aux_out": 0}, {}, "ld_aux_out="),
]
ACCEPT = [  # calls that must get past every argument check
    ("ln-plain", "ln", E_BDR, KM, KM, {}, {}),
    ("ln-ldyf-0-without-y_f32", "ln", E_BDR, KM, KM, {}, {"y_f32": None, "ldyf": 0}),
    ("ln-accepted-extras", "ln", E_BDR, KM, KM, {"force_kernel": 2, "debug_timing": "b00000", "force_bn": 256,
                                                 "force_splits": 1}, {}),
    ("ln-wide-lds", "ln", E_BDR, KM, KM, {"lda": 1024, "ldb": 520, "ldd": 776, "ld_aux_in": 788},
     {"ldy": 792, "ldyf": 780}),
    ("gemm-NT", "gemm", L.EPI_BIAS, KM, KM, {}, {}),
    ("gemm-NN", "gemm", L.EPI_NONE, KM, L.MAJOR_MN, {}, {}),
    ("gemm-TN", "gemm", L.EPI_NONE, L.MAJOR_MN, L.MAJOR_MN, {}, {}),
    ("gemm-NONE-ld_aux_in-0", "gemm", L.EPI_NONE, KM, KM, {"ld_aux_in": 0, "ld_aux_out": 0}, {}),
    ("gemm-ACCUM_F32-ld_aux_in-0", "gemm", L.EPI_ACCUM_F32, KM, L.MAJOR_MN, {"ld_aux_in": 0}, {}),
]


@pytest.fixture(scope="module")
def child_results():
    env = dict(os.environ)
    env["CUDA_VISIBLE_DEVICES"] = ""
    lib_py = os.path.join(ROOT, "pytorch-distributed-nlp_b200", "_lib.py")
    cases = [c[:7] for c in LN_REJECT + GEMM_REJECT] + ACCEPT
    r = subprocess.run([sys.executable, "-c", _CHILD, lib_py, json.dumps(cases)], env=env, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", LN_REJECT + GEMM_REJECT, ids=lambda c: c[0])
def test_argument_is_rejected(child_results, case):
    name, entry, word = case[0], case[1], case[7]
    st, err = child_results[name]
    prefix = "b2_gemm_ln_fwd: " if entry == "ln" else "b2_gemm_bf16: "
    assert st != 0 and err.startswith(prefix) and word in err, err


@pytest.mark.parametrize("case", ACCEPT, ids=lambda c: c[0])
def test_valid_arguments_pass_the_checks(child_results, case):
    """the same calls with valid arguments get past every argument check (and then fail for want of a device), so
    the rejections above are the checks' doing"""
    st, err = child_results[case[0]]
    assert st != 0, case[0]
    for phrase in ("must be NULL", "is below", "force_", "must be multiples", "aligned", "null"):
        assert phrase not in err, (case[0], err)
