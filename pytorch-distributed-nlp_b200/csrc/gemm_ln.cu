// Dense + bias + dropout + residual + LayerNorm in ONE kernel: BertSelfOutput.forward / BertOutput.forward
// (SP/transformers/models/bert/modeling_bert.py:294-298, :352-356: `LayerNorm(dropout(dense(h)) + input)`).
//
// Why a kernel of its own.
//  * precision: with separate kernels the pre-LayerNorm sum z and the LayerNorm output both travelled through HBM as
//    bf16, i.e. the RESIDUAL STREAM was rounded to bf16 four times per layer; the gradient error of the attention
//    query / key projections then grows with depth, where stock torch bf16 autocast -- which keeps the stream in fp32
//    and rounds only GEMM operands -- does not.  Here z never leaves the SM before it is normalised (fp32 accumulator
//    + fp32 residual -> statistics -> y), the residual comes in as fp32 and the LayerNorm output leaves both as bf16
//    (the next GEMM's operand) and as fp32 (the next block's residual).
//  * launches: one kernel instead of two per site, 24 sites per step.
// LayerNorm needs full rows, and a row of 768 / 1024 fp32 accumulators does not fit one CTA's registers next to the
// operand ring -- so the row is spread over a CLUSTER of N / 256 CTAs (3 for hidden 768, 4 for hidden 1024): CTA
// rank c owns columns [256 c, 256 c + 256) of the cluster's 128 rows and runs the GEMM mainloop of gemm.cu on them
// (TMA producer warp, two wgmma consumer warpgroups, fp32 tile left in shared memory).  The epilogue then works a
// row per warp, 8 columns per lane (coalesced global traffic, one Philox call per lane and row):
//   pass 1  z = (acc + bias -> dropout) + residual in fp32, kept in shared memory in place of the accumulator;
//           bf16(z) stored to D for the backward; the row's partial statistics over the CTA's 256 columns (mean,
//           M2 = sum (z - mean)^2) are written into the `stats` pad of every CTA of the cluster (distributed shared
//           memory), then one cluster barrier
//   pass 2  every warp merges the partials of its rows (Chan's parallel-variance formula: exact two-pass statistics,
//           no E[x^2] - mean^2 cancellation), normalises the staged z and stores y as bf16 and fp32; mean / rstd (fp32,
//           what the LayerNorm backward reads) are written by rank 0
#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

constexpr int kLnBM = 128, kLnBK = 64, kLnWgmmaK = 16;
constexpr int kLnBN = 256;                       // columns per CTA
constexpr int kLnThreads = 384;                  // producer warpgroup + two consumer warpgroups
constexpr int kLnEpiWarps = 8;                   // warps 4-11

template <int CL>   // CTAs per cluster = 256-column tiles per row: 3 (hidden 768) or 4 (hidden 1024)
struct GemmLnCfg {
  static constexpr int kCluster = CL;
  static constexpr int kABytes = kLnBM * kLnBK * 2;
  static constexpr int kBBytes = kLnBN * kLnBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;        // 48 KB
  static constexpr int kStages = 4;
  static constexpr int kPipeBytes = kStages * kStageBytes;
  static constexpr int kAccLd = kLnBN + 4;                     // fp32 row pitch of the accumulator / z tile
  static constexpr int kStatsBytes = CL * kLnBM * 8;           // [rank][row] float2 (mean, M2)
  static constexpr int kSmemBytes = kPipeBytes + kStatsBytes + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(kLnBM * kAccLd * 4 <= kPipeBytes, "the accumulator tile lives in the drained operand ring");
};

struct GemmLnParams {
  int M, N, kblocks;
  __nv_bfloat16* D; long long ldd;                 // pre-LayerNorm sum z, bf16 [M, N] (kept for the backward)
  const __nv_bfloat16* bias;
  const float* resid; long long ld_resid;          // residual input, FP32 [M, N]
  float dropout_p; const unsigned long long* rng; unsigned rng_site;
  const __nv_bfloat16* gamma; const __nv_bfloat16* beta; float eps;
  __nv_bfloat16* Y; long long ldy;                 // LayerNorm output, bf16 [M, N]: the next GEMM's operand
  float* Yf; long long ldyf;                       // LayerNorm output, fp32 [M, N]: the next block's residual (or null)
  float* mean; float* rstd;                        // fp32 [M]
};

__device__ __forceinline__ void unpack8(const uint4& t, float (&f)[8]) {
  f[0] = bf16_lo(t.x); f[1] = bf16_hi(t.x); f[2] = bf16_lo(t.y); f[3] = bf16_hi(t.y);
  f[4] = bf16_lo(t.z); f[5] = bf16_hi(t.z); f[6] = bf16_lo(t.w); f[7] = bf16_hi(t.w);
}

template <int CL>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(kLnThreads, 1)
gemm_ln_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmLnParams p) {
  using Cfg = GemmLnCfg<CL>;
  constexpr int BN = kLnBN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  float2* stats = reinterpret_cast<float2*>(smem + Cfg::kPipeBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kPipeBytes + Cfg::kStatsBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();            // 0 .. CL - 1: column tile of this CTA
  const int m0 = (blockIdx.x / CL) * kLnBM;
  const int n_tile = (int)rank * BN;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kLnEpiWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // PDL: nothing above touches global data
  pdl_wait();
  pdl_launch_dependents();

  if (warp == 0) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int kb = 0; kb < p.kblocks; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
        uint8_t* sa = smem + stage * Cfg::kStageBytes;
        tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * kLnBK, m0);                 // box {64 k, 128 rows}
        tma_load_2d(sa + Cfg::kABytes, &tmap_b, &full_bar[stage], kb * kLnBK, n_tile);   // box {64 k, 256 rows}
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------ wgmma consumers ------------------------------
    const int wg = (warp - 4) >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, prev = -1; uint32_t phase = 0;
    for (int kb = 0; kb < p.kblocks; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes) + wg * 8192;
      const uint32_t sb = smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kLnBK / kLnWgmmaK; ++k)
        wgmma_bf16<BN, 0, 0>(acc, make_smem_desc(sa + k * kLnWgmmaK * 2, 16, 1024),
                             make_smem_desc(sb + k * kLnWgmmaK * 2, 16, 1024), (kb > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    named_barrier_sync(1, kLnEpiWarps * 32);   // the ring is dead: the accumulator tile may overwrite it
    float* zs = reinterpret_cast<float*>(smem);
    {
      const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const int c = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<float2*>(zs + (size_t)r * Cfg::kAccLd + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(zs + (size_t)(r + 8) * Cfg::kAccLd + 8 * j + c) =
            make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    named_barrier_sync(1, kLnEpiWarps * 32);

    // ---- pass 1: warp e takes rows e, e + 8, ...; lane l columns [8 l, 8 l + 8) of the CTA's 256 ----
    const int ew = warp - 4;
    const int col = n_tile + 8 * lane;
    const DropCtx drop = make_drop_ctx(p.rng, p.rng_site, p.dropout_p);
    float b8[8];
    unpack8(*reinterpret_cast<const uint4*>(p.bias + col), b8);
#pragma unroll 1
    for (int r = ew; r < kLnBM; r += kLnEpiWarps) {
      const int m = m0 + r;
      float2 st = make_float2(0.f, 0.f);
      if (m < p.M) {                                  // warp-uniform
        float* zr = zs + (size_t)r * Cfg::kAccLd + 8 * lane;
        const float4 a0 = *reinterpret_cast<const float4*>(zr), a1 = *reinterpret_cast<const float4*>(zr + 4);
        const float* rp = p.resid + (size_t)m * p.ld_resid + col;
        const float4 r0 = *reinterpret_cast<const float4*>(rp), r1 = *reinterpret_cast<const float4*>(rp + 4);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float res[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
        const uint32_t keep = dropout_keep8(drop, (unsigned long long)m * p.N + col);
        float f[8];
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          f[i] = a[i] + b8[i];
          // (two roundings, as the unfused reference sequence dropout(...) + residual)
          f[i] = (((keep >> i) & 1u) ? f[i] * drop.scale : 0.f) + res[i];
          sum += f[i];
        }
        *reinterpret_cast<float4*>(zr) = make_float4(f[0], f[1], f[2], f[3]);
        *reinterpret_cast<float4*>(zr + 4) = make_float4(f[4], f[5], f[6], f[7]);
        uint4 o;
        o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
        *reinterpret_cast<uint4*>(p.D + (size_t)m * p.ldd + col) = o;          // bf16 z for the backward
        // partial statistics of the UNROUNDED z over this CTA's 256 columns (two passes over registers)
        const float mean_l = warp_sum(sum) * (1.0f / BN);
        float m2 = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) m2 = fmaf(f[i] - mean_l, f[i] - mean_l, m2);
        st = make_float2(mean_l, warp_sum(m2));
      }
      if (lane < CL) st_cluster_f32x2(mapa_u32(smem_u32(&stats[rank * kLnBM + r]), (uint32_t)lane), st.x, st.y);
    }
  }
  // every partial of every row of the cluster has been posted (release) and is visible (acquire); the producer
  // warpgroup takes part, as every thread of the cluster must
  cluster_sync_all();
  if (warp < 4) return;   // no CTA touches another's shared memory after the barrier: each may exit on its own

  // ---- pass 2 ----
  const int ew = warp - 4;
  const int col = n_tile + 8 * lane;
  float g8[8], e8[8];
  unpack8(*reinterpret_cast<const uint4*>(p.gamma + col), g8);
  unpack8(*reinterpret_cast<const uint4*>(p.beta + col), e8);
  const float* zs = reinterpret_cast<const float*>(smem);
#pragma unroll 1
  for (int r = ew; r < kLnBM; r += kLnEpiWarps) {
    const int m = m0 + r;
    if (m >= p.M) break;                              // rows ascend: the rest of this warp's rows are past M too
    // merge the CL partials of this row (equal counts BN): mean = avg(mean_i), M2 = sum M2_i + BN sum (mean_i - mean)^2
    float mean = 0.f;
#pragma unroll
    for (int i = 0; i < CL; ++i) mean += stats[i * kLnBM + r].x;
    mean *= 1.0f / CL;
    float m2 = 0.f;
#pragma unroll
    for (int i = 0; i < CL; ++i) {
      const float2 t = stats[i * kLnBM + r];
      const float d = t.x - mean;
      m2 += t.y + (float)BN * d * d;
    }
    const float rstd = rsqrtf(m2 / (float)p.N + p.eps);
    const float* zr = zs + (size_t)r * Cfg::kAccLd + 8 * lane;
    const float4 z0 = *reinterpret_cast<const float4*>(zr), z1 = *reinterpret_cast<const float4*>(zr + 4);
    float f[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = (f[i] - mean) * rstd * g8[i] + e8[i];
    uint4 o;
    o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
    *reinterpret_cast<uint4*>(p.Y + (size_t)m * p.ldy + col) = o;
    if (p.Yf != nullptr) {
      float* yf = p.Yf + (size_t)m * p.ldyf + col;
      *reinterpret_cast<float4*>(yf) = make_float4(f[0], f[1], f[2], f[3]);
      *reinterpret_cast<float4*>(yf + 4) = make_float4(f[4], f[5], f[6], f[7]);
    }
    if (rank == 0 && lane == 0) {
      p.mean[m] = mean;
      p.rstd[m] = rstd;
    }
  }
}

template <int CL>
static int32_t gemm_ln_prepare() {
  static int state = 0;    // 0 = not yet, 1 = ready, -1 = failed
  if (state == 0) {
    auto kern = gemm_ln_kernel<CL>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmLnCfg<CL>::kSmemBytes) !=
        cudaSuccess) {
      (void)cudaGetLastError();
      state = -1;
    } else {
      state = 1;
    }
  }
  return state;
}

template <int CL>
static int32_t gemm_ln_max_clusters() {
  if (gemm_ln_prepare<CL>() != 1) return 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(GemmLnCfg<CL>::kCluster);
  cfg.blockDim = dim3(kLnThreads);
  cfg.dynamicSmemBytes = GemmLnCfg<CL>::kSmemBytes;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = GemmLnCfg<CL>::kCluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, gemm_ln_kernel<CL>, &cfg) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  return n;
}

template <int CL>
static int32_t launch_gemm_ln(const b2_gemm_args_t& a, const void* gamma, const void* beta, float eps, void* y,
                              int64_t ldy, float* y_f32, int64_t ldyf, float* mean, float* rstd,
                              cudaStream_t stream) {
  using Cfg = GemmLnCfg<CL>;
  B2_REQUIRE(gemm_ln_prepare<CL>() == 1, "b2_gemm_ln_fwd: cannot reserve %d bytes of shared memory",
             Cfg::kSmemBytes);
  CUtensorMap ta, tb;
  int32_t st = get_tensor_map_2d(&ta, a.A, (uint64_t)a.M, (uint64_t)a.K, (uint64_t)a.lda * 2, kLnBM, 64);
  if (st) return st;
  st = get_tensor_map_2d(&tb, a.B, (uint64_t)a.N, (uint64_t)a.K, (uint64_t)a.ldb * 2, kLnBN, 64);
  if (st) return st;
  GemmLnParams p;
  p.M = (int)a.M; p.N = (int)a.N; p.kblocks = (int)((a.K + kLnBK - 1) / kLnBK);
  p.D = (__nv_bfloat16*)a.D; p.ldd = a.ldd;
  p.bias = (const __nv_bfloat16*)a.bias;
  p.resid = (const float*)a.aux_in; p.ld_resid = a.ld_aux_in;
  p.dropout_p = a.dropout_p; p.rng = (const unsigned long long*)a.rng_state; p.rng_site = a.rng_site;
  p.gamma = (const __nv_bfloat16*)gamma; p.beta = (const __nv_bfloat16*)beta; p.eps = eps;
  p.Y = (__nv_bfloat16*)y; p.ldy = ldy; p.Yf = y_f32; p.ldyf = ldyf; p.mean = mean; p.rstd = rstd;
  const int row_blocks = (int)((a.M + kLnBM - 1) / kLnBM);
  B2_LAUNCH(gemm_ln_kernel<CL>, Cfg::kCluster * row_blocks, kLnThreads, Cfg::kSmemBytes, stream, ta, tb, p);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace b2

using namespace b2;

extern "C" int32_t b2_gemm_ln_max_clusters(int64_t hidden) {
  if (hidden == 768) return gemm_ln_max_clusters<3>();
  if (hidden == 1024) return gemm_ln_max_clusters<4>();
  return 0;
}

extern "C" int32_t b2_gemm_ln_fwd(const b2_gemm_args_t* a, const void* gamma, const void* beta, float eps, void* y,
                                  int64_t ldy, float* y_f32, int64_t ldyf, float* mean, float* rstd, void* stream_) {
  B2_REQUIRE(a != nullptr, "b2_gemm_ln_fwd: null args");
  B2_REQUIRE(a->M > 0 && a->K > 0, "b2_gemm_ln_fwd: empty problem");
  B2_REQUIRE(a->N == 768 || a->N == 1024, "b2_gemm_ln_fwd: N=%lld: the row cluster covers hidden sizes 768 and 1024",
             (long long)a->N);
  B2_REQUIRE(a->a_major == B2_MAJOR_K && a->b_major == B2_MAJOR_K, "b2_gemm_ln_fwd: NT layout only (y = x W^T)");
  B2_REQUIRE(a->epilogue == B2_EPI_BIAS_DROPOUT_RESIDUAL, "b2_gemm_ln_fwd: epilogue must be BIAS_DROPOUT_RESIDUAL");
  B2_REQUIRE(a->A && a->B && a->D && a->bias && a->aux_in && gamma && beta && y && mean && rstd,
             "b2_gemm_ln_fwd: null pointer");
  // arguments of b2_gemm_bf16 this kernel has no use for: an error rather than a silent no-op
  B2_REQUIRE(a->colsum_out == nullptr, "b2_gemm_ln_fwd: the fused kernel takes no column sums: colsum_out must be NULL");
  B2_REQUIRE(a->aux_out == nullptr, "b2_gemm_ln_fwd: the fused kernel writes no aux_out: aux_out must be NULL");
  B2_REQUIRE(a->force_splits <= 1, "b2_gemm_ln_fwd: force_splits=%d: the fused kernel does not split K",
             (int)a->force_splits);
  B2_REQUIRE(a->force_bn == 0 || a->force_bn == 256, "b2_gemm_ln_fwd: force_bn=%d: the fused kernel's tiles are 256 "
             "wide", (int)a->force_bn);
  B2_REQUIRE(a->workspace == nullptr, "b2_gemm_ln_fwd: the fused kernel needs no workspace: workspace must be NULL");
  // a leading dimension shorter than its row would make rows overlap
  B2_REQUIRE(a->lda >= a->K, "b2_gemm_ln_fwd: lda=%lld is below K=%lld", (long long)a->lda, (long long)a->K);
  B2_REQUIRE(a->ldb >= a->K, "b2_gemm_ln_fwd: ldb=%lld is below K=%lld", (long long)a->ldb, (long long)a->K);
  B2_REQUIRE(a->ldd >= a->N, "b2_gemm_ln_fwd: ldd=%lld is below N=%lld", (long long)a->ldd, (long long)a->N);
  B2_REQUIRE(a->ld_aux_in >= a->N, "b2_gemm_ln_fwd: ld_aux_in=%lld is below N=%lld", (long long)a->ld_aux_in,
             (long long)a->N);
  B2_REQUIRE(ldy >= a->N, "b2_gemm_ln_fwd: ldy=%lld is below N=%lld", (long long)ldy, (long long)a->N);
  B2_REQUIRE(y_f32 == nullptr || ldyf >= a->N, "b2_gemm_ln_fwd: ldyf=%lld is below N=%lld", (long long)ldyf,
             (long long)a->N);
  B2_REQUIRE(a->K % 8 == 0 && a->lda % 8 == 0 && a->ldb % 8 == 0 && a->ldd % 8 == 0 && a->ld_aux_in % 4 == 0 &&
                 ldy % 8 == 0 && (y_f32 == nullptr || ldyf % 4 == 0),
             "b2_gemm_ln_fwd: K and leading dimensions must be multiples of 16 bytes");
  B2_REQUIRE(((uintptr_t)a->A % 16 == 0) && ((uintptr_t)a->B % 16 == 0) && ((uintptr_t)a->D % 16 == 0) &&
                 ((uintptr_t)a->aux_in % 16 == 0) && ((uintptr_t)y % 16 == 0) && ((uintptr_t)y_f32 % 16 == 0) &&
                 ((uintptr_t)a->bias % 16 == 0) && ((uintptr_t)gamma % 16 == 0) && ((uintptr_t)beta % 16 == 0),
             "b2_gemm_ln_fwd: operands must be 16-byte aligned");
  B2_REQUIRE(a->dropout_p >= 0.f && a->dropout_p < 1.f, "b2_gemm_ln_fwd: dropout_p out of range");
  B2_REQUIRE(!(a->dropout_p > 0.f) || a->rng_state != nullptr, "b2_gemm_ln_fwd: dropout needs rng_state");
  if (a->N == 768)
    return launch_gemm_ln<3>(*a, gamma, beta, eps, y, ldy, y_f32, ldyf, mean, rstd, (cudaStream_t)stream_);
  return launch_gemm_ln<4>(*a, gamma, beta, eps, y, ldy, y_f32, ldyf, mean, rstd, (cudaStream_t)stream_);
}
