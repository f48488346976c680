// bf16 GEMM on the Hopper tensor cores (wgmma): D[M,N] = op(A) * op(B) (+ fused epilogue), fp32 accumulate.
//
// Replaces the cuBLAS `addmm` calls issued by HF BertSelfAttention / BertSelfOutput / BertIntermediate /
// BertOutput (transformers modeling_bert.py:179-181, :295, :340, :353) and their autograd dgrad / wgrad
// twins (SURVEY.md §2.2 K2, K7, K8, K9).
//
// Two kernels share one mainloop and one epilogue:
//   gemm_bf16_kernel         one 128 x BN output tile (BN 128 / 256) per CTA, optional split-K over the contraction
//   gemm_grouped_tn_kernel   a table of up to four TN problems behind one launch: the weight gradients of one encoder
//                            layer (b2_gemm_bf16_grouped), optionally with the AdamW update fused into the epilogue
// CTA structure (384 threads, warp specialised):
//   warpgroup 0 (warps 0-3)    warp 0 lane 0: TMA producer, global -> 128B-swizzled smem ring (full/empty mbarriers)
//   warpgroups 1, 2 (4-11)     wgmma consumers, rows 0-63 / 64-127 of the tile, fp32 accumulators in registers; once
//                              the contraction is done the ring is dead, the accumulators go to shared memory (row
//                              major, over the ring) and the same 8 warps run the epilogue (gemm_epilogue.cuh)
// Operand layouts are expressed only through the TMA box + wgmma descriptor (no transposes in HBM):
//   NT  A[M,K] K-major,  B[N,K] K-major   (forward:  y = x W^T)
//   NN  A[M,K] K-major,  B[K,N] MN-major  (dgrad:    dx = dy W)
//   TN  A[K,M] MN-major, B[K,N] MN-major  (wgrad:    dW = dy^T x), optional split-K over the token axis
#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int WGMMA_K = 16;
constexpr int kGemmThreads = (4 + kEpiWarps) * 32;   // producer warpgroup + two consumer warpgroups

template <int BN>
struct GemmCfg {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (BN == 256) ? 4 : 6;
  static constexpr int kPipeBytes = kStages * kStageBytes;             // 192 KB
  static constexpr int kAccLd = BN + 4;                                 // fp32 row pitch of the accumulator tile
  static constexpr int kSmemBytes = kPipeBytes + kEpiWarps * kEpiStageBytes + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(BM * kAccLd * 4 <= kPipeBytes, "the accumulator tile lives in the drained operand ring");
};

// Contraction over k-blocks [kb0, kb1) of the tile at (m0, n0).  Warp 0 loads, warps 4-11 multiply; on return the
// consumer warps hold the fp32 tile in shared memory at `smem` (row pitch GemmCfg<BN>::kAccLd) and have synchronised.
template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void gemm_mainloop(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                              const CUtensorMap* tmap_a, const CUtensorMap* tmap_b, int m0, int n0,
                                              int kb0, int kb1, int warp, int lane) {
  using Cfg = GemmCfg<BN>;
  if (warp == 0) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
        uint8_t* sa = smem + stage * Cfg::kStageBytes;
        uint8_t* sb = sa + Cfg::kABytes;
        const int k0 = kb * BK;
        if (!A_MN) {
          tma_load_2d(sa, tmap_a, &full_bar[stage], k0, m0);              // box {64 k, 128 rows}
        } else {
#pragma unroll
          for (int j = 0; j < BM / 64; ++j)                                // box {64 m, 64 k-rows}
            tma_load_2d(sa + j * (BK * 128), tmap_a, &full_bar[stage], m0 + 64 * j, k0);
        }
        if (!B_MN) {
          tma_load_2d(sb, tmap_b, &full_bar[stage], k0, n0);              // box {64 k, BN rows}
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            tma_load_2d(sb + j * (BK * 128), tmap_b, &full_bar[stage], n0 + 64 * j, k0);
        }
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------ wgmma consumers ------------------------------
    const int wg = (warp - 4) >> 2;             // rows [64 wg, 64 wg + 64) of the tile
    constexpr uint32_t a_lbo = A_MN ? BK * 128 : 16, b_lbo = B_MN ? BK * 128 : 16;
    constexpr uint32_t a_kstep = A_MN ? WGMMA_K * 128 : WGMMA_K * 2;
    constexpr uint32_t b_kstep = B_MN ? WGMMA_K * 128 : WGMMA_K * 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, prev = -1; uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      // K-major A: the warpgroup's 64 rows start 64 x 128 B in; MN-major A: its 64 columns are the second slab
      const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes) + wg * 8192;
      const uint32_t sb = smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WGMMA_K; ++k)
        wgmma_bf16<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, make_smem_desc(sa + k * a_kstep, a_lbo, 1024),
                                                     make_smem_desc(sb + k * b_kstep, b_lbo, 1024),
                                                     (kb > kb0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();                            // the previous k-block's products are done: release its stage
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    // every consumer warp is past its last product and every TMA write has been consumed: the ring is dead
    named_barrier_sync(1, kEpiWarps * 32);
    float* accs = reinterpret_cast<float*>(smem);
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(accs + (size_t)r * Cfg::kAccLd + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(accs + (size_t)(r + 8) * Cfg::kAccLd + 8 * j + c) =
          make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    named_barrier_sync(1, kEpiWarps * 32);
  }
}

template <int BN>
__device__ __forceinline__ void gemm_setup(uint64_t* full_bar, uint64_t* empty_bar) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < GemmCfg<BN>::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kEpiWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();
}

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const GemmKernelParams p) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  uint8_t* epi_stage = smem + Cfg::kPipeBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi_stage + kEpiWarps * kEpiStageBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
  }
  gemm_setup<BN>(full_bar, empty_bar);
  // PDL: everything above touches no global data and may overlap the predecessor's tail
  pdl_wait();
  pdl_launch_dependents();

  const int tile = blockIdx.x / p.splits, split = blockIdx.x % p.splits;
  const int m0 = (tile / p.tiles_n) * BM, n0 = (tile % p.tiles_n) * BN;
  const int kb0 = split * p.kblocks_per_split;
  const int kb1 = min(kb0 + p.kblocks_per_split, p.kblocks_total);
  gemm_mainloop<BN, A_MN, B_MN>(smem, full_bar, empty_bar, &tmap_a, &tmap_b, m0, n0, kb0, kb1, warp, lane);
  if (warp >= 4) {
    const DropCtx drop = make_drop_ctx(p.rng, p.rng_site, p.dropout_p);
    epilogue_tile<BN>(p, drop, reinterpret_cast<const float*>(smem), Cfg::kAccLd, warp, lane, m0, n0, split,
                      epi_stage + (warp - 4) * kEpiStageBytes);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Grouped kernel: up to kMaxGroup independent TN problems (D_i[M_i,N_i] = A_i^T B_i, both operands MN-major, same
// contraction length) behind ONE launch.  This is the weight-gradient step of an encoder layer: its four GEMMs are
// small, so launched one by one each pays a launch's fixed cost and needs split-K partials plus a reduce kernel to
// fill the machine.  Mainloop and epilogue are those of gemm_bf16_kernel; only the work decode differs.
// ------------------------------------------------------------------------------------------------------------
constexpr int kMaxGroup = 4;
struct GroupedProblem {
  int M, N, tiles_n, tile_begin;   // tile_begin: first global work index of this problem
  __nv_bfloat16* D; long long ldd;
};
struct GroupedParams {
  int count, num_work, kblocks;
  GroupedProblem pr[kMaxGroup];
};

struct GroupedMaps {
  CUtensorMap a[kMaxGroup], b[kMaxGroup];
};
__device__ __forceinline__ int grouped_find(const GroupedParams& gp, int w) {
  int pi = 0;
#pragma unroll
  for (int i = 1; i < kMaxGroup; ++i)
    if (i < gp.count && w >= gp.pr[i].tile_begin) pi = i;
  return pi;
}

__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_grouped_tn_kernel(const __grid_constant__ GroupedMaps maps, const GroupedParams gp) {
  constexpr int BN = 256;
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  uint8_t* epi_stage = smem + Cfg::kPipeBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi_stage + kEpiWarps * kEpiStageBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int pi = grouped_find(gp, blockIdx.x);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.a[pi]);
    tma_prefetch_desc(&maps.b[pi]);
  }
  gemm_setup<BN>(full_bar, empty_bar);
  pdl_wait();
  pdl_launch_dependents();

  const GroupedProblem& pr = gp.pr[pi];
  const int lt = blockIdx.x - pr.tile_begin;
  const int m0 = (lt / pr.tiles_n) * BM;
  const int n0 = (lt % pr.tiles_n) * BN;
  gemm_mainloop<BN, true, true>(smem, full_bar, empty_bar, &maps.a[pi], &maps.b[pi], m0, n0, 0, gp.kblocks, warp,
                                lane);
  if (warp < 4) return;
  uint8_t* stage = epi_stage + (warp - 4) * kEpiStageBytes;
  GemmKernelParams q;
  q.splits = 1; q.epilogue = B2_EPI_NONE; q.bias = nullptr; q.aux_in = nullptr; q.aux_out = nullptr;
  q.partial = nullptr; q.dropout_p = 0.f; q.rng = nullptr; q.rng_site = 0; q.timing = nullptr; q.colsum = nullptr;
  q.ld_aux_in = 0; q.ld_aux_out = 0; q.K = 0; q.tiles_m = 0; q.kblocks_per_split = 0; q.kblocks_total = 0;
  q.M = pr.M; q.N = pr.N; q.tiles_n = pr.tiles_n; q.D = pr.D; q.ldd = pr.ldd;
  DropCtx drop;
  drop.k0 = 0; drop.k1 = 0; drop.step = 0; drop.site = 0; drop.thresh = 0; drop.scale = 1.f;
  epilogue_tile<BN>(q, drop, reinterpret_cast<const float*>(smem), Cfg::kAccLd, warp, lane, m0, n0, 0, stage);
}

// sums split-K partials [splits][M][N] fp32 -> bf16 D
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, __nv_bfloat16* __restrict__ D,
                                     long long ldd, int M, int N, int splits) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // one float4 (4 columns) each
  const long long total = (long long)M * N / 4;
  if (idx >= total) return;
  const long long e = idx * 4;
  const int m = (int)(e / N), n = (int)(e % N);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s = 0; s < splits; ++s) {
    const float4 v = *reinterpret_cast<const float4*>(partial + (size_t)s * M * N + e);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  uint2 o;
  o.x = pack_bf16(acc.x, acc.y);
  o.y = pack_bf16(acc.z, acc.w);
  *reinterpret_cast<uint2*>(D + (size_t)m * ldd + n) = o;
}

static int g_num_sms = 0;
static int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

static void fill_params(GemmKernelParams& p, const b2_gemm_args_t& a, int tile_m, int bn, int splits) {
  p.M = (int)a.M; p.N = (int)a.N; p.K = (int)a.K;
  p.tiles_m = (p.M + tile_m - 1) / tile_m;
  p.tiles_n = (p.N + bn - 1) / bn;
  p.kblocks_total = (p.K + BK - 1) / BK;
  p.splits = splits;
  p.kblocks_per_split = (p.kblocks_total + splits - 1) / splits;
  p.epilogue = (splits > 1 && a.epilogue != B2_EPI_ACCUM_F32) ? B2_EPI_PARTIAL_F32 : a.epilogue;
  p.D = (__nv_bfloat16*)a.D; p.ldd = a.ldd;
  p.bias = (const __nv_bfloat16*)a.bias;
  p.aux_in = (const __nv_bfloat16*)a.aux_in; p.ld_aux_in = a.ld_aux_in;
  p.aux_out = (__nv_bfloat16*)a.aux_out; p.ld_aux_out = a.ld_aux_out;
  p.partial = (float*)a.workspace;
  p.dropout_p = a.dropout_p; p.rng = (const unsigned long long*)a.rng_state; p.rng_site = a.rng_site;
  p.timing = (long long*)a.debug_timing;
  p.colsum = a.colsum_out;
}

static int32_t launch_splitk_reduce(const b2_gemm_args_t& a, int splits, cudaStream_t stream) {
  const long long total = (long long)a.M * a.N / 4;
  B2_LAUNCH(splitk_reduce_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, 
      (const float*)a.workspace, (__nv_bfloat16*)a.D, a.ldd, (int)a.M, (int)a.N, splits);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

template <int BN, bool A_MN, bool B_MN>
static int32_t launch_gemm(const b2_gemm_args_t& a, int splits, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  CUtensorMap ta, tb;
  int32_t st;
  if (!A_MN) st = get_tensor_map_2d(&ta, a.A, (uint64_t)a.M, (uint64_t)a.K, (uint64_t)a.lda * 2, BM, 64);
  else       st = get_tensor_map_2d(&ta, a.A, (uint64_t)a.K, (uint64_t)a.M, (uint64_t)a.lda * 2, BK, 64);
  if (st) return st;
  if (!B_MN) st = get_tensor_map_2d(&tb, a.B, (uint64_t)a.N, (uint64_t)a.K, (uint64_t)a.ldb * 2, BN, 64);
  else       st = get_tensor_map_2d(&tb, a.B, (uint64_t)a.K, (uint64_t)a.N, (uint64_t)a.ldb * 2, BK, 64);
  if (st) return st;
  GemmKernelParams p;
  fill_params(p, a, BM, BN, splits);
  auto kern = gemm_bf16_kernel<BN, A_MN, B_MN>;
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  const int work = p.tiles_m * p.tiles_n * p.splits;   // one tile (or split-K slice of one) per CTA
  B2_LAUNCH(kern, work, kGemmThreads, Cfg::kSmemBytes, stream, ta, tb, p);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  if (splits > 1 && a.epilogue != B2_EPI_ACCUM_F32) return launch_splitk_reduce(a, splits, stream);
  return 0;
}

// Tile-width / split-K choice.  Cost model per candidate: waves of CTAs x per-k-block time, where the k-block time
// is the larger of the tensor-pipe time (~2048 bf16 FMA per SM and cycle) and the L2->SM feed time.
struct Choice { int bn, splits; };
static Choice choose_config(const b2_gemm_args_t& a) {
  const int sms = num_sms();
  const int kblocks = (int)((a.K + BK - 1) / BK);
  const bool accum = a.epilogue == B2_EPI_ACCUM_F32;   // split-K slices add in place: no workspace, any split count
  // the split-K partials path has no column sums: a problem with colsum_out runs whole tiles
  const bool can_split = accum || ((a.epilogue == B2_EPI_NONE) && a.workspace != nullptr && a.bias == nullptr &&
                                   a.colsum_out == nullptr);
  double best = 1e30;
  Choice c{128, 1};
  const double l2_bytes_per_cycle = 3000.0;   // L2 -> SM bandwidth shared by the busy SMs, bytes per SM clock
  const int bns[2] = {256, 128};
  for (int bi = 0; bi < 2; ++bi) {
    const int bn = bns[bi];
    if (a.N % bn != 0 && bn != 128) continue;
    const int tiles = (int)((a.M + BM - 1) / BM) * (int)((a.N + bn - 1) / bn);
    const int max_s = can_split ? 8 : 1;
    for (int s = 1; s <= max_s; s = accum ? s + 1 : s * 2) {
      if (s > 1 && (kblocks / s < 8)) break;
      if (s > 1 && !accum && (size_t)s * a.M * a.N * 4 > (size_t)a.workspace_bytes) break;
      const int work = tiles * s;
      const int rounds = (work + sms - 1) / sms;
      const int busy_sms = work < sms ? work : sms;
      const double mma_cycles = 128.0 * bn * 64 / 2048.0;                    // per SM, per k-block
      const double bytes_per_sm = (128 + bn) * 128.0;
      const double feed_cycles = bytes_per_sm * busy_sms / l2_bytes_per_cycle;
      const double kb_cycles = mma_cycles > feed_cycles ? mma_cycles : feed_cycles;
      double t = rounds * ((double)((kblocks + s - 1) / s) * kb_cycles + 2500.0 /*prologue + epilogue tail*/);
      if (s > 1 && !accum) t += 1500.0 + (double)s * a.M * a.N * 8 / 3000.0;  // partial write + reduce pass
      if (s > 1 && accum) t += (double)(s - 1) * a.M * a.N * 4 / 3000.0;      // extra reduction traffic at L2
      if (t < best) { best = t; c = Choice{bn, s}; }
    }
  }
  return c;
}

}  // namespace b2

using namespace b2;

// Every argument check of b2_gemm_bf16, host-only (no device access), so that the grouped entry point can reject a
// table before it launches any of it.  An argument an epilogue would not read is an error, not a silent no-op.
static int32_t check_args(const b2_gemm_args_t* a) {
  B2_REQUIRE(a != nullptr, "b2_gemm_bf16: null args");
  B2_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "b2_gemm_bf16: empty problem M=%lld N=%lld K=%lld",
             (long long)a->M, (long long)a->N, (long long)a->K);
  B2_REQUIRE(a->A && a->B && a->D, "b2_gemm_bf16: null operand pointer");
  B2_REQUIRE(a->N % 64 == 0, "b2_gemm_bf16: N=%lld must be a multiple of 64", (long long)a->N);
  B2_REQUIRE(a->K % 8 == 0 && a->lda % 8 == 0 && a->ldb % 8 == 0 && a->ldd % 8 == 0,
             "b2_gemm_bf16: K and leading dimensions must be multiples of 8 elements (16 B)");
  B2_REQUIRE(((uintptr_t)a->A % 16 == 0) && ((uintptr_t)a->B % 16 == 0) && ((uintptr_t)a->D % 16 == 0),
             "b2_gemm_bf16: operands must be 16-byte aligned");
  // a leading dimension shorter than its row would make rows overlap: stores race, loads read the wrong elements
  const int64_t a_row = a->a_major == B2_MAJOR_MN ? a->M : a->K, b_row = a->b_major == B2_MAJOR_MN ? a->N : a->K;
  B2_REQUIRE(a->lda >= a_row, "b2_gemm_bf16: lda=%lld is below the row it describes (%lld)", (long long)a->lda,
             (long long)a_row);
  B2_REQUIRE(a->ldb >= b_row, "b2_gemm_bf16: ldb=%lld is below the row it describes (%lld)", (long long)a->ldb,
             (long long)b_row);
  B2_REQUIRE(a->ldd >= a->N, "b2_gemm_bf16: ldd=%lld is below N=%lld", (long long)a->ldd, (long long)a->N);
  const int e = a->epilogue;
  B2_REQUIRE(e >= B2_EPI_NONE && e <= B2_EPI_ACCUM_F32, "b2_gemm_bf16: bad epilogue %d", e);
  const bool with_bias = e == B2_EPI_BIAS || e == B2_EPI_BIAS_GELU || e == B2_EPI_BIAS_DROPOUT_RESIDUAL;
  const bool f32_out = e == B2_EPI_RESIDUAL_F32 || e == B2_EPI_ACCUM_F32;
  if (with_bias) B2_REQUIRE(a->bias != nullptr, "b2_gemm_bf16: epilogue %d needs a bias", e);
  else           B2_REQUIRE(a->bias == nullptr, "b2_gemm_bf16: epilogue %d adds no bias: bias must be NULL", e);
  // the epilogues that read aux_in / write aux_out need a full row of it; elsewhere its ld is not read (0 is fine)
  if (e == B2_EPI_BIAS_DROPOUT_RESIDUAL || e == B2_EPI_RESIDUAL || e == B2_EPI_GELU_BWD || e == B2_EPI_RESIDUAL_F32) {
    B2_REQUIRE(a->aux_in != nullptr && a->ld_aux_in % 8 == 0, "b2_gemm_bf16: epilogue %d needs aux_in", e);
    B2_REQUIRE(a->ld_aux_in >= a->N, "b2_gemm_bf16: ld_aux_in=%lld is below N=%lld", (long long)a->ld_aux_in,
               (long long)a->N);
  }
  if (e == B2_EPI_BIAS_GELU) {
    B2_REQUIRE(a->aux_out != nullptr && a->ld_aux_out % 8 == 0, "b2_gemm_bf16: BIAS_GELU needs aux_out");
    B2_REQUIRE(a->ld_aux_out >= a->N, "b2_gemm_bf16: ld_aux_out=%lld is below N=%lld", (long long)a->ld_aux_out,
               (long long)a->N);
  } else
    B2_REQUIRE(a->aux_out == nullptr, "b2_gemm_bf16: only BIAS_GELU writes aux_out: aux_out must be NULL");
  // bias, aux_in and aux_out move in 16-byte vectors (ldg16, cp.async, uint4 stores)
  B2_REQUIRE((uintptr_t)a->bias % 16 == 0, "b2_gemm_bf16: bias must be 16-byte aligned");
  B2_REQUIRE((uintptr_t)a->aux_in % 16 == 0, "b2_gemm_bf16: aux_in must be 16-byte aligned");
  B2_REQUIRE((uintptr_t)a->aux_out % 16 == 0, "b2_gemm_bf16: aux_out must be 16-byte aligned");
  B2_REQUIRE(a->dropout_p >= 0.f && a->dropout_p < 1.f, "b2_gemm_bf16: dropout_p out of range");
  if (e == B2_EPI_BIAS_DROPOUT_RESIDUAL && a->dropout_p > 0.f)
    B2_REQUIRE(a->rng_state != nullptr, "b2_gemm_bf16: dropout needs rng_state");
  if (e != B2_EPI_BIAS_DROPOUT_RESIDUAL)
    B2_REQUIRE(a->dropout_p == 0.f, "b2_gemm_bf16: epilogue %d applies no dropout: dropout_p must be 0", e);
  // column sums are taken in the bf16 epilogue of a whole (unsplit) tile
  B2_REQUIRE(a->colsum_out == nullptr || !f32_out, "b2_gemm_bf16: epilogue %d has no bf16 output: colsum_out must be "
             "NULL", e);
  B2_REQUIRE(a->colsum_out == nullptr || a->force_splits <= 1, "b2_gemm_bf16: colsum_out needs force_splits <= 1");
  if (a->force_bn == 128 || a->force_bn == 256)
    B2_REQUIRE(a->N % a->force_bn == 0 || a->force_bn == 128, "b2_gemm_bf16: force_bn does not divide N");
  if (a->force_splits > 1)
    B2_REQUIRE(e == B2_EPI_ACCUM_F32 ||
                   (e == B2_EPI_NONE && a->workspace &&
                    (size_t)a->force_splits * a->M * a->N * 4 <= (size_t)a->workspace_bytes),
               "b2_gemm_bf16: split-K needs EPI_ACCUM_F32, or EPI_NONE and a large enough workspace");
  B2_REQUIRE(!(a->a_major == B2_MAJOR_MN && a->b_major != B2_MAJOR_MN),
             "b2_gemm_bf16: layout TT (A MN-major, B K-major) is not on the path");
  return 0;
}

// one problem that has passed check_args: pick the configuration and launch
static int32_t launch_checked(const b2_gemm_args_t* a, cudaStream_t stream) {
  Choice c = choose_config(*a);
  // force_kernel (1 / 2) selects between kernels on other builds; this one has a single GEMM kernel
  if (a->force_bn == 128 || a->force_bn == 256) c.bn = a->force_bn;
  if (a->force_splits >= 1) c.splits = a->force_splits;
  const bool a_mn = a->a_major == B2_MAJOR_MN, b_mn = a->b_major == B2_MAJOR_MN;

#define B2_DISPATCH(BN_)                                                          \
  if (c.bn == BN_) {                                                              \
    if (!a_mn && !b_mn) return launch_gemm<BN_, false, false>(*a, c.splits, stream); \
    if (!a_mn && b_mn) return launch_gemm<BN_, false, true>(*a, c.splits, stream);   \
    return launch_gemm<BN_, true, true>(*a, c.splits, stream);                       \
  }
  B2_DISPATCH(128)
  B2_DISPATCH(256)
#undef B2_DISPATCH
  set_error("b2_gemm_bf16: no kernel for BN=%d", c.bn);
  return -2;
}

extern "C" int32_t b2_gemm_bf16(const b2_gemm_args_t* a, void* stream_) {
  const int32_t st = check_args(a);
  if (st) return st;
  return launch_checked(a, (cudaStream_t)stream_);
}

extern "C" int32_t b2_gemm_bf16_grouped(const b2_gemm_args_t* args, int32_t count, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  B2_REQUIRE(args != nullptr && count >= 1, "b2_gemm_bf16_grouped: no problems");
  for (int i = 0; i < count; ++i) {   // reject the whole table before any of it runs
    const int32_t st = check_args(&args[i]);
    if (st) return st;
  }
  // the one-launch path covers what the weight-gradient step needs: TN layouts, plain bf16 output, 256-wide tiles,
  // one contraction length; anything else is issued problem by problem (same results, more launches).  Every
  // problem has passed check_args, so only the tiling conditions are left to test here.
  bool groupable = count <= kMaxGroup;
  for (int i = 0; i < count && groupable; ++i) {
    const b2_gemm_args_t& a = args[i];
    groupable = a.a_major == B2_MAJOR_MN && a.b_major == B2_MAJOR_MN && a.epilogue == B2_EPI_NONE &&
                a.colsum_out == nullptr && a.N % 256 == 0 && a.K == args[0].K && a.force_splits <= 1 &&
                (a.force_bn == 0 || a.force_bn == 256);
  }
  if (!groupable) {
    for (int i = 0; i < count; ++i) {
      const int32_t st = launch_checked(&args[i], stream);
      if (st) return st;
    }
    return 0;
  }
  GroupedMaps maps;
  GroupedParams gp;
  gp.count = count;
  gp.kblocks = (int)((args[0].K + BK - 1) / BK);
  int work = 0;
  for (int i = 0; i < count; ++i) {
    const b2_gemm_args_t& a = args[i];
    int32_t st = get_tensor_map_2d(&maps.a[i], a.A, (uint64_t)a.K, (uint64_t)a.M, (uint64_t)a.lda * 2, BK, 64);
    if (st) return st;
    st = get_tensor_map_2d(&maps.b[i], a.B, (uint64_t)a.K, (uint64_t)a.N, (uint64_t)a.ldb * 2, BK, 64);
    if (st) return st;
    GroupedProblem& g = gp.pr[i];
    g.M = (int)a.M; g.N = (int)a.N; g.tiles_n = (int)(a.N / 256); g.tile_begin = work;
    g.D = (__nv_bfloat16*)a.D; g.ldd = a.ldd;
    work += (int)((a.M + BM - 1) / BM) * g.tiles_n;
  }
  for (int i = count; i < kMaxGroup; ++i) { gp.pr[i] = gp.pr[0]; gp.pr[i].tile_begin = 0x7fffffff; maps.a[i] = maps.a[0]; maps.b[i] = maps.b[0]; }
  gp.num_work = work;
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(gemm_grouped_tn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 GemmCfg<256>::kSmemBytes));
    attr_set = true;
  }
  B2_LAUNCH(gemm_grouped_tn_kernel, work, kGemmThreads, GemmCfg<256>::kSmemBytes, stream, maps, gp);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}
