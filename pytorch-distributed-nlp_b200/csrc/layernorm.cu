// LayerNorm forward / backward and column sums: HBM-bound, 16-byte vector accesses, fp32 statistics.  Forward and the
// generic backward: one warp per row.  The training engine's backward (layernorm_bwd_pair_kernel): a warp PAIR per
// row with cp.async operand rings, column sums added straight into caller-owned fp32 accumulators.  Replaces ATen native_layer_norm (+backward) issued by BertSelfOutput / BertOutput
// (SP/transformers/models/bert/modeling_bert.py:297, :355) and the bias-gradient reductions autograd runs
// for the dense layers (SURVEY.md §2.2 K7, K9).
#include "common.cuh"
#include "layernorm.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

template <int VPL>
__global__ void __launch_bounds__(128) layernorm_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                           const __nv_bfloat16* __restrict__ gamma,
                                                           const __nv_bfloat16* __restrict__ beta, int rows, float eps,
                                                           __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out,
                                                           float* __restrict__ rstd_out) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  constexpr int H = VPL * 256;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float v[VPL * 8];
  load_row<VPL>(x + (size_t)row * H, lane, v);
  float mean, rstd;
  row_stats<VPL>(v, eps, mean, rstd);
  normalize_store<VPL>(v, mean, rstd, gamma, beta, lane, y + (size_t)row * H);
  if (lane == 0) {
    mean_out[row] = mean;
    rstd_out[row] = rstd;
  }
}

// mode 0: dropout mask (if any) applies to the LN *input* branch -> emit dx_drop = dx*mask*scale (encoder LNs)
// mode 1: dropout mask applies to the LN *output* (embeddings: y = dropout(LN(x))) -> dy is masked on load
// DY_F32 / DX_F32: the gradient flowing along the residual stream (dy in, dx out) is fp32 in the training engine so
// that 12 layers of residual additions do not each round it to bf16; dx_drop (what the tensor cores read) is bf16.
template <int VPL, bool DY_F32, bool DX_F32>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(
    const void* __restrict__ dy_, const void* __restrict__ dy_add_,
    const __nv_bfloat16* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ rstd,
    const __nv_bfloat16* __restrict__ gamma, int rows, float dropout_p, const unsigned long long* rng,
    unsigned rng_site, int mode, void* __restrict__ dx_, __nv_bfloat16* __restrict__ dx_drop,
    float* __restrict__ partials /* [gridDim.x][3][H] */) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  constexpr int H = VPL * 256;
  constexpr int WARPS = 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const DropCtx drop = make_drop_ctx(rng, rng_site, dropout_p);

  float g[VPL * 8];
  load_row<VPL>(gamma, lane, g);
  float acc_g[VPL * 8], acc_b[VPL * 8], acc_d[VPL * 8];
#pragma unroll
  for (int i = 0; i < VPL * 8; ++i) acc_g[i] = acc_b[i] = acc_d[i] = 0.f;

  for (int row = blockIdx.x * WARPS + warp; row < rows; row += gridDim.x * WARPS) {
    float dyv[VPL * 8], xv[VPL * 8];
    if (DY_F32) load_row_f32<VPL>(reinterpret_cast<const float*>(dy_) + (size_t)row * H, lane, dyv);
    else load_row<VPL>(reinterpret_cast<const __nv_bfloat16*>(dy_) + (size_t)row * H, lane, dyv);
    if (dy_add_ != nullptr) {
      float t[VPL * 8];
      if (DY_F32) load_row_f32<VPL>(reinterpret_cast<const float*>(dy_add_) + (size_t)row * H, lane, t);
      else load_row<VPL>(reinterpret_cast<const __nv_bfloat16*>(dy_add_) + (size_t)row * H, lane, t);
#pragma unroll
      for (int i = 0; i < VPL * 8; ++i) dyv[i] += t[i];
    }
    if (mode == 1 && drop.thresh != 0) {
#pragma unroll
      for (int vv = 0; vv < VPL; ++vv) {
        const uint32_t keep = dropout_keep8(drop, (unsigned long long)row * H + (vv * 32 + lane) * 8);
#pragma unroll
        for (int i = 0; i < 8; ++i) dyv[vv * 8 + i] = ((keep >> i) & 1u) ? dyv[vv * 8 + i] * drop.scale : 0.f;
      }
    }
    load_row<VPL>(x + (size_t)row * H, lane, xv);
    const float mu = mean[row], rs = rstd[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPL * 8; ++i) {
      xv[i] = (xv[i] - mu) * rs;               // xhat
      const float dxh = dyv[i] * g[i];
      s1 += dxh;
      s2 += dxh * xv[i];
      acc_g[i] += dyv[i] * xv[i];
      acc_b[i] += dyv[i];
    }
    s1 = warp_sum(s1) * (1.0f / H);
    s2 = warp_sum(s2) * (1.0f / H);
    float dxv[VPL * 8];
#pragma unroll
    for (int i = 0; i < VPL * 8; ++i) dxv[i] = rs * (dyv[i] * g[i] - s1 - xv[i] * s2);
    if (DX_F32) store_row_f32<VPL>(reinterpret_cast<float*>(dx_) + (size_t)row * H, lane, dxv);
    else store_row<VPL>(reinterpret_cast<__nv_bfloat16*>(dx_) + (size_t)row * H, lane, dxv);
    if (mode == 0) {
      if (dx_drop != nullptr) {
#pragma unroll
        for (int vv = 0; vv < VPL; ++vv) {
          const uint32_t keep = dropout_keep8(drop, (unsigned long long)row * H + (vv * 32 + lane) * 8);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            // the GEMMs consume the bf16-rounded value; sum exactly what they see
            const float t = ((keep >> i) & 1u) ? dxv[vv * 8 + i] * drop.scale : 0.f;
            dxv[vv * 8 + i] = bf16_round(t);
          }
        }
        store_row<VPL>(dx_drop + (size_t)row * H, lane, dxv);
      } else {
#pragma unroll
        for (int i = 0; i < VPL * 8; ++i) dxv[i] = bf16_round(dxv[i]);
      }
#pragma unroll
      for (int i = 0; i < VPL * 8; ++i) acc_d[i] += dxv[i];
    }
  }

  // block reduction of the three column-sum sets (warps -> smem -> one partial row per block)
  __shared__ float red[WARPS][H];
  float* out = partials + (size_t)blockIdx.x * 3 * H;
#define B2_REDUCE_SET(ARR, WHICH)                                                          \
  {                                                                                        \
    _Pragma("unroll") for (int vv = 0; vv < VPL; ++vv)                                     \
        _Pragma("unroll") for (int i = 0; i < 8; ++i) red[warp][(vv * 32 + lane) * 8 + i] = ARR[vv * 8 + i]; \
    __syncthreads();                                                                       \
    for (int c = threadIdx.x; c < H; c += blockDim.x) {                                    \
      float s = 0.f;                                                                       \
      _Pragma("unroll") for (int w = 0; w < WARPS; ++w) s += red[w][c];                    \
      out[(WHICH)*H + c] = s;                                                              \
    }                                                                                      \
    __syncthreads();                                                                       \
  }
  B2_REDUCE_SET(acc_g, 0)
  B2_REDUCE_SET(acc_b, 1)
  B2_REDUCE_SET(acc_d, 2)
#undef B2_REDUCE_SET
}

// The training engine's LayerNorm backward (fp32 gradient stream in and out, mode 0, dropout mask on the input
// branch).  ncu on the one-warp-per-row kernel above: ~1000 instructions per row per warp, 191 registers (72 of them
// column-sum accumulators) => 8 warps per SM, each at IPC ~0.14: latency-bound on its own instruction stream, HBM at
// a third of peak.  Here a row is shared by a PAIR of warps (each owns H/2 columns: 36 accumulators, ~110 registers),
// so 16 warps fit per SM and every warp's stream is half as long; the two row sums cross the pair through shared
// memory and a 64-thread named barrier.  Lane l of half h owns the 4-element vectors ((h*NV + j)*32 + l), j < NV.
constexpr int kLnDepth = 3;   // ring stages per warp (rows in flight: kLnDepth - 1 ahead of the one being reduced)
template <int NV>
__global__ void __launch_bounds__(512) layernorm_bwd_pair_kernel(
    const float* __restrict__ dy, const __nv_bfloat16* __restrict__ x, const float* __restrict__ mean,
    const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ gamma, int rows, float dropout_p,
    const unsigned long long* rng, unsigned rng_site, float* __restrict__ dx, __nv_bfloat16* __restrict__ dx_drop,
    float* __restrict__ partials /* [gridDim.x][3][H] */, float* __restrict__ accum /* or: fp32 [3][H], += */) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  constexpr int H = NV * 256;
  constexpr int SLOTS = 8;                     // rows in flight per block
  constexpr int E = NV * 4;                    // elements per lane
  __shared__ float red[SLOTS][H];              // end-of-kernel column-sum reduction
  __shared__ float xchg[2][SLOTS][2][2];       // [row parity][slot][half][s1, s2]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slot = warp >> 1, half = warp & 1;
  const DropCtx drop = make_drop_ctx(rng, rng_site, dropout_p);

  float g[E];
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const uint2 t = __ldg(reinterpret_cast<const uint2*>(gamma + ((half * NV + j) * 32 + lane) * 4));
    g[4 * j + 0] = bf16_lo(t.x); g[4 * j + 1] = bf16_hi(t.x); g[4 * j + 2] = bf16_lo(t.y); g[4 * j + 3] = bf16_hi(t.y);
  }
  float acc_g[E], acc_b[E], acc_d[E];
#pragma unroll
  for (int i = 0; i < E; ++i) acc_g[i] = acc_b[i] = acc_d[i] = 0.f;

  // Row operands are prefetched kLnDepth rows ahead with per-lane cp.async into a private shared-memory ring (each
  // lane later reads back exactly the bytes it copied: no barrier, no registers held while the loads are in flight).
  extern __shared__ __align__(16) uint8_t ln_ring[];
  constexpr int kStageBytes = NV * (32 * 16 + 32 * 8);
  uint8_t* ring = ln_ring + (size_t)warp * kLnDepth * kStageBytes;
  const int row_first = blockIdx.x * SLOTS + slot, row_step = gridDim.x * SLOTS;
  auto issue = [&](int k) {
    const int row = row_first + k * row_step;
    if (row < rows) {
      uint8_t* st = ring + (size_t)(k % kLnDepth) * kStageBytes;
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const size_t e0 = (size_t)row * H + ((half * NV + j) * 32 + lane) * 4;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(st + j * 768 + lane * 16)), "l"(dy + e0)
                     : "memory");
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(st + j * 768 + 512 + lane * 8)), "l"(x + e0)
                     : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");   // always: keeps the group count uniform
  };
#pragma unroll
  for (int k = 0; k < kLnDepth - 1; ++k) issue(k);

  int it = 0;
  for (int row = row_first; row < rows; row += row_step, ++it) {
    issue(it + kLnDepth - 1);
    const float mu = mean[row], rs = rstd[row];
    asm volatile("cp.async.wait_group %0;" ::"n"(kLnDepth - 1) : "memory");
    float dyv[E], xv[E];
    {
      const uint8_t* st = ring + (size_t)(it % kLnDepth) * kStageBytes;
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const float4 a = *reinterpret_cast<const float4*>(st + j * 768 + lane * 16);
        const uint2 t = *reinterpret_cast<const uint2*>(st + j * 768 + 512 + lane * 8);
        dyv[4 * j + 0] = a.x; dyv[4 * j + 1] = a.y; dyv[4 * j + 2] = a.z; dyv[4 * j + 3] = a.w;
        xv[4 * j + 0] = bf16_lo(t.x); xv[4 * j + 1] = bf16_hi(t.x); xv[4 * j + 2] = bf16_lo(t.y); xv[4 * j + 3] = bf16_hi(t.y);
      }
    }
    float s1 = 0.f, s2 = 0.f;
    const float nmr = -mu * rs;
#pragma unroll
    for (int i = 0; i < E; ++i) {
      xv[i] = fmaf(xv[i], rs, nmr);            // xhat
      const float dxh = dyv[i] * g[i];
      s1 += dxh;
      s2 = fmaf(dxh, xv[i], s2);
      acc_g[i] = fmaf(dyv[i], xv[i], acc_g[i]);
      acc_b[i] += dyv[i];
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    // combine the two halves of the row
    float* mine = xchg[it & 1][slot][half];
    if (lane == 0) { mine[0] = s1; mine[1] = s2; }
    asm volatile("bar.sync %0, 64;" ::"r"(slot + 1) : "memory");
    const float* other = xchg[it & 1][slot][half ^ 1];
    // fixed summation order (half 0 + half 1) so both warps of the pair compute identical row sums
    const float t1 = half ? other[0] + s1 : s1 + other[0];
    const float t2 = half ? other[1] + s2 : s2 + other[1];
    s1 = t1 * (1.0f / H);
    s2 = t2 * (1.0f / H);
    float dxv[E];
#pragma unroll
    for (int i = 0; i < E; ++i) dxv[i] = rs * (fmaf(dyv[i], g[i], -s1) - xv[i] * s2);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const size_t e0 = (size_t)row * H + ((half * NV + j) * 32 + lane) * 4;
      *reinterpret_cast<float4*>(dx + e0) = make_float4(dxv[4 * j], dxv[4 * j + 1], dxv[4 * j + 2], dxv[4 * j + 3]);
    }
    // dropout mask of the branch input: one Philox call covers 8 consecutive elements = a PAIR of lanes.  For two
    // vectors j, j+1 the even lane draws for j, the odd lane for j+1 and they swap (a lone last vector is drawn twice).
#pragma unroll
    for (int j = 0; j < NV; j += 2) {
      const bool odd = lane & 1;
      const bool paired = j + 1 < NV;
      const int jm = (paired && odd) ? j + 1 : j;
      const unsigned long long idx = (unsigned long long)row * H + (size_t)(((half * NV + jm) * 32 + (lane & ~1)) * 4);
      const uint32_t mine8 = dropout_keep8(drop, idx);
      uint32_t k0, k1 = 0;
      if (paired) {
        const uint32_t other8 = __shfl_xor_sync(0xffffffffu, mine8, 1);
        k0 = odd ? other8 : mine8;
        k1 = odd ? mine8 : other8;
      } else {
        k0 = mine8;
      }
      const int sh = odd ? 4 : 0;
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        if (jj == 1 && !paired) break;
        const uint32_t keep = (jj == 0 ? k0 : k1) >> sh;
        const int b = 4 * (j + jj);
#pragma unroll
        for (int i = 0; i < 4; ++i) dxv[b + i] = ((keep >> i) & 1u) ? dxv[b + i] * drop.scale : 0.f;
        // the GEMMs consume the bf16-rounded value: round once while packing, sum exactly what they will read
        uint2 o;
        o.x = pack_bf16_round(dxv[b + 0], dxv[b + 1]);
        o.y = pack_bf16_round(dxv[b + 2], dxv[b + 3]);
        *reinterpret_cast<uint2*>(dx_drop + (size_t)row * H + ((half * NV + j + jj) * 32 + lane) * 4) = o;
      }
    }
#pragma unroll
    for (int i = 0; i < E; ++i) acc_d[i] += dxv[i];
  }

  // block reduction of the three column-sum sets (8 row slots -> one row per block), then either a partial row for
  // a finishing kernel, or -- accum -- straight into the caller's fp32 accumulators (one reduction per column and
  // block at L2; the caller converts them together with its other fused bias-gradient sums)
  float* out = accum != nullptr ? accum : partials + (size_t)blockIdx.x * 3 * H;
#define B2_REDUCE_SET(ARR, WHICH)                                                          \
  {                                                                                        \
    _Pragma("unroll") for (int j = 0; j < NV; ++j)                                         \
        _Pragma("unroll") for (int i = 0; i < 4; ++i)                                      \
            red[slot][((half * NV + j) * 32 + lane) * 4 + i] = ARR[4 * j + i];             \
    __syncthreads();                                                                       \
    for (int c = threadIdx.x; c < H; c += blockDim.x) {                                    \
      float s = 0.f;                                                                       \
      _Pragma("unroll") for (int w = 0; w < SLOTS; ++w) s += red[w][c];                    \
      if (accum != nullptr) atomicAdd(out + (WHICH)*H + c, s);                             \
      else out[(WHICH)*H + c] = s;                                                         \
    }                                                                                      \
    __syncthreads();                                                                       \
  }
  B2_REDUCE_SET(acc_g, 0)
  B2_REDUCE_SET(acc_b, 1)
  B2_REDUCE_SET(acc_d, 2)
#undef B2_REDUCE_SET
}

// partials [nparts][nsets][cols] fp32 -> up to three bf16 [cols] outputs.  Block = 32 columns x 8 part-lanes so the
// reduction over `nparts` is itself parallel (a serial per-column loop is latency-bound).
__global__ void __launch_bounds__(256) colsum_finish_kernel(const float* __restrict__ partials, int nparts, int nsets,
                                                           int cols, __nv_bfloat16* o0, __nv_bfloat16* o1,
                                                           __nv_bfloat16* o2) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  __shared__ float red[8][33];
  const int c = threadIdx.x & 31, pl = threadIdx.x >> 5;
  const int idx = blockIdx.x * 32 + c;
  const int total = nsets * cols;
  float s = 0.f;
  if (idx < total) {
    const size_t stride = (size_t)total;
    const float* base = partials + idx;
    int p = pl;
    for (; p + 24 < nparts; p += 32) {
      const float a0 = base[(size_t)p * stride], a1 = base[(size_t)(p + 8) * stride];
      const float a2 = base[(size_t)(p + 16) * stride], a3 = base[(size_t)(p + 24) * stride];
      s += (a0 + a1) + (a2 + a3);
    }
    for (; p < nparts; p += 8) s += base[(size_t)p * stride];
  }
  red[pl][c] = s;
  __syncthreads();
  if (pl == 0 && idx < total) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][c];
    const int set = idx / cols, col = idx % cols;
    __nv_bfloat16* o = set == 0 ? o0 : (set == 1 ? o1 : o2);
    if (o != nullptr) o[col] = __float2bfloat16_rn(t);
  }
}

// column sums of x[rows, cols] (bf16), optional row filter; block = 8 warps x (32 lanes x 8 columns)
__global__ void __launch_bounds__(256) colsum_partial_kernel(const __nv_bfloat16* __restrict__ x, int rows, int cols,
                                                            long long ldx, const int* __restrict__ filter,
                                                            int filter_value, float* __restrict__ partials) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = blockIdx.x * 256 + lane * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (col < cols) {
    for (int r = blockIdx.y * 8 + warp; r < rows; r += gridDim.y * 8) {
      if (filter != nullptr && filter[r] != filter_value) continue;
      const uint4 v = ldg16(x + (size_t)r * ldx + col);
      acc[0] += bf16_lo(v.x); acc[1] += bf16_hi(v.x); acc[2] += bf16_lo(v.y); acc[3] += bf16_hi(v.y);
      acc[4] += bf16_lo(v.z); acc[5] += bf16_hi(v.z); acc[6] += bf16_lo(v.w); acc[7] += bf16_hi(v.w);
    }
  }
  __shared__ float red[8][256];
#pragma unroll
  for (int i = 0; i < 8; ++i) red[warp][lane * 8 + i] = acc[i];
  __syncthreads();
  const int c = threadIdx.x;
  if (blockIdx.x * 256 + c < cols) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][c];
    partials[(size_t)blockIdx.y * cols + blockIdx.x * 256 + c] = s;
  }
}

int32_t launch_colsum(const void* x, int64_t rows, int64_t cols, int64_t ldx, const int* filter, int filter_value,
                      void* out, float* scratch, int64_t scratch_bytes, cudaStream_t stream) {
  B2_REQUIRE(cols % 8 == 0 && ldx % 8 == 0, "colsum: cols/ldx must be multiples of 8");
  int nparts = (int)(scratch_bytes / (cols * 4));
  if (nparts > 32) nparts = 32;
  B2_REQUIRE(nparts >= 1, "colsum: scratch too small (%lld bytes for %lld columns)", (long long)scratch_bytes,
             (long long)cols);
  dim3 grid((unsigned)((cols + 255) / 256), (unsigned)nparts);
  B2_LAUNCH(colsum_partial_kernel, grid, 256, 0, stream, (const __nv_bfloat16*)x, (int)rows, (int)cols, ldx, filter,
                                                  filter_value, scratch);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  B2_LAUNCH(colsum_finish_kernel, (unsigned)((cols + 31) / 32), 256, 0, stream, scratch, nparts, 1, (int)cols,
                                                                           (__nv_bfloat16*)out, nullptr, nullptr);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

static int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

int32_t launch_layernorm_bwd(const void* dy, const void* dy_add, const void* x, const float* mean, const float* rstd,
                             const void* gamma, int64_t rows, int64_t hidden, float dropout_p, const void* rng,
                             uint32_t site, int mode, int dy_f32, int dx_f32, void* dx, void* dx_drop, void* d_gamma,
                             void* d_beta, void* d_bias, float* scratch, int64_t scratch_bytes, cudaStream_t stream,
                             int32_t* deferred_nparts, float* accum) {
  B2_REQUIRE(hidden % 256 == 0 && hidden >= 256 && hidden <= 1024, "layernorm: hidden=%lld unsupported",
             (long long)hidden);
  int nblocks = accum != nullptr ? 1 << 20 : (int)(scratch_bytes / (3 * hidden * 4));
  const int want = 296;
  if (nblocks > want) nblocks = want;
  const int max_useful = (int)((rows + 7) / 8);
  if (nblocks > max_useful) nblocks = max_useful;
  B2_REQUIRE(nblocks >= 1, "layernorm_bwd: scratch too small");
#define B2_LN_ARGS                                                                                           \
  dy, dy_add, (const __nv_bfloat16*)x, mean, rstd, (const __nv_bfloat16*)gamma, (int)rows, dropout_p,        \
      (const unsigned long long*)rng, site, mode, dx, (__nv_bfloat16*)dx_drop, scratch
#define B2_LN_BWD(VPL_)                                                                                      \
  case VPL_:                                                                                                 \
    if (dy_f32 && dx_f32) B2_LAUNCH((layernorm_bwd_kernel<VPL_, true, true>), nblocks, 256, 0, stream, B2_LN_ARGS);   \
    else if (dy_f32) B2_LAUNCH((layernorm_bwd_kernel<VPL_, true, false>), nblocks, 256, 0, stream, B2_LN_ARGS);       \
    else B2_LAUNCH((layernorm_bwd_kernel<VPL_, false, false>), nblocks, 256, 0, stream, B2_LN_ARGS);                  \
    break;
  B2_REQUIRE(dy_f32 || !dx_f32, "layernorm_bwd: fp32 dx with bf16 dy is not on the path");
  const bool paired = dy_f32 && dx_f32 && mode == 0 && dy_add == nullptr && dx_drop != nullptr;
  if (paired) {
    // one resident 512-thread block per SM: a single wave, rows strided over the whole grid
    if (nblocks > num_sms()) nblocks = num_sms();
#define B2_LN_BWD_PAIR(NV_)                                                                                     \
  case NV_: {                                                                                                   \
    constexpr int smem = 16 * kLnDepth * NV_ * 768;                                                             \
    static bool attr = false;                                                                                   \
    if (!attr) {                                                                                                \
      B2_CUDA(cudaFuncSetAttribute(layernorm_bwd_pair_kernel<NV_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                   smem));                                                                      \
      attr = true;                                                                                              \
    }                                                                                                           \
    B2_LAUNCH((layernorm_bwd_pair_kernel<NV_>), nblocks, 512, smem, stream, (const float*)dy,                   \
              (const __nv_bfloat16*)x, mean, rstd, (const __nv_bfloat16*)gamma, (int)rows, dropout_p,           \
              (const unsigned long long*)rng, site, (float*)dx, (__nv_bfloat16*)dx_drop, scratch, accum);       \
  } break;
    switch ((int)(hidden / 256)) {
      B2_LN_BWD_PAIR(1) B2_LN_BWD_PAIR(2) B2_LN_BWD_PAIR(3) B2_LN_BWD_PAIR(4)
    }
#undef B2_LN_BWD_PAIR
  } else {
    B2_REQUIRE(accum == nullptr, "layernorm_bwd: accumulate mode needs the fp32-stream pair kernel");
    switch ((int)(hidden / 256)) {
      B2_LN_BWD(1) B2_LN_BWD(2) B2_LN_BWD(3) B2_LN_BWD(4)
    }
  }
#undef B2_LN_BWD
#undef B2_LN_ARGS
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  if (accum != nullptr) return 0;     // column sums already added into the caller's accumulators
  if (deferred_nparts != nullptr) {   // the caller runs b2_colsum_finish itself (e.g. on another stream)
    *deferred_nparts = nblocks;
    return 0;
  }
  B2_LAUNCH(colsum_finish_kernel, (unsigned)((3 * hidden + 31) / 32), 256, 0, stream, 
      scratch, nblocks, 3, (int)hidden, (__nv_bfloat16*)d_gamma, (__nv_bfloat16*)d_beta, (__nv_bfloat16*)d_bias);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace b2

using namespace b2;

extern "C" int32_t b2_layernorm_fwd(const void* x, const void* gamma, const void* beta, int64_t rows, int64_t hidden,
                                    float eps, void* y, float* mean, float* rstd, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  B2_REQUIRE(x && gamma && beta && y && mean && rstd, "layernorm_fwd: null pointer");
  B2_REQUIRE(rows > 0, "layernorm_fwd: rows=%lld", (long long)rows);
  B2_REQUIRE(hidden % 256 == 0 && hidden >= 256 && hidden <= 1024, "layernorm_fwd: hidden=%lld unsupported",
             (long long)hidden);
  const unsigned grid = (unsigned)((rows + 3) / 4);
#define B2_LN_FWD(VPL_)                                                                                       \
  case VPL_:                                                                                                  \
    B2_LAUNCH((layernorm_fwd_kernel<VPL_>), grid, 128, 0, stream, (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma, \
                                                         (const __nv_bfloat16*)beta, (int)rows, eps,           \
                                                         (__nv_bfloat16*)y, mean, rstd);                       \
    break;
  switch ((int)(hidden / 256)) {
    B2_LN_FWD(1) B2_LN_FWD(2) B2_LN_FWD(3) B2_LN_FWD(4)
  }
#undef B2_LN_FWD
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_layernorm_bwd(const void* dy, const void* dy_add, const void* x, const float* mean,
                                    const float* rstd, const void* gamma, int64_t rows, int64_t hidden,
                                    float dropout_p, const void* rng_state, uint32_t rng_site, int32_t grad_fp32,
                                    void* dx, void* dx_drop, void* d_gamma, void* d_beta, void* d_bias,
                                    float* scratch_partials, int64_t scratch_partials_bytes, int32_t* deferred_nparts,
                                    void* stream_) {
  B2_REQUIRE(dy && x && mean && rstd && gamma && dx && d_gamma && d_beta && scratch_partials,
             "layernorm_bwd: null pointer");
  B2_REQUIRE(rows > 0, "layernorm_bwd: rows=%lld", (long long)rows);
  B2_REQUIRE(!(dropout_p > 0.f) || (rng_state && dx_drop), "layernorm_bwd: dropout needs rng_state and dx_drop");
  B2_REQUIRE(!grad_fp32 || dx_drop, "layernorm_bwd: the fp32 gradient stream needs dx_drop (the bf16 GEMM operand)");
  return launch_layernorm_bwd(dy, dy_add, x, mean, rstd, gamma, rows, hidden, dropout_p, rng_state, rng_site, 0,
                              grad_fp32 ? 1 : 0, grad_fp32 ? 1 : 0, dx,
                              (dropout_p > 0.f || grad_fp32) ? dx_drop : nullptr, d_gamma, d_beta, d_bias,
                              scratch_partials, scratch_partials_bytes, (cudaStream_t)stream_, deferred_nparts);
}

extern "C" int32_t b2_colsum_finish(const float* partials, int32_t nparts, int32_t nsets, int64_t cols, void* out0,
                                    void* out1, void* out2, void* stream_) {
  B2_REQUIRE(partials && nparts > 0 && nsets >= 1 && nsets <= 3 && cols > 0, "colsum_finish: bad args");
  B2_LAUNCH(colsum_finish_kernel, (unsigned)((nsets * cols + 31) / 32), 256, 0, stream_, partials, (int)nparts,
            (int)nsets, (int)cols, (__nv_bfloat16*)out0, (__nv_bfloat16*)out1, (__nv_bfloat16*)out2);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_colsum(const void* x, int64_t rows, int64_t cols, int64_t ldx, void* out,
                             float* scratch_partials, int64_t scratch_partials_bytes, void* stream_) {
  B2_REQUIRE(x && out && scratch_partials, "colsum: null pointer");
  B2_REQUIRE(rows > 0 && cols > 0, "colsum: empty input");
  return launch_colsum(x, rows, cols, ldx, nullptr, 0, out, scratch_partials, scratch_partials_bytes,
                       (cudaStream_t)stream_);
}

extern "C" int32_t b2_layernorm_bwd_accum(const float* dy, const void* x, const float* mean, const float* rstd,
                                          const void* gamma, int64_t rows, int64_t hidden, float dropout_p,
                                          const void* rng_state, uint32_t rng_site, float* dx, void* dx_drop,
                                          float* accum, void* stream_) {
  B2_REQUIRE(dy && x && mean && rstd && gamma && dx && dx_drop && accum, "layernorm_bwd_accum: null pointer");
  B2_REQUIRE(rows > 0, "layernorm_bwd_accum: rows=%lld", (long long)rows);
  B2_REQUIRE(!(dropout_p > 0.f) || rng_state, "layernorm_bwd_accum: dropout needs rng_state");
  return launch_layernorm_bwd(dy, nullptr, x, mean, rstd, gamma, rows, hidden, dropout_p, rng_state, rng_site, 0, 1, 1,
                              dx, dx_drop, nullptr, nullptr, nullptr, nullptr, 0, (cudaStream_t)stream_, nullptr,
                              accum);
}
