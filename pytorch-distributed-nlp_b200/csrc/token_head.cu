// Token-classification head (HF BertForTokenClassification, no pooler): classifier dropout + Linear on every token of
// the last hidden state, forward and backward.  x is the last layer's bf16 output [M, H] (M = batch x seq, or
// bins x bin_len when packed: the head is token-wise), W / b the bf16 classifier [C, H] / [C], logits fp32 [M, C].
// Dropout is the engine's Philox stream at element m * H + h; the backward regenerates it, nothing is stored.
// The parameter gradients are summed in a fixed order (fp32 partials per row block, added in ascending block order,
// one rounding to bf16), so the head's gradients are bitwise repeatable without atomics.
#include "common.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

constexpr int kTokMaxLabels = 64;     // tag sets are far smaller; the host rejects larger C
constexpr int kTokRowsPerWarp = 2;    // forward: rows sharing each loaded weight chunk
constexpr int kTokWgradLabels = 8;    // parameter gradient: labels per block (8 x 8 fp32 accumulators per thread)
constexpr int kTokMaxRowBlocks = 128; // parameter gradient: row blocks (partials) at most

// x[row, k .. k+8) with the dropout of element row * H + k applied (scale 1/(1-p) on kept elements), as fp32
__device__ __forceinline__ void load_drop8(const __nv_bfloat16* __restrict__ x, int H, long long row, int k,
                                           const DropCtx& drop, float v[8]) {
  const uint4 u = ldg16(x + (size_t)row * H + k);
  const uint32_t keep = dropout_keep8(drop, (unsigned long long)row * H + k);
  v[0] = bf16_lo(u.x); v[1] = bf16_hi(u.x); v[2] = bf16_lo(u.y); v[3] = bf16_hi(u.y);
  v[4] = bf16_lo(u.z); v[5] = bf16_hi(u.z); v[6] = bf16_lo(u.w); v[7] = bf16_hi(u.w);
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = ((keep >> i) & 1u) ? v[i] * drop.scale : 0.f;
}

// logits[m, c] = b[c] + sum_h drop(x[m, h]) W[c, h].  One warp per kTokRowsPerWarp rows; each lane keeps its NCH
// chunks of 8 elements of those rows in registers (the dropout is drawn once per element), and every weight chunk it
// loads serves all of them.  NCH = H / 256.
template <int NCH>
__global__ void __launch_bounds__(256) token_head_fwd_kernel(const __nv_bfloat16* __restrict__ x, int M, int H,
                                                            const __nv_bfloat16* __restrict__ W,
                                                            const __nv_bfloat16* __restrict__ bias, int C,
                                                            float dropout_p, const unsigned long long* rng,
                                                            unsigned site, float* __restrict__ logits) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const long long m0 = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * kTokRowsPerWarp;
  if (m0 >= M) return;
  const DropCtx drop = make_drop_ctx(rng, site, dropout_p);
  float xv[kTokRowsPerWarp][NCH][8];
#pragma unroll
  for (int r = 0; r < kTokRowsPerWarp; ++r) {
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      if (m0 + r < M) {
        load_drop8(x, H, m0 + r, j * 256 + lane * 8, drop, xv[r][j]);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) xv[r][j][i] = 0.f;
      }
    }
  }
  for (int c = 0; c < C; ++c) {
    float s[kTokRowsPerWarp];
#pragma unroll
    for (int r = 0; r < kTokRowsPerWarp; ++r) s[r] = 0.f;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      const uint4 w = ldg16(W + (size_t)c * H + j * 256 + lane * 8);
      const float wv[8] = {bf16_lo(w.x), bf16_hi(w.x), bf16_lo(w.y), bf16_hi(w.y),
                           bf16_lo(w.z), bf16_hi(w.z), bf16_lo(w.w), bf16_hi(w.w)};
#pragma unroll
      for (int r = 0; r < kTokRowsPerWarp; ++r)
#pragma unroll
        for (int i = 0; i < 8; ++i) s[r] = fmaf(xv[r][j][i], wv[i], s[r]);
    }
    const float bc = __bfloat162float(bias[c]);
#pragma unroll
    for (int r = 0; r < kTokRowsPerWarp; ++r) {
      const float t = warp_sum(s[r]);
      if (lane == 0 && m0 + r < M) logits[(size_t)(m0 + r) * C + c] = t + bc;
    }
  }
}

// d_hidden[m, h] = keep(m, h) / (1 - p) * sum_c dlogits[m, c] W[c, h], fp32, every row.  One warp per row, each lane
// NCH chunks of 8 columns; dlogits[m, :] is read once per warp (broadcast).
template <int NCH>
__global__ void __launch_bounds__(256) token_head_bwd_data_kernel(const float* __restrict__ dlogits, int M, int H,
                                                                 const __nv_bfloat16* __restrict__ W, int C,
                                                                 float dropout_p, const unsigned long long* rng,
                                                                 unsigned site, float* __restrict__ d_hidden) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const long long m = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (m >= M) return;
  const DropCtx drop = make_drop_ctx(rng, site, dropout_p);
  float acc[NCH][8];
#pragma unroll
  for (int j = 0; j < NCH; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
  for (int c = 0; c < C; ++c) {
    const float d = dlogits[(size_t)m * C + c];
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      const uint4 w = ldg16(W + (size_t)c * H + j * 256 + lane * 8);
      acc[j][0] = fmaf(d, bf16_lo(w.x), acc[j][0]); acc[j][1] = fmaf(d, bf16_hi(w.x), acc[j][1]);
      acc[j][2] = fmaf(d, bf16_lo(w.y), acc[j][2]); acc[j][3] = fmaf(d, bf16_hi(w.y), acc[j][3]);
      acc[j][4] = fmaf(d, bf16_lo(w.z), acc[j][4]); acc[j][5] = fmaf(d, bf16_hi(w.z), acc[j][5]);
      acc[j][6] = fmaf(d, bf16_lo(w.w), acc[j][6]); acc[j][7] = fmaf(d, bf16_hi(w.w), acc[j][7]);
    }
  }
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    const int k = j * 256 + lane * 8;
    const uint32_t keep = dropout_keep8(drop, (unsigned long long)m * H + k);
    float4 lo, hi;
    lo.x = ((keep >> 0) & 1u) ? acc[j][0] * drop.scale : 0.f;
    lo.y = ((keep >> 1) & 1u) ? acc[j][1] * drop.scale : 0.f;
    lo.z = ((keep >> 2) & 1u) ? acc[j][2] * drop.scale : 0.f;
    lo.w = ((keep >> 3) & 1u) ? acc[j][3] * drop.scale : 0.f;
    hi.x = ((keep >> 4) & 1u) ? acc[j][4] * drop.scale : 0.f;
    hi.y = ((keep >> 5) & 1u) ? acc[j][5] * drop.scale : 0.f;
    hi.z = ((keep >> 6) & 1u) ? acc[j][6] * drop.scale : 0.f;
    hi.w = ((keep >> 7) & 1u) ? acc[j][7] * drop.scale : 0.f;
    float4* o = reinterpret_cast<float4*>(d_hidden + (size_t)m * H + k);
    o[0] = lo;
    o[1] = hi;
  }
}

// Parameter-gradient partials of row block blockIdx.x (rows [blk * rows_per_block, ...) ), labels
// [blockIdx.y * 8, +8): part[blk][c][h] = sum_m dlogits[m, c] drop(x[m, h]) (m ascending), and part[blk][C][c] (the
// bias row, written by the block's thread 0) = sum_m dlogits[m, c].  Thread t owns columns [8t, 8t + 8): H / 8
// threads.  The block's dlogits are staged in shared memory.
__global__ void __launch_bounds__(128) token_head_wgrad_partial_kernel(
    const float* __restrict__ dlogits, const __nv_bfloat16* __restrict__ x, int M, int H, int C, int rows_per_block,
    float dropout_p, const unsigned long long* rng, unsigned site, float* __restrict__ part) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float sdl[];     // [rows_per_block][8]
  const int blk = blockIdx.x, c0 = blockIdx.y * kTokWgradLabels;
  const int nc = min(kTokWgradLabels, C - c0);
  const long long r0 = (long long)blk * rows_per_block;
  const int nr = (int)min((long long)rows_per_block, (long long)M - r0);
  for (int i = threadIdx.x; i < nr * kTokWgradLabels; i += blockDim.x) {
    const int r = i / kTokWgradLabels, c = i % kTokWgradLabels;
    sdl[i] = c < nc ? dlogits[(size_t)(r0 + r) * C + c0 + c] : 0.f;
  }
  __syncthreads();
  float* out = part + (size_t)blk * (C + 1) * H;
  if (threadIdx.x == 0) {
    for (int c = 0; c < nc; ++c) {
      float sb = 0.f;
      for (int r = 0; r < nr; ++r) sb += sdl[r * kTokWgradLabels + c];
      out[(size_t)C * H + c0 + c] = sb;
    }
  }
  const int k = threadIdx.x * 8;
  if (k >= H) return;
  const DropCtx drop = make_drop_ctx(rng, site, dropout_p);
  float acc[kTokWgradLabels][8];
#pragma unroll
  for (int c = 0; c < kTokWgradLabels; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
#pragma unroll 4
  for (int r = 0; r < nr; ++r) {
    float v[8];
    load_drop8(x, H, r0 + r, k, drop, v);
#pragma unroll
    for (int c = 0; c < kTokWgradLabels; ++c) {
      const float d = sdl[r * kTokWgradLabels + c];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[c][i] = fmaf(d, v[i], acc[c][i]);
    }
  }
#pragma unroll
  for (int c = 0; c < kTokWgradLabels; ++c) {
    if (c < nc) {
      float4* o = reinterpret_cast<float4*>(out + (size_t)(c0 + c) * H + k);
      o[0] = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
      o[1] = make_float4(acc[c][4], acc[c][5], acc[c][6], acc[c][7]);
    }
  }
}

// dW[c, h] / db[c] = bf16(sum over row blocks, ascending, of the partials): one thread per element of the [C + 1][H]
// partial plane (row C carries the bias in its first C columns)
__global__ void __launch_bounds__(256) token_head_wgrad_finish_kernel(const float* __restrict__ part, int nblk, int H,
                                                                     int C, __nv_bfloat16* __restrict__ dW,
                                                                     __nv_bfloat16* __restrict__ db) {
  pdl_wait();
  pdl_launch_dependents();
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long plane = (long long)(C + 1) * H;
  if (e >= (long long)C * H + C) return;
  float s = 0.f;
#pragma unroll 8
  for (int b = 0; b < nblk; ++b) s += part[(size_t)b * plane + e];
  if (e < (long long)C * H) dW[e] = __float2bfloat16_rn(s);
  else db[e - (long long)C * H] = __float2bfloat16_rn(s);
}

}  // namespace b2

using namespace b2;

// the row blocks of the parameter gradient: at most kTokMaxRowBlocks, at least 32 rows each
static void token_row_blocks(int64_t M, int64_t* rows_per_block, int64_t* nblk) {
  int64_t rpb = (M + kTokMaxRowBlocks - 1) / kTokMaxRowBlocks;
  if (rpb < 32) rpb = 32;
  *rows_per_block = rpb;
  *nblk = (M + rpb - 1) / rpb;
}

extern "C" int64_t b2_token_head_scratch_floats(int64_t tokens, int64_t hidden, int64_t num_labels) {
  int64_t rpb, nblk;
  token_row_blocks(tokens, &rpb, &nblk);
  return nblk * (num_labels + 1) * hidden;
}

#define B2_TOKEN_NCH_SWITCH(H, ...)                 \
  switch ((H) / 256) {                              \
    case 1: { constexpr int NCH = 1; __VA_ARGS__; } break; \
    case 2: { constexpr int NCH = 2; __VA_ARGS__; } break; \
    case 3: { constexpr int NCH = 3; __VA_ARGS__; } break; \
    default: { constexpr int NCH = 4; __VA_ARGS__; } break; \
  }

static int32_t token_head_check(const char* fn, int64_t tokens, int64_t hidden, int64_t num_labels, float dropout_p,
                                const void* rng_state) {
  B2_REQUIRE(tokens > 0, "%s: no tokens", fn);
  // the parameter gradient stages a row block's dlogits in shared memory: 1 024 rows x 8 labels x 4 B = 32 KB
  B2_REQUIRE(tokens <= (int64_t)kTokMaxRowBlocks * 1024, "%s: tokens=%lld is more than %d", fn, (long long)tokens,
             kTokMaxRowBlocks * 1024);
  B2_REQUIRE(hidden % 256 == 0 && hidden >= 256 && hidden <= 1024,
             "%s: hidden=%lld must be a multiple of 256 in [256, 1024]", fn, (long long)hidden);
  B2_REQUIRE(num_labels >= 1 && num_labels <= kTokMaxLabels, "%s: num_labels=%lld must be in [1, %d]", fn,
             (long long)num_labels, kTokMaxLabels);
  B2_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "%s: dropout_p=%g must be in [0, 1)", fn, (double)dropout_p);
  B2_REQUIRE(!(dropout_p > 0.f) || rng_state, "%s: dropout needs rng_state", fn);
  return 0;
}

extern "C" int32_t b2_token_head_fwd(const void* hidden_states, int64_t tokens, int64_t hidden, const void* cls_w,
                                     const void* cls_b, int64_t num_labels, float dropout_p, const void* rng_state,
                                     uint32_t rng_site, float* logits, void* stream_) {
  B2_REQUIRE(hidden_states && cls_w && cls_b && logits, "token_head_fwd: null pointer");
  if (int32_t e = token_head_check("token_head_fwd", tokens, hidden, num_labels, dropout_p, rng_state)) return e;
  const unsigned grid = (unsigned)((tokens + 8 * kTokRowsPerWarp - 1) / (8 * kTokRowsPerWarp));
  B2_TOKEN_NCH_SWITCH(hidden,
      B2_LAUNCH(token_head_fwd_kernel<NCH>, grid, 256, 0, (cudaStream_t)stream_,
                (const __nv_bfloat16*)hidden_states, (int)tokens, (int)hidden, (const __nv_bfloat16*)cls_w,
                (const __nv_bfloat16*)cls_b, (int)num_labels, dropout_p, (const unsigned long long*)rng_state,
                rng_site, logits));
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_token_head_bwd_split(const float* dlogits, const void* hidden_states, int64_t tokens,
                                           int64_t hidden, const void* cls_w, int64_t num_labels, float dropout_p,
                                           const void* rng_state, uint32_t rng_site, void* d_cls_w, void* d_cls_b,
                                           float* d_hidden, float* scratch, int64_t scratch_floats, void* stream_,
                                           void* weight_stream_) {
  B2_REQUIRE(dlogits && hidden_states && cls_w && d_cls_w && d_cls_b && d_hidden && scratch,
             "token_head_bwd_split: null pointer");
  if (int32_t e = token_head_check("token_head_bwd_split", tokens, hidden, num_labels, dropout_p, rng_state)) return e;
  B2_REQUIRE(scratch_floats >= b2_token_head_scratch_floats(tokens, hidden, num_labels),
             "token_head_bwd_split: scratch of %lld floats, need %lld", (long long)scratch_floats,
             (long long)b2_token_head_scratch_floats(tokens, hidden, num_labels));
  cudaStream_t stream = (cudaStream_t)stream_;
  const auto* rng = (const unsigned long long*)rng_state;
  B2_TOKEN_NCH_SWITCH(hidden,
      B2_LAUNCH(token_head_bwd_data_kernel<NCH>, (unsigned)((tokens + 7) / 8), 256, 0, stream, dlogits, (int)tokens,
                (int)hidden, (const __nv_bfloat16*)cls_w, (int)num_labels, dropout_p, rng, rng_site, d_hidden));
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  // the parameter part is off the critical path: on the caller's weight-gradient stream, ordered behind what the
  // main stream has issued so far (dlogits and x are final there)
  cudaStream_t wstream = stream;
  if (weight_stream_ != nullptr && (cudaStream_t)weight_stream_ != stream) {
    static thread_local cudaEvent_t ev = nullptr;
    if (ev == nullptr) B2_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    B2_CUDA(cudaEventRecord(ev, stream));
    wstream = (cudaStream_t)weight_stream_;
    B2_CUDA(cudaStreamWaitEvent(wstream, ev, 0));
  }
  int64_t rpb, nblk;
  token_row_blocks(tokens, &rpb, &nblk);
  const dim3 pgrid((unsigned)nblk, (unsigned)((num_labels + kTokWgradLabels - 1) / kTokWgradLabels));
  B2_LAUNCH(token_head_wgrad_partial_kernel, pgrid, 128, (size_t)rpb * kTokWgradLabels * sizeof(float), wstream,
            dlogits, (const __nv_bfloat16*)hidden_states, (int)tokens, (int)hidden, (int)num_labels, (int)rpb,
            dropout_p, rng, rng_site, scratch);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  const int64_t n = num_labels * hidden + num_labels;
  B2_LAUNCH(token_head_wgrad_finish_kernel, (unsigned)((n + 255) / 256), 256, 0, wstream, (const float*)scratch,
            (int)nblk, (int)hidden, (int)num_labels, (__nv_bfloat16*)d_cls_w, (__nv_bfloat16*)d_cls_b);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}
