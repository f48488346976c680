// Masked-language-model head (HF BertForMaskedLM's cls.predictions) around the wgmma GEMMs: what the GEMM cannot do.
// The head runs on the labelled rows only.  b2_mlm_compact lists them (in token order) into a capacity the host picks;
// the unused capacity rows gather zeros, carry label -1 and get a zero gradient row, so they contribute exactly 0.
// The projection onto the vocabulary is one GEMM with N = vocab_pad (vocab rounded up to 64: the extra rows of the
// word-embedding table and the extra bias entries are zero), added onto logits rows pre-filled with the decoder bias
// (b2_mlm_bias_fill), so the logits stay fp32.  b2_mlm_ce is the vocabulary cross-entropy: one block per row, an
// online max / log-sum-exp over the first vocab columns, the row's loss term, the argmax and the bf16 d_logits.  Its
// mean over the labelled rows is summed in a fixed order, so the loss is bitwise repeatable.
#include "common.cuh"
#include "../../include/b2_ddp_bert.h"

#include <climits>

namespace b2 {

constexpr int kCompactThreads = 1024;
constexpr int kCeThreads = 256;

// One block: the rows whose label is not ignore_index, in token order, and each row's slot (-1: none).  A label outside
// [0, vocab) that is not ignore_index traps, as the loss kernels do.
__global__ void __launch_bounds__(kCompactThreads) mlm_compact_kernel(const long long* __restrict__ labels, int M,
                                                                      long long ignore, long long V, int cap,
                                                                      int* __restrict__ rows, int* __restrict__ slot,
                                                                      int* __restrict__ slot_labels, int* count) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ int warp_tot[kCompactThreads / 32];
  __shared__ int base;
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  if (t == 0) base = 0;
  __syncthreads();
  for (int c0 = 0; c0 < M; c0 += kCompactThreads) {
    const int m = c0 + t;
    long long y = ignore;
    if (m < M) y = labels[m];
    const bool lab = m < M && y != ignore;
    if (lab && (y < 0 || y >= V)) {
      printf("b2 masked-lm: label %lld of token %d is outside [0, %lld) and is not the ignore_index\n", y, m, V);
      __trap();
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, lab);
    if (lane == 0) warp_tot[wid] = __popc(ballot);
    __syncthreads();
    int before = base;
    for (int w = 0; w < wid; ++w) before += warp_tot[w];
    const int s = before + __popc(ballot & ((1u << lane) - 1u));
    if (m < M) {
      slot[m] = lab ? s : -1;
      if (lab) {
        if (s >= cap) {
          printf("b2 masked-lm: more than %d labelled tokens for a capacity of %d rows\n", s, cap);
          __trap();
        }
        rows[s] = m;
        slot_labels[s] = (int)y;
      }
    }
    __syncthreads();
    if (t == kCompactThreads - 1) base = s + (lab ? 1 : 0);
    __syncthreads();
  }
  const int n = base;
  for (int i = n + t; i < cap; i += kCompactThreads) {
    rows[i] = 0;
    slot_labels[i] = -1;
  }
  if (t == 0) *count = n;
}

// out[i] = x[rows[i]] for i < count, zero for the rest of the capacity.  One block per row, 8 bf16 per thread.
__global__ void mlm_gather_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ rows, const int* count,
                                  int H, __nv_bfloat16* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  const long long i = blockIdx.x;
  const int k = threadIdx.x * 8;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (i < *count) v = ldg16(x + (size_t)rows[i] * H + k);
  *reinterpret_cast<uint4*>(out + (size_t)i * H + k) = v;
}

// dx[m] = src[slot[m]] for a labelled token, zero for every other: each row of dx is written.  4 fp32 per thread.
__global__ void mlm_scatter_kernel(const float* __restrict__ src, const int* __restrict__ slot, int H,
                                   float* __restrict__ dx) {
  pdl_wait();
  pdl_launch_dependents();
  const long long m = blockIdx.x;
  const int k = threadIdx.x * 4;
  const int s = slot[m];
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (s >= 0) v = *reinterpret_cast<const float4*>(src + (size_t)s * H + k);
  *reinterpret_cast<float4*>(dx + (size_t)m * H + k) = v;
}

// du = bf16(dg * gelu'(u)): the GELU' the LayerNorm backward of the transform cannot apply itself (gelu_erf_grad, the
// derivative the GEMM's EPI_GELU_BWD epilogue uses)
__global__ void mlm_gelu_bwd_kernel(const float* __restrict__ dg, const __nv_bfloat16* __restrict__ u, long long n8,
                                    __nv_bfloat16* __restrict__ du) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 uu = ldg16(u + i * 8);
    const float4 a = *reinterpret_cast<const float4*>(dg + i * 8);
    const float4 b = *reinterpret_cast<const float4*>(dg + i * 8 + 4);
    uint4 o;
    o.x = pack_bf16(a.x * gelu_erf_grad(bf16_lo(uu.x)), a.y * gelu_erf_grad(bf16_hi(uu.x)));
    o.y = pack_bf16(a.z * gelu_erf_grad(bf16_lo(uu.y)), a.w * gelu_erf_grad(bf16_hi(uu.y)));
    o.z = pack_bf16(b.x * gelu_erf_grad(bf16_lo(uu.z)), b.y * gelu_erf_grad(bf16_hi(uu.z)));
    o.w = pack_bf16(b.z * gelu_erf_grad(bf16_lo(uu.w)), b.w * gelu_erf_grad(bf16_hi(uu.w)));
    *reinterpret_cast<uint4*>(du + i * 8) = o;
  }
}

// logits[r, c] = bias[c] for every row, c < vocab_pad (the GEMM then adds the product, EPI_ACCUM_F32)
__global__ void mlm_bias_fill_kernel(const __nv_bfloat16* __restrict__ bias, long long n4, int Vp4,
                                     float* __restrict__ logits) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Vp4) * 4;
    const uint2 b = *reinterpret_cast<const uint2*>(bias + c);
    *reinterpret_cast<float4*>(logits + i * 4) = make_float4(bf16_lo(b.x), bf16_hi(b.x), bf16_lo(b.y), bf16_hi(b.y));
  }
}

// online (max, sum of exp) pair: merge (m2, s2) into (m, s); a pair with m = -inf is empty
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) { m = m2; s = s2; return; }
  if (m2 > m) { s = s * expf(m - m2) + s2; m = m2; }
  else        { s = s + s2 * expf(m2 - m); }
}
// argmax pair: the larger value, the smaller index on ties (torch.argmax's first occurrence)
__device__ __forceinline__ void arg_merge(float& v, int& i, float v2, int i2) {
  if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}

// One block per row.  labels[r] = -1: no loss term (ignored, or a padding row of the capacity).  Rows at or past
// *n_rows are capacity padding: zero gradient row, no loss, pred -1.
//   row_loss[r] = lse - x[y],  pred[r] = argmax_c<V x[c]
//   d_logits[r, c] = bf16(extra[r, c] + (softmax - onehot) * d_loss / n_labelled) for c < V, 0 for V <= c < V_pad
__global__ void __launch_bounds__(kCeThreads) mlm_ce_kernel(const float* __restrict__ logits, int V, int Vp,
                                                            const int* __restrict__ labels, const int* n_rows,
                                                            const int* n_lab, const float* d_loss,
                                                            const float* __restrict__ extra, long long ld_extra,
                                                            float* __restrict__ row_loss, int* __restrict__ pred,
                                                            __nv_bfloat16* __restrict__ dlog) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float sm_m[kCeThreads / 32], sm_s[kCeThreads / 32], sm_v[kCeThreads / 32];
  __shared__ int sm_i[kCeThreads / 32];
  const long long r = blockIdx.x;
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const bool live = n_rows == nullptr || r < *n_rows;
  const int y = (live && labels != nullptr) ? labels[r] : -1;
  if (y < -1 || y >= V) {
    if (t == 0) printf("b2 masked-lm cross-entropy: label %d of row %lld is outside [0, %d)\n", y, r, V);
    __trap();
  }
  const float* row = logits + (size_t)r * Vp;
  const float* erow = (extra != nullptr && live) ? extra + (size_t)r * ld_extra : nullptr;
  __nv_bfloat16* drow = dlog != nullptr ? dlog + (size_t)r * Vp : nullptr;
  if (y < 0) {
    if (drow != nullptr)
      for (int c = t * 4; c < Vp; c += kCeThreads * 4) {
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = (erow != nullptr && c + j < V) ? erow[c + j] : 0.f;
        *reinterpret_cast<uint2*>(drow + c) = make_uint2(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]));
      }
    if (t == 0) {
      row_loss[r] = 0.f;
      if (pred != nullptr) pred[r] = -1;
    }
    return;
  }
  float m = -INFINITY, s = 0.f, best = -INFINITY;
  int bi = INT_MAX;
  for (int c = t * 4; c < V; c += kCeThreads * 4) {
    const float4 q = *reinterpret_cast<const float4*>(row + c);
    const float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c + j >= V) break;
      lse_merge(m, s, v[j], 1.f);
      if (v[j] > best) { best = v[j]; bi = c + j; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
    arg_merge(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
  }
  if (lane == 0) { sm_m[wid] = m; sm_s[wid] = s; sm_v[wid] = best; sm_i[wid] = bi; }
  __syncthreads();
  m = sm_m[0]; s = sm_s[0]; best = sm_v[0]; bi = sm_i[0];
  for (int w = 1; w < kCeThreads / 32; ++w) {     // every thread merges the warps in the same order
    lse_merge(m, s, sm_m[w], sm_s[w]);
    arg_merge(best, bi, sm_v[w], sm_i[w]);
  }
  const float lse = m + logf(s);
  if (t == 0) {
    row_loss[r] = lse - row[y];
    if (pred != nullptr) pred[r] = bi;
  }
  if (drow == nullptr) return;
  const float scale = (d_loss != nullptr ? *d_loss : 1.f) / (float)*n_lab;
  for (int c = t * 4; c < Vp; c += kCeThreads * 4) {
    float v[4];
    if (c < V) {
      const float4 q = *reinterpret_cast<const float4*>(row + c);
      const float x[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int cj = c + j;
        if (cj < V) {
          const float p = expf(x[j] - lse);
          v[j] = (cj == y ? p - 1.f : p) * scale;
          if (erow != nullptr) v[j] += erow[cj];
        } else {
          v[j] = 0.f;
        }
      }
    } else {
      v[0] = v[1] = v[2] = v[3] = 0.f;
    }
    *reinterpret_cast<uint2*>(drow + c) = make_uint2(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]));
  }
}

// loss = sum_r row_loss[r] / n_labelled, in a fixed order (thread-strided partial sums, then a fixed tree); nan when
// no row is labelled, as torch's mean over an all-ignored batch
__global__ void __launch_bounds__(1024) mlm_ce_mean_kernel(const float* __restrict__ row_loss, int rows,
                                                           const int* n_lab, float* loss) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[1024];
  const int t = threadIdx.x;
  float s = 0.f;
  for (int i = t; i < rows; i += 1024) s += row_loss[i];
  red[t] = s;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (t < w) red[t] += red[t + w];
    __syncthreads();
  }
  if (t == 0) *loss = red[0] / (float)*n_lab;
}

// grad = bf16(grad + dec): the decoder's dense part of the tied word-embedding gradient added to the embedding scatter
__global__ void mlm_tied_add_kernel(const float* __restrict__ dec, __nv_bfloat16* __restrict__ grad, long long n8) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    uint4 g = *reinterpret_cast<const uint4*>(grad + i * 8);
    const float4 a = *reinterpret_cast<const float4*>(dec + i * 8);
    const float4 b = *reinterpret_cast<const float4*>(dec + i * 8 + 4);
    g.x = pack_bf16(bf16_lo(g.x) + a.x, bf16_hi(g.x) + a.y);
    g.y = pack_bf16(bf16_lo(g.y) + a.z, bf16_hi(g.y) + a.w);
    g.z = pack_bf16(bf16_lo(g.z) + b.x, bf16_hi(g.z) + b.y);
    g.w = pack_bf16(bf16_lo(g.w) + b.z, bf16_hi(g.w) + b.w);
    *reinterpret_cast<uint4*>(grad + i * 8) = g;
  }
}

static unsigned grid_for(long long n, int threads) {
  long long g = (n + threads - 1) / threads;
  if (g > 132 * 16) g = 132 * 16;
  return (unsigned)(g < 1 ? 1 : g);
}

}  // namespace b2

using namespace b2;

extern "C" int32_t b2_mlm_compact(const int64_t* labels, int64_t tokens, int64_t ignore_index, int64_t vocab,
                                  int64_t capacity, int32_t* rows, int32_t* slot, int32_t* slot_labels,
                                  int32_t* count, void* stream) {
  B2_REQUIRE(labels && rows && slot && slot_labels && count, "mlm_compact: null pointer");
  B2_REQUIRE(tokens > 0 && tokens <= INT_MAX && vocab > 0, "mlm_compact: tokens=%lld vocab=%lld", (long long)tokens,
             (long long)vocab);
  B2_REQUIRE(capacity > 0 && capacity <= tokens, "mlm_compact: capacity=%lld must be in [1, tokens=%lld]",
             (long long)capacity, (long long)tokens);
  B2_LAUNCH(mlm_compact_kernel, 1, kCompactThreads, 0, stream, (const long long*)labels, (int)tokens,
            (long long)ignore_index, (long long)vocab, (int)capacity, (int*)rows, (int*)slot, (int*)slot_labels,
            (int*)count);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_mlm_gather_rows(const void* x, const int32_t* rows, const int32_t* count, int64_t capacity,
                                      int64_t hidden, void* out, void* stream) {
  B2_REQUIRE(x && rows && count && out, "mlm_gather_rows: null pointer");
  B2_REQUIRE(capacity > 0 && hidden % 8 == 0 && hidden >= 8 && hidden <= 8192,
             "mlm_gather_rows: capacity=%lld hidden=%lld", (long long)capacity, (long long)hidden);
  B2_LAUNCH(mlm_gather_kernel, (unsigned)capacity, (unsigned)(hidden / 8), 0, stream, (const __nv_bfloat16*)x,
            (const int*)rows, (const int*)count, (int)hidden, (__nv_bfloat16*)out);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_mlm_scatter_rows(const float* src, const int32_t* slot, int64_t tokens, int64_t hidden,
                                       float* dx, void* stream) {
  B2_REQUIRE(src && slot && dx, "mlm_scatter_rows: null pointer");
  B2_REQUIRE(tokens > 0 && hidden % 4 == 0 && hidden >= 4 && hidden <= 4096,
             "mlm_scatter_rows: tokens=%lld hidden=%lld", (long long)tokens, (long long)hidden);
  B2_LAUNCH(mlm_scatter_kernel, (unsigned)tokens, (unsigned)(hidden / 4), 0, stream, src, (const int*)slot,
            (int)hidden, dx);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_mlm_gelu_bwd(const float* dg, const void* u, int64_t n, void* du, void* stream) {
  B2_REQUIRE(dg && u && du, "mlm_gelu_bwd: null pointer");
  B2_REQUIRE(n > 0 && n % 8 == 0, "mlm_gelu_bwd: n=%lld must be a positive multiple of 8", (long long)n);
  B2_LAUNCH(mlm_gelu_bwd_kernel, grid_for(n / 8, 256), 256, 0, stream, dg, (const __nv_bfloat16*)u,
            (long long)(n / 8), (__nv_bfloat16*)du);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_mlm_bias_fill(const void* bias, int64_t rows, int64_t vocab_pad, float* logits, void* stream) {
  B2_REQUIRE(bias && logits, "mlm_bias_fill: null pointer");
  B2_REQUIRE(rows > 0 && vocab_pad > 0 && vocab_pad % 64 == 0, "mlm_bias_fill: rows=%lld vocab_pad=%lld",
             (long long)rows, (long long)vocab_pad);
  const long long n4 = rows * vocab_pad / 4;
  B2_LAUNCH(mlm_bias_fill_kernel, grid_for(n4, 256), 256, 0, stream, (const __nv_bfloat16*)bias, n4,
            (int)(vocab_pad / 4), logits);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_mlm_ce(const float* logits, int64_t rows, int64_t vocab, int64_t vocab_pad,
                             const int32_t* labels, const int32_t* n_rows, const int32_t* n_labelled,
                             const float* d_loss, const float* d_extra, int64_t ld_extra, float* row_loss,
                             int32_t* pred, void* d_logits, float* loss, void* stream) {
  B2_REQUIRE(logits && row_loss && n_labelled, "mlm_ce: null pointer");
  B2_REQUIRE(rows > 0 && rows <= INT_MAX, "mlm_ce: rows=%lld", (long long)rows);
  B2_REQUIRE(vocab > 0 && vocab_pad % 64 == 0 && vocab_pad >= vocab && vocab_pad - vocab < 64,
             "mlm_ce: vocab=%lld vocab_pad=%lld (the vocabulary rounded up to 64)", (long long)vocab,
             (long long)vocab_pad);
  B2_REQUIRE(d_extra == nullptr || (d_logits != nullptr && ld_extra >= vocab),
             "mlm_ce: d_extra needs d_logits and ld_extra >= vocab");
  B2_LAUNCH(mlm_ce_kernel, (unsigned)rows, kCeThreads, 0, stream, logits, (int)vocab, (int)vocab_pad,
            (const int*)labels, (const int*)n_rows, (const int*)n_labelled, d_loss, d_extra, (long long)ld_extra,
            row_loss, (int*)pred, (__nv_bfloat16*)d_logits);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  if (loss != nullptr) {
    B2_LAUNCH(mlm_ce_mean_kernel, 1, 1024, 0, stream, (const float*)row_loss, (int)rows, (const int*)n_labelled, loss);
    B2_CUDA(cudaGetLastError());
    count_launches(1);
  }
  return 0;
}

extern "C" int32_t b2_mlm_tied_add(const float* dec, void* grad, int64_t n, void* stream) {
  B2_REQUIRE(dec && grad, "mlm_tied_add: null pointer");
  B2_REQUIRE(n > 0 && n % 8 == 0, "mlm_tied_add: n=%lld must be a positive multiple of 8", (long long)n);
  B2_LAUNCH(mlm_tied_add_kernel, grid_for(n / 8, 256), 256, 0, stream, dec, (__nv_bfloat16*)grad, (long long)(n / 8));
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}
