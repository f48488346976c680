// Classification head: BertPooler (tanh(h[:,0] Wp^T + bp), modeling_bert.py:462-468), classifier dropout + Linear
// (:1123-1124) and the mean cross-entropy the reference's Trainer applies (multi-gpu-distributed-cls.py:169,343),
// forward and backward.  Work is tiny (batch x hidden): warp-per-output dot products, fp32 math, launch-latency
// bound by construction (SURVEY.md K10-K12).
#include "common.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

// dot of two bf16 vectors of length H (H % 256 == 0) spread over a warp
__device__ __forceinline__ float warp_dot_bf16(const __nv_bfloat16* __restrict__ a,
                                               const __nv_bfloat16* __restrict__ b, int H, int lane) {
  float s = 0.f;
  for (int c = lane * 8; c < H; c += 256) {
    const uint4 x = ldg16(a + c), y = ldg16(b + c);
    s += bf16_lo(x.x) * bf16_lo(y.x) + bf16_hi(x.x) * bf16_hi(y.x) + bf16_lo(x.y) * bf16_lo(y.y) +
         bf16_hi(x.y) * bf16_hi(y.y) + bf16_lo(x.z) * bf16_lo(y.z) + bf16_hi(x.z) * bf16_hi(y.z) +
         bf16_lo(x.w) * bf16_lo(y.w) + bf16_hi(x.w) * bf16_hi(y.w);
  }
  return warp_sum(s);
}

// pooled[b, j] = tanh(h[b*seq, :] . Wp[j, :] + bp[j]); one warp per (j, group of 8 batch rows): the weight row is
// read once per warp and reused for the 8 dot products.  grid = (H/8, ceil(batch/8))
// cls_rows (optional, packed bins): row of sequence b's first token; default b * seq
__global__ void __launch_bounds__(256) pooler_fwd_kernel(const __nv_bfloat16* __restrict__ h,
                                                        const long long* __restrict__ cls_rows, int batch, int seq,
                                                        int H, const __nv_bfloat16* __restrict__ Wp,
                                                        const __nv_bfloat16* __restrict__ bp,
                                                        __nv_bfloat16* __restrict__ pooled) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int b0 = blockIdx.y * 8;
  if (j >= H) return;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int c = lane * 8; c < H; c += 256) {
    const uint4 w = ldg16(Wp + (size_t)j * H + c);
    const float wv[8] = {bf16_lo(w.x), bf16_hi(w.x), bf16_lo(w.y), bf16_hi(w.y),
                         bf16_lo(w.z), bf16_hi(w.z), bf16_lo(w.w), bf16_hi(w.w)};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (b0 + i < batch) {
        const size_t r = cls_rows != nullptr ? (size_t)cls_rows[b0 + i] : (size_t)(b0 + i) * seq;
        const uint4 x = ldg16(h + r * H + c);
        acc[i] += wv[0] * bf16_lo(x.x) + wv[1] * bf16_hi(x.x) + wv[2] * bf16_lo(x.y) + wv[3] * bf16_hi(x.y) +
                  wv[4] * bf16_lo(x.z) + wv[5] * bf16_hi(x.z) + wv[6] * bf16_lo(x.w) + wv[7] * bf16_hi(x.w);
      }
    }
  }
  const float bias = __bfloat162float(bp[j]);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float s = warp_sum(acc[i]);
    if (lane == 0 && b0 + i < batch) pooled[(size_t)(b0 + i) * H + j] = __float2bfloat16_rn(tanhf(s + bias));
  }
}

// logits[b, c] = dropout(pooled[b, :]) . Wc[c, :] + bc[c]; one warp per (b, c)
__global__ void __launch_bounds__(256) classifier_fwd_kernel(const __nv_bfloat16* __restrict__ pooled, int batch,
                                                            int H, const __nv_bfloat16* __restrict__ Wc,
                                                            const __nv_bfloat16* __restrict__ bc, int C,
                                                            float dropout_p, const unsigned long long* rng,
                                                            unsigned site, float* __restrict__ logits) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int o = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (o >= batch * C) return;
  const int b = o / C, c = o % C;
  const DropCtx drop = make_drop_ctx(rng, site, dropout_p);
  float s = 0.f;
  for (int k = lane * 8; k < H; k += 256) {
    const uint4 x = ldg16(pooled + (size_t)b * H + k), w = ldg16(Wc + (size_t)c * H + k);
    const uint32_t keep = dropout_keep8(drop, (unsigned long long)b * H + k);
    const float xv[8] = {bf16_lo(x.x), bf16_hi(x.x), bf16_lo(x.y), bf16_hi(x.y),
                         bf16_lo(x.z), bf16_hi(x.z), bf16_lo(x.w), bf16_hi(x.w)};
    const float wv[8] = {bf16_lo(w.x), bf16_hi(w.x), bf16_lo(w.y), bf16_hi(w.y),
                         bf16_lo(w.z), bf16_hi(w.z), bf16_lo(w.w), bf16_hi(w.w)};
#pragma unroll
    for (int i = 0; i < 8; ++i) s += (((keep >> i) & 1u) ? xv[i] * drop.scale : 0.f) * wv[i];
  }
  s = warp_sum(s);
  if (lane == 0) logits[o] = s + __bfloat162float(bc[c]);
}

// mean CE over the batch + dlogits = (softmax - onehot) / batch.  One block, one thread per sample (strided).
__global__ void __launch_bounds__(256) ce_fwd_bwd_kernel(const float* __restrict__ logits,
                                                        const long long* __restrict__ labels, int batch, int C,
                                                        float* __restrict__ loss, float* __restrict__ dlogits) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  // torch.nn.CrossEntropyLoss semantics (multi-gpu-distributed-cls.py:343, defaults): labels equal to ignore_index
  // (-100) contribute nothing and the mean runs over the other samples; any other label outside [0, C) is an error
  // (torch raises a device-side assert: here a message + trap)
  __shared__ float red[256];
  __shared__ int cnt[256];
  int valid = 0;
  for (int b = threadIdx.x; b < batch; b += blockDim.x) {
    const long long y = labels[b];
    if (y == -100) continue;
    if (y < 0 || y >= C) {
      printf("b2 ce_fwd_bwd: label %lld of sample %d is outside [0, %d) (and is not ignore_index -100)\n", y, b, C);
      __trap();
    }
    ++valid;
  }
  cnt[threadIdx.x] = valid;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) cnt[threadIdx.x] += cnt[threadIdx.x + s];
    __syncthreads();
  }
  const int n_valid = cnt[0];
  const float inv = n_valid > 0 ? 1.0f / (float)n_valid : 0.f;
  float local = 0.f;
  for (int b = threadIdx.x; b < batch; b += blockDim.x) {
    const float* z = logits + (size_t)b * C;
    const long long y = labels[b];
    if (y == -100) {
      if (dlogits != nullptr)
        for (int c = 0; c < C; ++c) dlogits[(size_t)b * C + c] = 0.f;
      continue;
    }
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, z[c]);
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(z[c] - mx);
    const float lse = mx + logf(se);
    local += lse - z[y];
    if (dlogits != nullptr) {
      for (int c = 0; c < C; ++c)
        dlogits[(size_t)b * C + c] = (expf(z[c] - lse) - (c == (int)y ? 1.f : 0.f)) * inv;
    }
  }
  red[threadIdx.x] = local;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  // all samples ignored: torch returns nan (0 / 0)
  if (threadIdx.x == 0) *loss = n_valid > 0 ? red[0] * inv : __int_as_float(0x7fc00000);
}

// ---- backward ----
// k1: one thread per (b, j): dpd = sum_c dlogits[b,c] Wc[c,j] -> d_pooled = mask*scale*dpd -> d_pre = d_pooled*(1 -
//     pooled^2) (fp32 scratch [batch, H]); also pm[b,j] = dropout(pooled)[b,j] (second fp32 scratch plane) for k1b.
//     grid = (ceil(H/256), batch).  (Looping over the batch inside a few blocks is pure latency at the head of the
//     backward critical path.)
__global__ void __launch_bounds__(256) head_bwd_k1(const float* __restrict__ dlogits,
                                                  const __nv_bfloat16* __restrict__ pooled, int batch, int H,
                                                  const __nv_bfloat16* __restrict__ Wc, int C, float dropout_p,
                                                  const unsigned long long* rng, unsigned site,
                                                  float* __restrict__ d_pre, float* __restrict__ pm) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (j >= H) return;
  const DropCtx drop = make_drop_ctx(rng, site, dropout_p);
  const float p = __bfloat162float(pooled[(size_t)b * H + j]);
  const uint32_t keep8 = dropout_keep8(drop, ((unsigned long long)b * H + j) & ~7ull);
  const float m = ((keep8 >> (j & 7)) & 1u) ? drop.scale : 0.f;
  float dpd = 0.f;
  for (int c = 0; c < C; ++c) dpd = fmaf(dlogits[(size_t)b * C + c], __bfloat162float(Wc[(size_t)c * H + j]), dpd);
  d_pre[(size_t)b * H + j] = dpd * m * (1.f - p * p);
  pm[(size_t)b * H + j] = p * m;
}
// k1b: classifier grads: d_cls_w[c,j] = sum_b dlogits[b,c] * pm[b,j];  d_cls_b[c] = sum_b dlogits[b,c].
//     grid = (ceil(H/256), C)
__global__ void __launch_bounds__(256) head_bwd_k1b(const float* __restrict__ dlogits, const float* __restrict__ pm,
                                                   int batch, int H, int C, __nv_bfloat16* __restrict__ d_cls_w,
                                                   __nv_bfloat16* __restrict__ d_cls_b) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (j >= H) return;
  float s = 0.f, sb = 0.f;
  for (int b = 0; b < batch; ++b) {
    const float dl = dlogits[(size_t)b * C + c];
    s = fmaf(dl, pm[(size_t)b * H + j], s);
    sb += dl;
  }
  d_cls_w[(size_t)c * H + j] = __float2bfloat16_rn(s);
  if (j == 0) d_cls_b[c] = __float2bfloat16_rn(sb);
}

// k2: d_pool_w[j, k] = sum_b d_pre[b, j] * h0[b, k];  d_pool_b[j] = sum_b d_pre[b, j].
//     grid = H rows (j), threads = H/8 (each 8 consecutive k)
__global__ void head_bwd_k2(const float* __restrict__ d_pre, const __nv_bfloat16* __restrict__ h,
                            const long long* __restrict__ cls_rows, int batch, int seq, int H,
                            __nv_bfloat16* __restrict__ d_pool_w, __nv_bfloat16* __restrict__ d_pool_b) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int j = blockIdx.x;
  const int k = threadIdx.x * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float sb = 0.f;
  for (int b = 0; b < batch; ++b) {
    const float d = d_pre[(size_t)b * H + j];
    sb += d;
    const size_t r = cls_rows != nullptr ? (size_t)cls_rows[b] : (size_t)b * seq;
    const uint4 x = ldg16(h + r * H + k);
    acc[0] += d * bf16_lo(x.x); acc[1] += d * bf16_hi(x.x); acc[2] += d * bf16_lo(x.y); acc[3] += d * bf16_hi(x.y);
    acc[4] += d * bf16_lo(x.z); acc[5] += d * bf16_hi(x.z); acc[6] += d * bf16_lo(x.w); acc[7] += d * bf16_hi(x.w);
  }
  uint4 o;
  o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]);
  o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
  stg16(d_pool_w + (size_t)j * H + k, o);
  if (threadIdx.x == 0) d_pool_b[j] = __float2bfloat16_rn(sb);
}

// k3: d_h0[b, k] = sum_j d_pre[b, j] * Wp[j, k]  -> written into row b*seq of d_hidden (other rows pre-zeroed)
//     grid = (batch, H/64), 8 warps: warp w sums its eighth of the j range for 64 columns (2 per lane), smem reduce
__global__ void __launch_bounds__(256) head_bwd_k3(const float* __restrict__ d_pre,
                                                  const __nv_bfloat16* __restrict__ Wp,
                                                  const long long* __restrict__ cls_rows, int seq, int H,
                                                  void* __restrict__ d_hidden, int out_f32) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  __shared__ float red[8][64];
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k = blockIdx.y * 64 + lane * 2;
  const int jn = H / 8;
  float a0 = 0.f, a1 = 0.f;
  for (int j = warp * jn; j < (warp + 1) * jn; ++j) {
    const float d = d_pre[(size_t)b * H + j];
    const uint32_t w = *reinterpret_cast<const uint32_t*>(Wp + (size_t)j * H + k);
    a0 = fmaf(d, bf16_lo(w), a0);
    a1 = fmaf(d, bf16_hi(w), a1);
  }
  red[warp][lane * 2] = a0;
  red[warp][lane * 2 + 1] = a1;
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    const size_t r = cls_rows != nullptr ? (size_t)cls_rows[b] : (size_t)b * seq;
    const size_t o = r * H + blockIdx.y * 64 + threadIdx.x;
    if (out_f32) reinterpret_cast<float*>(d_hidden)[o] = s;
    else reinterpret_cast<__nv_bfloat16*>(d_hidden)[o] = __float2bfloat16_rn(s);
  }
}

}  // namespace b2

using namespace b2;

static int32_t head_fwd_impl(const void* hidden_states, const int64_t* cls_rows, int64_t batch, int64_t seq,
                             int64_t hidden, const void* pool_w, const void* pool_b, const void* cls_w,
                             const void* cls_b, int64_t num_labels, float dropout_p, const void* rng_state,
                             uint32_t rng_site, void* pooled, float* logits, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  B2_REQUIRE(hidden_states && pool_w && pool_b && cls_w && cls_b && pooled && logits, "head_fwd: null pointer");
  B2_REQUIRE(batch > 0 && seq > 0 && num_labels > 0, "head_fwd: empty problem");
  B2_REQUIRE(hidden % 256 == 0, "head_fwd: hidden=%lld must be a multiple of 256", (long long)hidden);
  B2_REQUIRE(!(dropout_p > 0.f) || rng_state, "head_fwd: dropout needs rng_state");
  B2_LAUNCH(pooler_fwd_kernel, dim3((unsigned)((hidden + 7) / 8), (unsigned)((batch + 7) / 8)), 256, 0, stream, 
      (const __nv_bfloat16*)hidden_states, (const long long*)cls_rows, (int)batch, (int)seq, (int)hidden,
      (const __nv_bfloat16*)pool_w, (const __nv_bfloat16*)pool_b, (__nv_bfloat16*)pooled);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  B2_LAUNCH(classifier_fwd_kernel, (unsigned)((batch * num_labels + 7) / 8), 256, 0, stream, 
      (const __nv_bfloat16*)pooled, (int)batch, (int)hidden, (const __nv_bfloat16*)cls_w, (const __nv_bfloat16*)cls_b,
      (int)num_labels, dropout_p, (const unsigned long long*)rng_state, rng_site, logits);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_head_fwd(const void* hidden_states, int64_t batch, int64_t seq, int64_t hidden,
                               const void* pool_w, const void* pool_b, const void* cls_w, const void* cls_b,
                               int64_t num_labels, float dropout_p, const void* rng_state, uint32_t rng_site,
                               void* pooled, float* logits, void* stream_) {
  return head_fwd_impl(hidden_states, nullptr, batch, seq, hidden, pool_w, pool_b, cls_w, cls_b, num_labels,
                       dropout_p, rng_state, rng_site, pooled, logits, stream_);
}

extern "C" int32_t b2_head_fwd_packed(const void* hidden_states, const int64_t* cls_rows, int64_t batch,
                                      int64_t hidden, const void* pool_w, const void* pool_b, const void* cls_w,
                                      const void* cls_b, int64_t num_labels, float dropout_p, const void* rng_state,
                                      uint32_t rng_site, void* pooled, float* logits, void* stream_) {
  B2_REQUIRE(cls_rows != nullptr, "head_fwd_packed: null cls_rows");
  return head_fwd_impl(hidden_states, cls_rows, batch, 1, hidden, pool_w, pool_b, cls_w, cls_b, num_labels,
                       dropout_p, rng_state, rng_site, pooled, logits, stream_);
}

extern "C" int32_t b2_ce_fwd_bwd(const float* logits, const int64_t* labels, int64_t batch, int64_t num_labels,
                                 float* loss, float* dlogits, void* stream_) {
  B2_REQUIRE(logits && labels && loss, "ce_fwd_bwd: null pointer");
  B2_REQUIRE(batch > 0 && num_labels > 0, "ce_fwd_bwd: empty batch");
  B2_LAUNCH(ce_fwd_bwd_kernel, 1, 256, 0, (cudaStream_t)stream_, logits, (const long long*)labels, (int)batch,
                                                          (int)num_labels, loss, dlogits);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

static int32_t head_bwd_impl(const float* dlogits, const void* hidden_states, const void* pooled,
                             const int64_t* cls_rows, int64_t tokens, int64_t batch,
                               int64_t seq, int64_t hidden, const void* pool_w, const void* cls_w, int64_t num_labels,
                               float dropout_p, const void* rng_state, uint32_t rng_site, void* d_pool_w,
                               void* d_pool_b, void* d_cls_w, void* d_cls_b, void* d_hidden, int32_t d_hidden_fp32,
                               float* scratch, void* stream_, void* weight_stream_ = nullptr) {
  cudaStream_t stream = (cudaStream_t)stream_;
  B2_REQUIRE(dlogits && hidden_states && pooled && pool_w && cls_w && d_pool_w && d_pool_b && d_cls_w && d_cls_b &&
                 d_hidden && scratch,
             "head_bwd: null pointer");
  B2_REQUIRE(batch > 0 && seq > 0, "head_bwd: empty batch");
  B2_REQUIRE(hidden % 256 == 0 && hidden / 8 <= 1024, "head_bwd: hidden=%lld unsupported", (long long)hidden);
  B2_REQUIRE(num_labels >= 1 && num_labels <= 65535, "head_bwd: num_labels=%lld", (long long)num_labels);
  B2_CUDA(cudaMemsetAsync(d_hidden, 0, (size_t)tokens * hidden * (d_hidden_fp32 ? 4 : 2), stream));
  float* pm = scratch + (size_t)batch * hidden;   // second scratch plane: dropout(pooled)
  B2_LAUNCH(head_bwd_k1, dim3((unsigned)((hidden + 255) / 256), (unsigned)batch), 256, 0, stream, dlogits,
            (const __nv_bfloat16*)pooled, (int)batch, (int)hidden, (const __nv_bfloat16*)cls_w, (int)num_labels,
            dropout_p, (const unsigned long long*)rng_state, rng_site, scratch, pm);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  // the critical path continues with k3 (d_hidden); the two weight-gradient kernels follow it
  B2_LAUNCH(head_bwd_k3, dim3((unsigned)batch, (unsigned)(hidden / 64)), 256, 0, stream, scratch,
            (const __nv_bfloat16*)pool_w, (const long long*)cls_rows, (int)seq, (int)hidden, d_hidden,
            d_hidden_fp32 ? 1 : 0);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  // The two parameter-gradient kernels are off the critical path (only the optimizer / exchange consumes them): on
  // request they go to the caller's weight-gradient stream, ordered behind k1 (which fills `scratch` / `pm`) by an
  // event, so the main stream continues with the encoder's backward right after k3
  cudaStream_t wstream = stream;
  if (weight_stream_ != nullptr && (cudaStream_t)weight_stream_ != stream) {
    static thread_local cudaEvent_t ev = nullptr;
    if (ev == nullptr) B2_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    B2_CUDA(cudaEventRecord(ev, stream));
    wstream = (cudaStream_t)weight_stream_;
    B2_CUDA(cudaStreamWaitEvent(wstream, ev, 0));
  }
  B2_LAUNCH(head_bwd_k1b, dim3((unsigned)((hidden + 255) / 256), (unsigned)num_labels), 256, 0, wstream, dlogits, pm,
            (int)batch, (int)hidden, (int)num_labels, (__nv_bfloat16*)d_cls_w, (__nv_bfloat16*)d_cls_b);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  B2_LAUNCH(head_bwd_k2, (unsigned)hidden, (unsigned)(hidden / 8), 0, wstream, 
      scratch, (const __nv_bfloat16*)hidden_states, (const long long*)cls_rows, (int)batch, (int)seq, (int)hidden,
      (__nv_bfloat16*)d_pool_w, (__nv_bfloat16*)d_pool_b);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_head_bwd(const float* dlogits, const void* hidden_states, const void* pooled, int64_t batch,
                               int64_t seq, int64_t hidden, const void* pool_w, const void* cls_w, int64_t num_labels,
                               float dropout_p, const void* rng_state, uint32_t rng_site, void* d_pool_w,
                               void* d_pool_b, void* d_cls_w, void* d_cls_b, void* d_hidden, int32_t d_hidden_fp32,
                               float* scratch, void* stream_) {
  return head_bwd_impl(dlogits, hidden_states, pooled, nullptr, batch * seq, batch, seq, hidden, pool_w, cls_w,
                       num_labels, dropout_p, rng_state, rng_site, d_pool_w, d_pool_b, d_cls_w, d_cls_b, d_hidden,
                       d_hidden_fp32, scratch, stream_);
}

extern "C" int32_t b2_head_bwd_packed(const float* dlogits, const void* hidden_states, const void* pooled,
                                      const int64_t* cls_rows, int64_t tokens, int64_t batch, int64_t hidden,
                                      const void* pool_w, const void* cls_w, int64_t num_labels, float dropout_p,
                                      const void* rng_state, uint32_t rng_site, void* d_pool_w, void* d_pool_b,
                                      void* d_cls_w, void* d_cls_b, void* d_hidden, int32_t d_hidden_fp32,
                                      float* scratch, void* stream_) {
  B2_REQUIRE(cls_rows != nullptr && tokens > 0, "head_bwd_packed: null cls_rows / no tokens");
  return head_bwd_impl(dlogits, hidden_states, pooled, cls_rows, tokens, batch, 1, hidden, pool_w, cls_w, num_labels,
                       dropout_p, rng_state, rng_site, d_pool_w, d_pool_b, d_cls_w, d_cls_b, d_hidden, d_hidden_fp32,
                       scratch, stream_);
}

// b2_head_bwd / b2_head_bwd_packed with the two parameter-gradient kernels on a second stream (cls_rows may be NULL:
// row of sequence b = b * seq).  The caller must order whatever consumes d_pool_w / d_pool_b / d_cls_w / d_cls_b
// behind `weight_stream`.
extern "C" int32_t b2_head_bwd_split(const float* dlogits, const void* hidden_states, const void* pooled,
                                     const int64_t* cls_rows, int64_t tokens, int64_t batch, int64_t seq,
                                     int64_t hidden, const void* pool_w, const void* cls_w, int64_t num_labels,
                                     float dropout_p, const void* rng_state, uint32_t rng_site, void* d_pool_w,
                                     void* d_pool_b, void* d_cls_w, void* d_cls_b, void* d_hidden,
                                     int32_t d_hidden_fp32, float* scratch, void* stream_, void* weight_stream_) {
  B2_REQUIRE(tokens > 0 && (cls_rows != nullptr || tokens == batch * seq), "head_bwd_split: tokens / seq mismatch");
  return head_bwd_impl(dlogits, hidden_states, pooled, cls_rows, tokens, batch, cls_rows ? 1 : seq, hidden, pool_w,
                       cls_w, num_labels, dropout_p, rng_state, rng_site, d_pool_w, d_pool_b, d_cls_w, d_cls_b,
                       d_hidden, d_hidden_fp32, scratch, stream_, weight_stream_);
}
