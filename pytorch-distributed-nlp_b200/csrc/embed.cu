// BertEmbeddings forward / backward (SP/transformers/models/bert/modeling_bert.py:72-112; SURVEY.md K1).
// forward : word + position + token-type gather, add, LayerNorm, dropout, one warp per token, one pass over HBM.
// backward: LayerNorm backward, then deterministic scatter-adds:
//   word rows      keyed by the "owner" token of each touched vocabulary row (lowest token index wins an atomicMin):
//                  fast path = every token adds its row into fp32 acc[owner] (vector reductions at L2: the order of a
//                  duplicated row's adds varies), the owner converts; ordered entry points and fallback (scratch too
//                  small) = the owner CTA scans the later tokens in order (no float atomics, bit-reproducible);
//   position rows  row s = sum over the batch of dx[b, s, :]  } one pass (embed_pos_type_kernel) on the fast path,
//   type rows      filtered column sums                        } separate kernels on the fallback.
#include "common.cuh"
#include "layernorm.cuh"
#include "../../include/b2_ddp_bert.h"

#include <climits>

namespace b2 {

template <int VPL>
__global__ void __launch_bounds__(128) embed_fwd_kernel(
    const long long* __restrict__ input_ids, const long long* __restrict__ token_type_ids,
    const long long* __restrict__ position_ids /* null: position = token index % seq */, int max_pos,
    int* __restrict__ pos32 /* null unless position_ids */, int tokens, int seq,
    const __nv_bfloat16* __restrict__ word, const __nv_bfloat16* __restrict__ pos,
    const __nv_bfloat16* __restrict__ type, const __nv_bfloat16* __restrict__ gamma,
    const __nv_bfloat16* __restrict__ beta, int vocab, int type_vocab, float eps, float dropout_p,
    const unsigned long long* rng, unsigned rng_site, __nv_bfloat16* __restrict__ y,
    float* __restrict__ y_f32 /* optional: the same output unrounded, the first residual of the fp32 stream */,
    __nv_bfloat16* __restrict__ pre_ln, float* __restrict__ mean_out, float* __restrict__ rstd_out,
    int* __restrict__ ids32, int* __restrict__ tt32) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  constexpr int H = VPL * 256;
  const int t = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= tokens) return;
  long long id = input_ids[t];
  long long tt = token_type_ids ? token_type_ids[t] : 0;
  // out-of-range ids would be a host bug; clamp so a bad batch cannot fault the GPU (host validates too)
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  tt = tt < 0 ? 0 : (tt >= type_vocab ? type_vocab - 1 : tt);
  int s = t % seq;
  if (position_ids != nullptr) {       // packed bins: every token keeps the position it had in its own sequence
    const long long ps = position_ids[t];
    s = ps < 0 ? 0 : (ps >= max_pos ? max_pos - 1 : (int)ps);
  }
  float v[VPL * 8], a[VPL * 8];
  load_row<VPL>(word + (size_t)id * H, lane, v);
  load_row<VPL>(pos + (size_t)s * H, lane, a);
#pragma unroll
  for (int i = 0; i < VPL * 8; ++i) v[i] += a[i];
  load_row<VPL>(type + (size_t)tt * H, lane, a);
#pragma unroll
  for (int i = 0; i < VPL * 8; ++i) v[i] += a[i];
  store_row<VPL>(pre_ln + (size_t)t * H, lane, v);
  float mean, rstd;
  row_stats<VPL>(v, eps, mean, rstd);
  normalize<VPL>(v, mean, rstd, gamma, beta, lane);
  const DropCtx drop = make_drop_ctx(rng, rng_site, dropout_p);
  if (drop.thresh != 0) {
#pragma unroll
    for (int vv = 0; vv < VPL; ++vv) {
      const uint32_t keep = dropout_keep8(drop, (unsigned long long)t * H + (vv * 32 + lane) * 8);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[vv * 8 + i] = ((keep >> i) & 1u) ? v[vv * 8 + i] * drop.scale : 0.f;
    }
  }
  store_row<VPL>(y + (size_t)t * H, lane, v);
  if (y_f32 != nullptr) store_row_f32<VPL>(y_f32 + (size_t)t * H, lane, v);
  if (lane == 0) {
    mean_out[t] = mean;
    rstd_out[t] = rstd;
    ids32[t] = (int)id;
    tt32[t] = (int)tt;
    if (pos32 != nullptr) pos32[t] = s;
  }
}

__global__ void embed_owner_kernel(const int* __restrict__ ids32, int tokens, int pad_id,
                                   int* __restrict__ owner) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < tokens && ids32[t] != pad_id) atomicMin(&owner[ids32[t]], t);
}

// one CTA per token; only the owner of a vocabulary row does work.  Threads = H/8 (one 16-byte vector each).
__global__ void embed_word_scatter_kernel(const __nv_bfloat16* __restrict__ dx, const int* __restrict__ ids32,
                                          int tokens, int H, int pad_id, int* __restrict__ owner,
                                          __nv_bfloat16* __restrict__ d_word) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int t = blockIdx.x;
  const int id = ids32[t];
  // nn.Embedding(padding_idx=pad_token_id): the pad row never receives gradient (stays at the caller's zero fill)
  if (id == pad_id || owner[id] != t) return;
  const int nvec = H / 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  // occurrences of `id` can only be at token indices >= t (t is the minimum)
  for (int base = t; base < tokens; base += blockDim.x) {
    const int tp = base + threadIdx.x;
    const bool hit = (tp < tokens) && (ids32[tp] == id);
    // every warp needs the hits of the whole block: exchange through smem
    __shared__ unsigned hits[32];
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0) hits[threadIdx.x >> 5] = b;
    __syncthreads();
    const int nw = blockDim.x >> 5;
    for (int w = 0; w < nw; ++w) {
      unsigned m = hits[w];
      while (m) {
        const int bit = __ffs(m) - 1;
        m &= m - 1;
        const int src = base + w * 32 + bit;
        if ((int)threadIdx.x < nvec) {
          const uint4 v = ldg16(dx + (size_t)src * H + threadIdx.x * 8);
          acc[0] += bf16_lo(v.x); acc[1] += bf16_hi(v.x); acc[2] += bf16_lo(v.y); acc[3] += bf16_hi(v.y);
          acc[4] += bf16_lo(v.z); acc[5] += bf16_hi(v.z); acc[6] += bf16_lo(v.w); acc[7] += bf16_hi(v.w);
        }
      }
    }
    __syncthreads();
  }
  if ((int)threadIdx.x < nvec) {
    uint4 o;
    o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]);
    o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
    stg16(d_word + (size_t)id * H + threadIdx.x * 8, o);
  }
  if (threadIdx.x == 0) owner[id] = INT_MAX;  // leave the table armed for the next step
}

// d_pos[s] = sum_b dx[b*seq + s]  (rows >= seq get zero).  grid = max_pos rows, threads = H/8
__global__ void embed_pos_kernel(const __nv_bfloat16* __restrict__ dx, int batch, int seq, int H,
                                 __nv_bfloat16* __restrict__ d_pos) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int s = blockIdx.x;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (s < seq) {
    for (int b = 0; b < batch; ++b) {
      const uint4 v = ldg16(dx + ((size_t)b * seq + s) * H + threadIdx.x * 8);
      acc[0] += bf16_lo(v.x); acc[1] += bf16_hi(v.x); acc[2] += bf16_lo(v.y); acc[3] += bf16_hi(v.y);
      acc[4] += bf16_lo(v.z); acc[5] += bf16_hi(v.z); acc[6] += bf16_lo(v.w); acc[7] += bf16_hi(v.w);
    }
  }
  uint4 o;
  o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]);
  o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
  stg16(d_pos + (size_t)s * H + threadIdx.x * 8, o);
}

// ---- fast word-row path: fp32 accumulation keyed by the OWNER TOKEN of each vocabulary row ---------------------
// acc[owner[id]][:] += dx[t][:] for every token (vector reductions at L2; a row met once is a single add into
// zero, i.e. exact), then the owner converts its row to bf16.  Two fully parallel passes instead of one CTA per
// token scanning all later tokens for duplicates; the summation order of duplicated rows is
// no longer fixed (fp32 accumulation, rounded once).
__global__ void embed_word_accum_kernel(const __nv_bfloat16* __restrict__ dx, const int* __restrict__ ids32, int H,
                                        int pad_id, const int* __restrict__ owner, float* __restrict__ acc) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int t = blockIdx.x;
  const int id = ids32[t];
  if (id == pad_id) return;   // nn.Embedding(padding_idx): the pad row never receives gradient
  const int o = owner[id];
  const uint4 v = ldg16(dx + (size_t)t * H + threadIdx.x * 8);
  float* dst = acc + (size_t)o * H + threadIdx.x * 8;
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(bf16_lo(v.x)), "f"(bf16_hi(v.x)),
               "f"(bf16_lo(v.y)), "f"(bf16_hi(v.y))
               : "memory");
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + 4), "f"(bf16_lo(v.z)), "f"(bf16_hi(v.z)),
               "f"(bf16_lo(v.w)), "f"(bf16_hi(v.w))
               : "memory");
}
__global__ void embed_word_finish_kernel(const float* __restrict__ acc, const int* __restrict__ ids32, int H, int pad_id,
                                         int* __restrict__ owner, __nv_bfloat16* __restrict__ d_word) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int t = blockIdx.x;
  const int id = ids32[t];
  if (id == pad_id || owner[id] != t) return;   // non-owners never match: owner[id] is the minimum index or INT_MAX
  const float4 a = *reinterpret_cast<const float4*>(acc + (size_t)t * H + threadIdx.x * 8);
  const float4 b = *reinterpret_cast<const float4*>(acc + (size_t)t * H + threadIdx.x * 8 + 4);
  uint4 o;
  o.x = pack_bf16(a.x, a.y); o.y = pack_bf16(a.z, a.w);
  o.z = pack_bf16(b.x, b.y); o.w = pack_bf16(b.z, b.w);
  stg16(d_word + (size_t)id * H + threadIdx.x * 8, o);
  __syncthreads();
  if (threadIdx.x == 0) owner[id] = INT_MAX;    // leave the table armed for the next step
}

// position rows and per-position token-type partial sums in one pass: CTA s walks the batch once.
//   d_pos[s] = sum_b dx[b*seq + s];  type_part[s][ty] = sum over the same rows with tt == ty (fp32, ty < T <= 3)
constexpr int kMaxTypeFast = 3;
__global__ void embed_pos_type_kernel(const __nv_bfloat16* __restrict__ dx, const int* __restrict__ tt32,
                                      const int* __restrict__ pos32 /* null: position = token index % seq */,
                                      int batch, int seq, int H, int T, __nv_bfloat16* __restrict__ d_pos,
                                      float* __restrict__ type_part /* [seq][T][H] */) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int s = blockIdx.x;
  float all[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float ty[kMaxTypeFast][8];
#pragma unroll
  for (int k = 0; k < kMaxTypeFast; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) ty[k][i] = 0.f;
  // packed bins (pos32): the rows with position s are scattered -- walk every token, block-uniform test
  const int nrows = pos32 != nullptr ? batch * seq : batch;
  for (int b = 0; b < nrows; ++b) {
    const size_t r = pos32 != nullptr ? (size_t)b : (size_t)b * seq + s;
    if (pos32 != nullptr && pos32[r] != s) continue;
    const int tt = tt32[r];
    const uint4 v = ldg16(dx + r * H + threadIdx.x * 8);
    const float f[8] = {bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y),
                        bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w)};
#pragma unroll
    for (int i = 0; i < 8; ++i) all[i] += f[i];
#pragma unroll
    for (int k = 0; k < kMaxTypeFast; ++k)
      if (tt == k) {
#pragma unroll
        for (int i = 0; i < 8; ++i) ty[k][i] += f[i];
      }
  }
  uint4 o;
  o.x = pack_bf16(all[0], all[1]); o.y = pack_bf16(all[2], all[3]);
  o.z = pack_bf16(all[4], all[5]); o.w = pack_bf16(all[6], all[7]);
  stg16(d_pos + (size_t)s * H + threadIdx.x * 8, o);
#pragma unroll
  for (int k = 0; k < kMaxTypeFast; ++k)
    if (k < T) {
      float* dst = type_part + ((size_t)s * T + k) * H + threadIdx.x * 8;
      *reinterpret_cast<float4*>(dst) = make_float4(ty[k][0], ty[k][1], ty[k][2], ty[k][3]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(ty[k][4], ty[k][5], ty[k][6], ty[k][7]);
    }
}

__global__ void fill_int_kernel(int* p, int n, int v) {
  pdl_wait();               // PDL: predecessors complete + visible before any global access
  pdl_launch_dependents();  // let the next kernel in the stream begin launching
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

}  // namespace b2

using namespace b2;

static int32_t embed_fwd_impl(const int64_t* input_ids, const int64_t* token_type_ids, const int64_t* position_ids,
                              int64_t max_pos, int32_t* pos32, int64_t batch, int64_t seq, const void* word_emb,
                              const void* pos_emb, const void* type_emb, const void* gamma, const void* beta,
                              int64_t hidden, int64_t vocab, int64_t type_vocab, float eps, float dropout_p,
                              const void* rng_state, uint32_t rng_site, void* y, float* y_f32, void* pre_ln,
                              float* mean, float* rstd, int32_t* ids32, int32_t* tt32, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  B2_REQUIRE(input_ids && word_emb && pos_emb && type_emb && gamma && beta && y && pre_ln && mean && rstd && ids32 &&
                 tt32,
             "embed_fwd: null pointer");
  B2_REQUIRE(batch > 0 && seq > 0, "embed_fwd: empty batch (batch=%lld seq=%lld)", (long long)batch, (long long)seq);
  B2_REQUIRE(hidden % 256 == 0 && hidden >= 256 && hidden <= 1024, "embed_fwd: hidden=%lld unsupported",
             (long long)hidden);
  B2_REQUIRE(!(dropout_p > 0.f) || rng_state, "embed_fwd: dropout needs rng_state");
  const int tokens = (int)(batch * seq);
  const unsigned grid = (unsigned)((tokens + 3) / 4);
#define B2_EMB(VPL_)                                                                                              \
  case VPL_:                                                                                                      \
    B2_LAUNCH((embed_fwd_kernel<VPL_>), grid, 128, 0, stream,                                                              \
        (const long long*)input_ids, (const long long*)token_type_ids, (const long long*)position_ids,            \
        (int)max_pos, pos32, tokens, (int)seq,                                                                    \
        (const __nv_bfloat16*)word_emb, (const __nv_bfloat16*)pos_emb, (const __nv_bfloat16*)type_emb,            \
        (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta, (int)vocab, (int)type_vocab, eps, dropout_p,     \
        (const unsigned long long*)rng_state, rng_site, (__nv_bfloat16*)y, y_f32, (__nv_bfloat16*)pre_ln, mean,   \
        rstd,                                                                                                     \
        ids32, tt32);                                                                                             \
    break;
  switch ((int)(hidden / 256)) { B2_EMB(1) B2_EMB(2) B2_EMB(3) B2_EMB(4) }
#undef B2_EMB
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_embed_fwd(const int64_t* input_ids, const int64_t* token_type_ids, int64_t batch, int64_t seq,
                                const void* word_emb, const void* pos_emb, const void* type_emb, const void* gamma,
                                const void* beta, int64_t hidden, int64_t vocab, int64_t type_vocab, float eps,
                                float dropout_p, const void* rng_state, uint32_t rng_site, void* y, float* y_f32,
                                void* pre_ln, float* mean, float* rstd, int32_t* ids32, int32_t* tt32, void* stream_) {
  return embed_fwd_impl(input_ids, token_type_ids, nullptr, 0, nullptr, batch, seq, word_emb, pos_emb, type_emb, gamma,
                        beta, hidden, vocab, type_vocab, eps, dropout_p, rng_state, rng_site, y, y_f32, pre_ln, mean,
                        rstd, ids32, tt32, stream_);
}

extern "C" int32_t b2_embed_fwd_packed(const int64_t* input_ids, const int64_t* token_type_ids,
                                       const int64_t* position_ids, int64_t max_positions, int64_t bins, int64_t seq,
                                       const void* word_emb, const void* pos_emb, const void* type_emb,
                                       const void* gamma, const void* beta, int64_t hidden, int64_t vocab,
                                       int64_t type_vocab, float eps, float dropout_p, const void* rng_state,
                                       uint32_t rng_site, void* y, float* y_f32, void* pre_ln, float* mean,
                                       float* rstd, int32_t* ids32, int32_t* tt32, int32_t* pos32, void* stream_) {
  B2_REQUIRE(position_ids && pos32 && max_positions > 0, "embed_fwd_packed: position ids / pos32 / max_positions");
  return embed_fwd_impl(input_ids, token_type_ids, position_ids, max_positions, pos32, bins, seq, word_emb, pos_emb,
                        type_emb, gamma, beta, hidden, vocab, type_vocab, eps, dropout_p, rng_state, rng_site, y,
                        y_f32, pre_ln, mean, rstd, ids32, tt32, stream_);
}

static int32_t embed_bwd_impl(const void* dy, int32_t dy_fp32, const void* pre_ln, const float* mean,
                                const float* rstd,
                                const void* gamma, const int32_t* ids32, const int32_t* tt32, const int32_t* pos32,
                                int64_t batch,
                                int64_t seq, int64_t hidden, int64_t vocab, int64_t type_vocab, int64_t pad_token_id,
                                float dropout_p, const void* rng_state, uint32_t rng_site, void* d_word, void* d_pos,
                                void* d_type,
                                void* d_gamma, void* d_beta, void* scratch_dx, float* scratch_partials,
                                int64_t scratch_partials_bytes, int32_t* owner, void* stream_,
                                bool ordered = false) {
  cudaStream_t stream = (cudaStream_t)stream_;
  B2_REQUIRE(dy && pre_ln && mean && rstd && gamma && ids32 && tt32 && d_word && d_pos && d_type && d_gamma &&
                 d_beta && scratch_dx && scratch_partials && owner,
             "embed_bwd: null pointer");
  B2_REQUIRE(batch > 0 && seq > 0, "embed_bwd: empty batch");
  B2_REQUIRE(hidden % 256 == 0 && hidden <= 1024, "embed_bwd: hidden=%lld unsupported", (long long)hidden);
  const int tokens = (int)(batch * seq);
  // 1. LayerNorm backward (dropout sits on the LN output here -> mode 1); dx lands in scratch_dx
  int32_t st = launch_layernorm_bwd(dy, nullptr, pre_ln, mean, rstd, gamma, tokens, hidden, dropout_p, rng_state,
                                    rng_site, 1, dy_fp32 ? 1 : 0, 0, scratch_dx, nullptr, d_gamma, d_beta, nullptr,
                                    scratch_partials, scratch_partials_bytes, stream);
  if (st) return st;
  // 2. word rows (d_word pre-zeroed by the caller)
  B2_LAUNCH(embed_owner_kernel, (tokens + 255) / 256, 256, 0, stream, ids32, tokens, (int)pad_token_id, owner);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  // fast path: fp32 owner-row accumulation + fused position/type pass (needs scratch for [tokens + seq*T][H] fp32);
  // ordered: the in-order owner scan for the word rows + the same position/type pass (scratch for [seq*T][H] fp32)
  const int64_t acc_rows = ordered ? 0 : (int64_t)tokens;
  const int64_t fast_bytes = 4 * hidden * (acc_rows + seq * type_vocab);
  if (type_vocab <= kMaxTypeFast && scratch_partials_bytes >= fast_bytes) {
    float* acc = scratch_partials;
    float* type_part = scratch_partials + (size_t)acc_rows * hidden;
    if (ordered) {
      B2_LAUNCH(embed_word_scatter_kernel, tokens, 128, 0, stream, (const __nv_bfloat16*)scratch_dx, ids32, tokens,
                (int)hidden, (int)pad_token_id, owner, (__nv_bfloat16*)d_word);
      B2_CUDA(cudaGetLastError());
      count_launches(1);
    } else {
      B2_CUDA(cudaMemsetAsync(acc, 0, (size_t)tokens * hidden * 4, stream));
      B2_LAUNCH(embed_word_accum_kernel, tokens, (unsigned)(hidden / 8), 0, stream, (const __nv_bfloat16*)scratch_dx,
                ids32, (int)hidden, (int)pad_token_id, owner, acc);
      B2_CUDA(cudaGetLastError());
      count_launches(1);
      B2_LAUNCH(embed_word_finish_kernel, tokens, (unsigned)(hidden / 8), 0, stream, acc, ids32, (int)hidden,
                (int)pad_token_id, owner, (__nv_bfloat16*)d_word);
      B2_CUDA(cudaGetLastError());
      count_launches(1);
    }
    B2_LAUNCH(embed_pos_type_kernel, (unsigned)seq, (unsigned)(hidden / 8), 0, stream, (const __nv_bfloat16*)scratch_dx,
              tt32, pos32, (int)batch, (int)seq, (int)hidden, (int)type_vocab, (__nv_bfloat16*)d_pos, type_part);
    B2_CUDA(cudaGetLastError());
    count_launches(1);
    __nv_bfloat16* dt = (__nv_bfloat16*)d_type;
    return b2_colsum_finish(type_part, (int32_t)seq, (int32_t)type_vocab, hidden, dt,
                            type_vocab > 1 ? dt + hidden : nullptr, type_vocab > 2 ? dt + 2 * hidden : nullptr, stream_);
  }
  B2_REQUIRE(pos32 == nullptr, "embed_bwd_packed: scratch too small for the packed path (%lld bytes needed)",
             (long long)fast_bytes);
  B2_LAUNCH(embed_word_scatter_kernel, tokens, 128, 0, stream, (const __nv_bfloat16*)scratch_dx, ids32, tokens, (int)hidden,
                                                        (int)pad_token_id, owner, (__nv_bfloat16*)d_word);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  // 3. position rows: the table has `max_pos` rows but only the first `seq` receive gradient; the caller passes
  //    d_pos sized [seq rows used]; rows beyond are zeroed by the caller's bucket memset
  B2_LAUNCH(embed_pos_kernel, (unsigned)seq, (unsigned)(hidden / 8), 0, stream, (const __nv_bfloat16*)scratch_dx, (int)batch,
                                                                         (int)seq, (int)hidden, (__nv_bfloat16*)d_pos);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  // 4. token-type rows
  for (int ty = 0; ty < (int)type_vocab; ++ty) {
    st = launch_colsum(scratch_dx, tokens, hidden, hidden, tt32, ty, (__nv_bfloat16*)d_type + (size_t)ty * hidden,
                       scratch_partials, scratch_partials_bytes, stream);
    if (st) return st;
  }
  return 0;
}

extern "C" int32_t b2_embed_bwd(const void* dy, int32_t dy_fp32, const void* pre_ln, const float* mean,
                                const float* rstd, const void* gamma, const int32_t* ids32, const int32_t* tt32,
                                int64_t batch, int64_t seq, int64_t hidden, int64_t vocab, int64_t type_vocab,
                                int64_t pad_token_id, float dropout_p, const void* rng_state, uint32_t rng_site,
                                void* d_word, void* d_pos, void* d_type, void* d_gamma, void* d_beta, void* scratch_dx,
                                float* scratch_partials, int64_t scratch_partials_bytes, int32_t* owner,
                                void* stream_) {
  return embed_bwd_impl(dy, dy_fp32, pre_ln, mean, rstd, gamma, ids32, tt32, nullptr, batch, seq, hidden, vocab,
                        type_vocab, pad_token_id, dropout_p, rng_state, rng_site, d_word, d_pos, d_type, d_gamma,
                        d_beta, scratch_dx, scratch_partials, scratch_partials_bytes, owner, stream_);
}

extern "C" int32_t b2_embed_bwd_packed(const void* dy, int32_t dy_fp32, const void* pre_ln, const float* mean,
                                       const float* rstd, const void* gamma, const int32_t* ids32,
                                       const int32_t* tt32, const int32_t* pos32, int64_t bins, int64_t seq,
                                       int64_t hidden, int64_t vocab, int64_t type_vocab, int64_t pad_token_id,
                                       float dropout_p, const void* rng_state, uint32_t rng_site, void* d_word,
                                       void* d_pos, void* d_type, void* d_gamma, void* d_beta, void* scratch_dx,
                                       float* scratch_partials, int64_t scratch_partials_bytes, int32_t* owner,
                                       void* stream_) {
  B2_REQUIRE(pos32 != nullptr, "embed_bwd_packed: null pos32");
  return embed_bwd_impl(dy, dy_fp32, pre_ln, mean, rstd, gamma, ids32, tt32, pos32, bins, seq, hidden, vocab,
                        type_vocab, pad_token_id, dropout_p, rng_state, rng_site, d_word, d_pos, d_type, d_gamma,
                        d_beta, scratch_dx, scratch_partials, scratch_partials_bytes, owner, stream_);
}

// The ordered forms: word rows always by the in-order owner scan (embed_word_scatter_kernel), never by the fp32
// owner-row reductions, so a row's duplicates are summed in token order and the result is the same on every run.
extern "C" int32_t b2_embed_bwd_ordered(const void* dy, int32_t dy_fp32, const void* pre_ln, const float* mean,
                                        const float* rstd, const void* gamma, const int32_t* ids32, const int32_t* tt32,
                                        int64_t batch, int64_t seq, int64_t hidden, int64_t vocab, int64_t type_vocab,
                                        int64_t pad_token_id, float dropout_p, const void* rng_state, uint32_t rng_site,
                                        void* d_word, void* d_pos, void* d_type, void* d_gamma, void* d_beta,
                                        void* scratch_dx, float* scratch_partials, int64_t scratch_partials_bytes,
                                        int32_t* owner, void* stream_) {
  return embed_bwd_impl(dy, dy_fp32, pre_ln, mean, rstd, gamma, ids32, tt32, nullptr, batch, seq, hidden, vocab,
                        type_vocab, pad_token_id, dropout_p, rng_state, rng_site, d_word, d_pos, d_type, d_gamma,
                        d_beta, scratch_dx, scratch_partials, scratch_partials_bytes, owner, stream_, true);
}

extern "C" int32_t b2_embed_bwd_packed_ordered(const void* dy, int32_t dy_fp32, const void* pre_ln, const float* mean,
                                               const float* rstd, const void* gamma, const int32_t* ids32,
                                               const int32_t* tt32, const int32_t* pos32, int64_t bins, int64_t seq,
                                               int64_t hidden, int64_t vocab, int64_t type_vocab, int64_t pad_token_id,
                                               float dropout_p, const void* rng_state, uint32_t rng_site, void* d_word,
                                               void* d_pos, void* d_type, void* d_gamma, void* d_beta, void* scratch_dx,
                                               float* scratch_partials, int64_t scratch_partials_bytes, int32_t* owner,
                                               void* stream_) {
  B2_REQUIRE(pos32 != nullptr, "embed_bwd_packed_ordered: null pos32");
  return embed_bwd_impl(dy, dy_fp32, pre_ln, mean, rstd, gamma, ids32, tt32, pos32, bins, seq, hidden, vocab,
                        type_vocab, pad_token_id, dropout_p, rng_state, rng_site, d_word, d_pos, d_type, d_gamma,
                        d_beta, scratch_dx, scratch_partials, scratch_partials_bytes, owner, stream_, true);
}

// arms the owner table (INT_MAX) once; the scatter kernel re-arms what it touched
extern "C" int32_t b2_embed_owner_init(int32_t* owner, int64_t vocab, void* stream_) {
  B2_REQUIRE(owner && vocab > 0, "embed_owner_init: bad args");
  B2_LAUNCH(fill_int_kernel, (unsigned)((vocab + 255) / 256), 256, 0, (cudaStream_t)stream_, owner, (int)vocab, INT_MAX);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}
