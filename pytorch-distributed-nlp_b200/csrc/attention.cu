// Fused multi-head self-attention, forward and backward, on Hopper tensor cores (wgmma; head_dim 64, seq % 128 == 0).
//
// Replaces the eager attention of BertSelfAttention (SP/transformers/models/bert/modeling_bert.py:115-140:
// matmul -> *scale -> +mask -> softmax -> dropout -> matmul, and the transpose/contiguous head merge at :138,:206)
// plus its autograd backward (SURVEY.md K3-K6).  The [B,12,S,S] probability tensor never exists in HBM: the
// backward recomputes it from Q, K and the saved log-sum-exp.
//
// One CTA = 256 threads = two warpgroups = 128 query (fwd) or key (bwd) rows: warpgroup g computes rows
// [64 g, 64 g + 64) of every product with wgmma m64nNk16, accumulators in registers.  In the accumulator layout a
// row's columns are spread over the four lanes of a quad (lane / 4 picks the row, lane % 4 the column pair in each
// 8-column group), so row maxima and sums take two quad shuffles, and each lane draws the dropout decisions of a
// quarter of the row's 8-key groups and shares them within the quad.  Tiles move HBM->smem by TMA straight out of
// the packed [tokens, 3*hidden] QKV activation (128B swizzle); the same smem tile serves as a K-major operand for
// one product and as an MN-major operand for another (e.g. dO is A of dP = dO V^T and B of dV = P^T dO), so nothing
// is ever transposed in memory.  Results leave the same way: the context tile, dQ, dK and dV are written into
// operand tiles the last products have released and stored with TMA.  Kernels: attention_fwd128_kernel (seq 128),
// attention_fwd_kernel (any seq <= 512, online softmax), attention_bwd128_kernel (seq 128), attention_bwd_kernel.
// The seq-128 backward is persistent: a CTA walks (batch, head) items and loads the next item's tiles under this
// one's compute.  Each kernel has a packed-bin form (kSeg) that masks with per-row segments; the long forms visit
// only the 128-key (fwd) or 128-query (bwd) blocks that some row of the CTA's block can see.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

constexpr int ATT_THREADS = 256;
constexpr int TILE_BYTES = 128 * 64 * 2;  // one [128 x 64] bf16 tile = 16 KB
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr float kMaskBias = -3.4028234663852886e38f;  // torch.finfo(float32).min, what HF adds for masked keys

// Byte offset of element (row, col) in a [128 rows x 64 cols] bf16 tile of 128-byte swizzled rows (the TMA layout).
__device__ __forceinline__ uint32_t sw_off(int row, int col) {
  return row * 128 + ((((col >> 3) ^ (row & 7))) << 4) + (col & 7) * 2;
}
// two adjacent bf16 (col even) of a [128 x 128] tile kept as two 64-column sub-tiles `lo`, `hi`
__device__ __forceinline__ void st_pair(uint8_t* lo, uint8_t* hi, int row, int col, float a, float b) {
  *reinterpret_cast<uint32_t*>((col < 64 ? lo : hi) + sw_off(row, col & 63)) = pack_bf16(a, b);
}

struct AttnParams {
  int batch, seq, heads, hidden;  // hidden = heads * 64
  float scale;                    // 1/sqrt(64)
  float neg_log2_seq;             // -log2(seq): backward exponent of a row with no visible key (row_masked_x)
  float dropout_p; const unsigned long long* rng; unsigned rng_site;
  const long long* mask;          // [batch, seq] or null
  __nv_bfloat16* ctx;             // fwd out [tokens, hidden]
  float* lse;                     // [batch, heads, seq] natural log
  // backward
  const __nv_bfloat16* ctx_in; const __nv_bfloat16* d_ctx;
  __nv_bfloat16* d_qkv; float* dq_accum;
  float* dbias;                   // optional fp32 [3*hidden]: += column sums of d_qkv (QKV bias gradient)
  // optional (seq == 128, dropout on): the forward's dropout decisions, one 64-bit word per (b, h, query row, key
  // half) -- written by the forward, read by the backward instead of regenerating Philox
  unsigned long long* keep_bits;
  // optional: packed bins -- row r of bin b may attend to keys [lo, hi) of the same bin only,
  // seg[b * seq + r] = lo | hi << 16 (pytorch-distributed-nlp_b200/packing.py); replaces the key-padding mask.  The
  // segments of a bin are contiguous and every row lies in its own (lo <= r < hi), which the long kernels' block
  // skipping relies on.
  const int* seg;
};

// Fragment coordinates of this thread in a warpgroup-wide m64 accumulator (see wgmma.cuh): rows r and r + 8 of the
// CTA's 128, column pair 2 t (+1) of every 8-column group.
struct Frag {
  int r, t;
  __device__ __forceinline__ Frag(int warp, int lane)
      : r((warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2)), t(lane & 3) {}
  // accumulator index i of an n-wide product -> row (0: r, 1: r + 8) and column
  __device__ __forceinline__ static int hi(int i) { return (i >> 1) & 1; }
  __device__ __forceinline__ int col(int i) const { return 8 * (i >> 2) + 2 * t + (i & 1); }
};

// Dropout decisions of the 16 eight-key groups of one 128-key row whose key 0 has Philox element index `base`:
// lane t of the quad draws groups t, t + 4, t + 8, t + 12; after the exchange keep[j] holds group j's 8 bits.
__device__ __forceinline__ void quad_keep16(const DropCtx& d, unsigned long long base, int lane, uint32_t (&keep)[16]) {
  uint32_t own[4];
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) own[jj] = dropout_keep8(d, base + 8ull * (4 * jj + (lane & 3)));
#pragma unroll
  for (int j = 0; j < 16; ++j) keep[j] = __shfl_sync(0xffffffffu, own[j >> 2], (lane & ~3) | (j & 3));
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// is key `col` (0..127 within the block) masked for a row: packed bins compare against the row's own [lo, hi); the
// key-padding mask is one bit per key (mw: the block's four 32-key words)
template <bool kSeg>
__device__ __forceinline__ bool key_masked(const uint32_t (&mw)[4], int seg_word, int col) {
  if (kSeg) return col < (seg_word & 0xffff) || col >= (seg_word >> 16);
  return (mw[col >> 5] >> (col & 31)) & 1u;
}
// a row's segment word lo | hi << 16 (bin coordinates) relative to the 128-key block that starts at key k0, both ends
// clamped to [0, 128]: key_masked<true> then tests the block's columns 0..127
__device__ __forceinline__ int seg_in_block(int seg_word, int k0) {
  const int lo = min(max((seg_word & 0xffff) - k0, 0), 128), hi = min(max((seg_word >> 16) - k0, 0), 128);
  return lo | hi << 16;
}
// Backward: the log2-domain exponent of a masked key of a query row whose log2 LSE is lse2.  A row with no visible key
// (an all-zero attention_mask row) has all scores equal to finfo.min in HF, so its softmax is uniform.  The forward
// gets that right (m = kMaskBias, every p = 1, l = seq) and stores lse = (kMaskBias + log2 seq) ln2, in which log2 seq
// is lost to rounding: exp2(kMaskBias - lse2) would be 0, not 1/seq.  Such an lse2 (~kMaskBias) is far below that of
// any row with a visible key (>= its largest finite score), so the row is recognised here and every key gets
// P = 1/seq.  One select per row, nothing in the per-key loop.
__device__ __forceinline__ float row_masked_x(float lse2, float neg_log2_seq) {
  return lse2 < 0.5f * kMaskBias ? neg_log2_seq : kMaskBias - lse2;
}
// Column sums over the 128 rows of an m64n64 accumulator pair (one warpgroup per 64 rows), added into out[0, 64)
__device__ __forceinline__ void frag_colsum64(const float (&f)[32], int lane, float* out) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float v = f[4 * j + e] + f[4 * j + 2 + e];
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (lane < 4) atomicAdd(out + 8 * j + 2 * lane + e, v);
    }
  }
}
// S[128 x 128] (+)= A[128 x 64] B[128 x 64]^T, both K-major tiles (Q K^T, dO V^T): warpgroup wg's 64 rows
__device__ __forceinline__ void mma_nt_128(float (&s)[64], const uint8_t* a, const uint8_t* b, int wg) {
  const uint32_t aa = smem_u32(a) + wg * 8192, ab = smem_u32(b);
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_bf16<128, 0, 0>(s, make_smem_desc(aa + k * 32, 16, 1024), make_smem_desc(ab + k * 32, 16, 1024),
                          k > 0 ? 1u : 0u);
}
// O[128 x 64] = P[128 x 128] V[128 x 64]: P K-major in two 64-key sub-tiles, V MN-major (rows = keys)
__device__ __forceinline__ void mma_pv(float (&o)[32], const uint8_t* p_lo, const uint8_t* p_hi, const uint8_t* v,
                                       int wg) {
  const uint32_t a0 = smem_u32(p_lo) + wg * 8192, a1 = smem_u32(p_hi) + wg * 8192, av = smem_u32(v);
#pragma unroll
  for (int k = 0; k < 8; ++k)
    wgmma_bf16<64, 0, 1>(o, make_smem_desc((k < 4 ? a0 : a1) + (k & 3) * 32, 16, 1024),
                         make_smem_desc(av + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
}

// ------------------------------------------------------------------------------------------------------------
// forward: grid (seq/128, heads, batch)
// ------------------------------------------------------------------------------------------------------------
// kSeg: packed bins.  The CTA's 128 query rows see keys in [min lo, max hi) of their segments only, so it visits just
// the key blocks that range meets.  A skipped block would add exactly 0 (every key masked: p = exp2(kMaskBias - m) =
// 0, alpha = 1), and a visited block before a row's first visible key is cancelled exactly by the next block's
// alpha = exp2(kMaskBias - m) = 0, so per sequence the arithmetic is that of the padded kernel.
template <bool kSeg>
__global__ void __launch_bounds__(ATT_THREADS, 1) attention_fwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                                                                      const __grid_constant__ CUtensorMap tmap_ctx,
                                                                      const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sK = smem + TILE_BYTES;
  uint8_t* sV = smem + 2 * TILE_BYTES;
  uint8_t* sP = smem + 3 * TILE_BYTES;  // 2 tiles
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(smem + 5 * TILE_BYTES);
  // [seq / 32 <= 16] masked-key bits; kSeg: [0, 4) each warp's smallest lo, [4, 8) its largest hi
  uint32_t* s_mbits = reinterpret_cast<uint32_t*>(smem + 5 * TILE_BYTES + 64);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const Frag fr(warp, lane);
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nkv = p.seq / 128;

  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_ctx);
    mbar_init(bar_load, 1);
    fence_mbar_init();
  }
  pdl_wait();               // PDL: setup above overlapped the predecessor's tail; global reads start below
  pdl_launch_dependents();
  int seg[2] = {0, 0};      // kSeg: this thread's two rows' segment words
  if (kSeg) {
    seg[0] = p.seg[(size_t)b * p.seq + qb * 128 + fr.r];
    seg[1] = p.seg[(size_t)b * p.seq + qb * 128 + fr.r + 8];
    if (tid < 128) {
      const int w = p.seg[(size_t)b * p.seq + qb * 128 + tid];
      const unsigned lo = __reduce_min_sync(0xffffffffu, (unsigned)(w & 0xffff));
      const unsigned hi = __reduce_max_sync(0xffffffffu, (unsigned)w >> 16);
      if (lane == 0) {
        s_mbits[warp] = lo;
        s_mbits[4 + warp] = hi;
      }
    }
  } else {
    for (int c = tid; c < p.seq; c += ATT_THREADS) {   // seq % 128 == 0: whole warps take part in every round
      const bool masked = p.mask != nullptr && p.mask[(size_t)b * p.seq + c] == 0;
      const unsigned bits = __ballot_sync(0xffffffffu, masked);
      if (lane == 0) s_mbits[c >> 5] = bits;
    }
  }
  __syncthreads();
  int j0 = 0, j1 = nkv;     // the key blocks this CTA visits
  if (kSeg) {
    const unsigned lo = min(min(s_mbits[0], s_mbits[1]), min(s_mbits[2], s_mbits[3]));
    const unsigned hi = max(max(s_mbits[4], s_mbits[5]), max(s_mbits[6], s_mbits[7]));
    // kept inside the bin and around the block's own keys (which every valid segment of its rows contains), so that
    // malformed segments cannot take the loads past the bin or leave the loop empty
    j0 = min((int)(lo >> 7), qb);
    j1 = min(max((int)((hi + 127) >> 7), qb + 1), nkv);
  }

  const int row0 = b * p.seq;           // first token row of this sequence
  const int col_q = h * 64, col_k = p.hidden + h * 64, col_v = 2 * p.hidden + h * 64;
  const DropCtx drop = make_drop_ctx(p.rng, p.rng_site, p.dropout_p);
  const float c2 = p.scale * kLog2e;

  float o_acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o_acc[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: this lane's share of the row sum
  uint32_t ph_load = 0;

  for (int j = j0; j < j1; ++j) {
    if (tid == 0) {
      mbar_expect_tx(bar_load, (j == j0 ? 3 : 2) * TILE_BYTES);
      if (j == j0) tma_load_2d(sQ, &tmap_qkv, bar_load, col_q, row0 + qb * 128);
      tma_load_2d(sK, &tmap_qkv, bar_load, col_k, row0 + j * 128);
      tma_load_2d(sV, &tmap_qkv, bar_load, col_v, row0 + j * 128);
    }
    mbar_wait(bar_load, ph_load);
    ph_load ^= 1;
    float s[64];
    wgmma_fence();
    mma_nt_128(s, sQ, sK, wg);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    const uint32_t mw[4] = {s_mbits[j * 4], s_mbits[j * 4 + 1], s_mbits[j * 4 + 2], s_mbits[j * 4 + 3]};
    const int sw[2] = {kSeg ? seg_in_block(seg[0], j * 128) : 0, kSeg ? seg_in_block(seg[1], j * 128) : 0};
    // maximum of the row's scaled + masked scores (log2 domain); a masked key counts as score*c2 + (-3.4e38),
    // which is -3.4e38 in fp32
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 64; ++i)
      if (!key_masked<kSeg>(mw, sw[Frag::hi(i)], fr.col(i))) mx[Frag::hi(i)] = fmaxf(mx[Frag::hi(i)], s[i]);
    float m_new[2], alpha[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const float mb = fmaxf(quad_max(mx[u]) * c2, kMaskBias);   // scale after the max (c2 > 0)
      m_new[u] = fmaxf(m_run[u], mb);
      alpha[u] = exp2f(m_run[u] - m_new[u]);                      // first block: exp2(-inf) = 0
    }
    // probabilities -> (dropout) -> bf16 P tile in smem
    uint32_t keep[2][16];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int q_row = qb * 128 + fr.r + 8 * u;
      quad_keep16(drop, (((unsigned long long)(b * p.heads + h) * p.seq + q_row) * p.seq) + j * 128, lane, keep[u]);
    }
    float l_blk[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int u = Frag::hi(i), c = fr.col(i);
      float q2[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float x = fmaf(s[i + e], c2, -m_new[u]);
        if (key_masked<kSeg>(mw, sw[u], c + e)) x = kMaskBias - m_new[u];
        const float pr = ex2_approx(x);
        l_blk[u] += pr;
        q2[e] = ((keep[u][c >> 3] >> ((c + e) & 7)) & 1u) ? pr * drop.scale : 0.f;
      }
      st_pair(sP, sP + TILE_BYTES, fr.r + 8 * u, c, q2[0], q2[1]);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      l_run[u] = l_run[u] * alpha[u] + l_blk[u];
      m_run[u] = m_new[u];
    }
    fence_proxy_async_smem();
    __syncthreads();
    float ob[32];
    wgmma_fence();
    mma_pv(ob, sP, sP + TILE_BYTES, sV, wg);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(ob);
#pragma unroll
    for (int i = 0; i < 32; ++i) o_acc[i] = o_acc[i] * alpha[Frag::hi(i)] + ob[i];
    __syncthreads();   // every product of this block is complete: K, V and P may be overwritten
  }

  // the context tile leaves through Q's tile (its last reader, the final QK^T, completed) as one TMA store
  float inv_l[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const float l_tot = quad_sum(l_run[u]);
    inv_l[u] = 1.0f / l_tot;
    if (p.lse != nullptr && fr.t == 0)   // no visible key: m = kMaskBias, lse ~ kMaskBias * ln2 (see row_masked_x)
      p.lse[((size_t)b * p.heads + h) * p.seq + qb * 128 + fr.r + 8 * u] = (m_run[u] + log2f(l_tot)) * kLn2;
  }
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int u = Frag::hi(i);
    st_pair(sQ, sQ, fr.r + 8 * u, fr.col(i), o_acc[i] * inv_l[u], o_acc[i + 1] * inv_l[u]);
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    tma_store_2d(&tmap_ctx, sQ, h * 64, row0 + qb * 128);
    tma_store_commit_and_wait();
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward, seq == 128 (the benchmark shape): one key block, so no online rescale and no accumulator carried across
// iterations.  3 smem tiles (P overwrites Q and K once S = QK^T has completed, the context tile overwrites V).
// Same arithmetic, same Philox indexing as attention_fwd_kernel; also records the dropout decisions (keep_bits) for
// the backward.
// ------------------------------------------------------------------------------------------------------------
template <bool kSeg>   // kSeg: packed bins (per-row segment mask, p.seg) instead of the key-padding mask
__global__ void __launch_bounds__(ATT_THREADS, 2) attention_fwd128_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                                                                         const __grid_constant__ CUtensorMap tmap_ctx,
                                                                         const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  uint8_t* sQ = smem;                      // later: keys 0-63 of P
  uint8_t* sK = smem + TILE_BYTES;         // later: keys 64-127 of P
  uint8_t* sV = smem + 2 * TILE_BYTES;     // later: the context tile on its way out
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(smem + 3 * TILE_BYTES);
  uint32_t* s_mbits = reinterpret_cast<uint32_t*>(smem + 3 * TILE_BYTES + 48);   // [4]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const Frag fr(warp, lane);
  const int h = blockIdx.y, b = blockIdx.z;

  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_ctx);
    mbar_init(bar_load, 1);
    fence_mbar_init();
  }
  pdl_wait();               // PDL: setup above overlapped the predecessor's tail; global reads start below
  pdl_launch_dependents();
  if (tid < 128) {
    const bool masked = p.mask != nullptr && p.mask[(size_t)b * 128 + tid] == 0;
    const unsigned bits = __ballot_sync(0xffffffffu, masked);
    if (lane == 0) s_mbits[warp] = bits;
  }
  __syncthreads();
  const int row0 = b * 128;
  const int col_q = h * 64, col_k = p.hidden + h * 64, col_v = 2 * p.hidden + h * 64;
  if (tid == 0) {
    mbar_expect_tx(bar_load, 3 * TILE_BYTES);
    tma_load_2d(sQ, &tmap_qkv, bar_load, col_q, row0);
    tma_load_2d(sK, &tmap_qkv, bar_load, col_k, row0);
    tma_load_2d(sV, &tmap_qkv, bar_load, col_v, row0);
  }
  const DropCtx drop = make_drop_ctx(p.rng, p.rng_site, p.dropout_p);
  const float c2 = p.scale * kLog2e;
  const uint32_t mw[4] = {s_mbits[0], s_mbits[1], s_mbits[2], s_mbits[3]};
  int seg[2] = {0, 0};
  if (kSeg) {                            // packed bins: the keys of this row's own sequence only
    seg[0] = p.seg[(size_t)b * 128 + fr.r];
    seg[1] = p.seg[(size_t)b * 128 + fr.r + 8];
  }
  // the dropout decisions do not depend on the scores: drawn while the operands are in flight
  uint32_t keep[2][16];
#pragma unroll
  for (int u = 0; u < 2; ++u)
    quad_keep16(drop, ((unsigned long long)(b * p.heads + h) * 128 + fr.r + 8 * u) * 128, lane, keep[u]);

  mbar_wait(bar_load, 0);
  float s[64];
  wgmma_fence();
  mma_nt_128(s, sQ, sK, wg);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(s);

  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 64; ++i)
    if (!key_masked<kSeg>(mw, seg[Frag::hi(i)], fr.col(i))) mx[Frag::hi(i)] = fmaxf(mx[Frag::hi(i)], s[i]);
  float m_new[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) m_new[u] = fmaxf(quad_max(mx[u]) * c2, kMaskBias);   // see attention_fwd_kernel
  __syncthreads();   // both warpgroups' products have read Q and K: P may overwrite them

  float l_loc[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    const int u = Frag::hi(i), c = fr.col(i);
    float q2[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float x = fmaf(s[i + e], c2, -m_new[u]);
      if (key_masked<kSeg>(mw, seg[u], c + e)) x = kMaskBias - m_new[u];
      const float pr = ex2_approx(x);
      l_loc[u] += pr;
      q2[e] = ((keep[u][c >> 3] >> ((c + e) & 7)) & 1u) ? pr * drop.scale : 0.f;
    }
    st_pair(sQ, sK, fr.r + 8 * u, c, q2[0], q2[1]);
  }
  if (p.keep_bits != nullptr && fr.t == 0) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      unsigned long long w0 = 0ull, w1 = 0ull;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        w0 |= (unsigned long long)(keep[u][j] & 0xffu) << (8 * j);
        w1 |= (unsigned long long)(keep[u][j + 8] & 0xffu) << (8 * j);
      }
      unsigned long long* kb = p.keep_bits + (((size_t)b * p.heads + h) * 128 + fr.r + 8 * u) * 2;
      kb[0] = w0;
      kb[1] = w1;
    }
  }
  fence_proxy_async_smem();
  __syncthreads();
  float o[32];
  wgmma_fence();
  mma_pv(o, sQ, sK, sV, wg);
  wgmma_commit();
  float inv_l[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const float l_tot = quad_sum(l_loc[u]);
    inv_l[u] = 1.0f / l_tot;
    if (p.lse != nullptr && fr.t == 0)   // see attention_fwd_kernel
      p.lse[((size_t)b * p.heads + h) * 128 + fr.r + 8 * u] = (m_new[u] + log2f(l_tot)) * kLn2;
  }
  wgmma_wait<0>();
  wgmma_fence_regs(o);
  __syncthreads();   // both warpgroups' products have read V: the context tile may overwrite it
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int u = Frag::hi(i);
    st_pair(sV, sV, fr.r + 8 * u, fr.col(i), o[i] * inv_l[u], o[i + 1] * inv_l[u]);
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    tma_store_2d(&tmap_ctx, sV, h * 64, row0);
    tma_store_commit_and_wait();
  }
}

// the key-padding mask of batch row b as four 32-key words (bit set: masked), in every warp
__device__ __forceinline__ void mask_words128(const long long* mask, int b, int lane, uint32_t (&mw)[4]) {
#pragma unroll
  for (int w = 0; w < 4; ++w)
    mw[w] = __ballot_sync(0xffffffffu, mask != nullptr && mask[(size_t)b * 128 + 32 * w + lane] == 0);
}
// the dropout decisions of one 128-key row (quad_keep16) as two 64-bit words, keys 0-63 and 64-127: bit c % 64 set
// when key c is kept -- the keep_bits layout
__device__ __forceinline__ void quad_keep128(const DropCtx& d, unsigned long long base, int lane,
                                             unsigned long long (&kept)[2]) {
  uint32_t keep[16];
  quad_keep16(d, base, lane, keep);
  kept[0] = kept[1] = 0ull;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    kept[0] |= (unsigned long long)(keep[j] & 0xffu) << (8 * j);
    kept[1] |= (unsigned long long)(keep[j + 8] & 0xffu) << (8 * j);
  }
}

// A thread's 32 columns of one accumulator row (Frag::col: 8 j + 2 t + e) as the bits 2 j + e of one word, so that
// the per-element loops test a bit at a constant position: frag_bit(i) is that bit for accumulator index i.
__device__ __forceinline__ constexpr int frag_bit(int i) { return 2 * (i >> 2) + (i & 1); }
template <bool kSeg>   // key_masked for this thread's columns
__device__ __forceinline__ uint32_t frag_masked_bits(const uint32_t (&mw)[4], int seg_word, int t) {
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < 32; ++i) m |= (uint32_t)key_masked<kSeg>(mw, seg_word, 8 * (i >> 1) + 2 * t + (i & 1)) << i;
  return m;
}
// keep decisions of this thread's columns, from a row's two keep_bits words
__device__ __forceinline__ uint32_t frag_keep_bits(const unsigned long long (&kept)[2], int t) {
  const unsigned long long k0 = kept[0] >> (2 * t), k1 = kept[1] >> (2 * t);
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int j = i >> 1, e = i & 1;
    m |= (uint32_t)(((j < 8 ? k0 : k1) >> (8 * (j & 7) + e)) & 1ull) << i;
  }
  return m;
}

// ------------------------------------------------------------------------------------------------------------
// backward: grid (seq/128 kv blocks, heads, batch); loops over query blocks
// ------------------------------------------------------------------------------------------------------------
//
// seq > 128 (attention_bwd128_kernel takes seq == 128).  O comes in with Q and dO (into P's second half, free until
// the dS pass) so delta = rowsum(dO * O) reads two swizzled smem rows while S and dP are being multiplied; dK / dV
// leave through the operand tiles that the last products have released, as TMA tile stores.
// kSeg: packed bins.  Segments are contiguous and symmetric, so the rows that see a key of this block are those of
// the segments of its first and last keys, [lo(first), hi(last)): only the query blocks they fall in are visited.  A
// skipped query block would add exactly 0 to dK, dV (P = 0) and to its rows' dQ.
template <bool kSeg>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_do,
                     const __grid_constant__ CUtensorMap tmap_o, const __grid_constant__ CUtensorMap tmap_dqkv,
                     const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  constexpr int kTiles = 8;
  uint8_t* sK = smem;
  uint8_t* sV = smem + TILE_BYTES;
  uint8_t* sQ = smem + 2 * TILE_BYTES;
  uint8_t* sdO = smem + 3 * TILE_BYTES;
  uint8_t* sP0 = smem + 4 * TILE_BYTES;   // keys 0-63 of P
  uint8_t* sP1 = smem + 5 * TILE_BYTES;   // keys 64-127 of P; holds O before that
  uint8_t* sdS = smem + 6 * TILE_BYTES;   // 2 tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kTiles * TILE_BYTES);
  uint64_t* bar_kv = &bars[0];
  uint64_t* bar_q = &bars[1];
  uint32_t* s_mbits = reinterpret_cast<uint32_t*>(smem + kTiles * TILE_BYTES + 48);  // [4]: masked-key bits of this block
  float* s_delta = reinterpret_cast<float*>(smem + kTiles * TILE_BYTES + 64);         // [128]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const Frag fr(warp, lane);
  const int jb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nq = p.seq / 128;

  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    tma_prefetch_desc(&tmap_o);
    tma_prefetch_desc(&tmap_dqkv);
    mbar_init(bar_kv, 1);
    mbar_init(bar_q, 1);
    fence_mbar_init();
  }
  pdl_wait();               // PDL: setup above overlapped the predecessor's tail; global reads start below
  pdl_launch_dependents();
  if (!kSeg && tid < 128) {
    const bool masked = p.mask != nullptr && p.mask[(size_t)b * p.seq + jb * 128 + tid] == 0;
    const unsigned bits = __ballot_sync(0xffffffffu, masked);
    if (lane == 0) s_mbits[warp] = bits;
  }
  __syncthreads();
  const uint32_t mw[4] = {s_mbits[0], s_mbits[1], s_mbits[2], s_mbits[3]};
  int i0 = 0, i1 = nq;      // the query blocks this CTA visits
  if (kSeg) {
    const int* sg = p.seg + (size_t)b * p.seq + jb * 128;
    // kept inside the bin and around the block's own rows (which every valid segment of its keys contains), so that
    // malformed segments cannot take the lse / segment reads and dQ atomics past the bin, or skip the K / V wait
    i0 = min((int)(((unsigned)sg[0] & 0xffffu) >> 7), jb);
    i1 = min(max((int)((((unsigned)sg[127] >> 16) + 127) >> 7), jb + 1), nq);
  }

  const int row0 = b * p.seq;
  const int col_q = h * 64, col_k = p.hidden + h * 64, col_v = 2 * p.hidden + h * 64;
  const DropCtx drop0 = make_drop_ctx(p.rng, p.rng_site, p.dropout_p);
  const float c2 = p.scale * kLog2e;
  const size_t bh = (size_t)b * p.heads + h;

  if (tid == 0) {
    mbar_expect_tx(bar_kv, 2 * TILE_BYTES);
    tma_load_2d(sK, &tmap_qkv, bar_kv, col_k, row0 + jb * 128);
    tma_load_2d(sV, &tmap_qkv, bar_kv, col_v, row0 + jb * 128);
  }
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  uint32_t ph_q = 0;

  for (int i = i0; i < i1; ++i) {
    // kSeg: read per query block, so that the Philox key does not hold registers through the products
    const DropCtx drop = kSeg ? make_drop_ctx(p.rng, p.rng_site, p.dropout_p) : drop0;
    if (tid == 0) {
      mbar_expect_tx(bar_q, 3 * TILE_BYTES);
      tma_load_2d(sQ, &tmap_qkv, bar_q, col_q, row0 + i * 128);
      tma_load_2d(sdO, &tmap_do, bar_q, h * 64, row0 + i * 128);
      tma_load_2d(sP1, &tmap_o, bar_q, h * 64, row0 + i * 128);   // O, consumed by the delta pass below
    }
    if (i == i0) mbar_wait(bar_kv, 0);
    mbar_wait(bar_q, ph_q);
    ph_q ^= 1;
    float s[64], dp[64];
    wgmma_fence();
    mma_nt_128(s, sQ, sK, wg);
    mma_nt_128(dp, sdO, sV, wg);
    wgmma_commit();
    // delta = rowsum(dO * O) from the two smem tiles while the products run
    if (tid < 128) {
      float delta = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int off = tid * 128 + ((c ^ (tid & 7)) << 4);
        const uint4 a = *reinterpret_cast<const uint4*>(sP1 + off);
        const uint4 g = *reinterpret_cast<const uint4*>(sdO + off);
        delta += bf16_lo(a.x) * bf16_lo(g.x) + bf16_hi(a.x) * bf16_hi(g.x) + bf16_lo(a.y) * bf16_lo(g.y) +
                 bf16_hi(a.y) * bf16_hi(g.y) + bf16_lo(a.z) * bf16_lo(g.z) + bf16_hi(a.z) * bf16_hi(g.z) +
                 bf16_lo(a.w) * bf16_lo(g.w) + bf16_hi(a.w) * bf16_hi(g.w);
      }
      s_delta[tid] = delta;
    }
    float lse2[2], xm[2], delta[2];
    uint32_t keep[2][16];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int q_row = i * 128 + fr.r + 8 * u;   // this thread's query rows in the sequence
      lse2[u] = p.lse[bh * p.seq + q_row] * kLog2e;
      if (!kSeg) quad_keep16(drop, ((bh * p.seq + q_row) * p.seq) + jb * 128, lane, keep[u]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    __syncthreads();   // delta is in; O has been read and every product has read V: P may overwrite both
    if (kSeg) {
      // keys outside the row's segment: score -inf, so P = ex2(-inf) = 0 -- what the masked exponent gives every
      // row with a visible key (each packed row sees itself).  The mask is a pass of its own, and the dropout
      // decisions are drawn after it rather than under the products: testing the segment inside the loop below, or
      // holding keep through the products next to the segment words, spills.
      const int sw[2] = {seg_in_block(p.seg[(size_t)row0 + i * 128 + fr.r], jb * 128),
                         seg_in_block(p.seg[(size_t)row0 + i * 128 + fr.r + 8], jb * 128)};
#pragma unroll
      for (int ii = 0; ii < 64; ++ii)
        if (key_masked<true>(mw, sw[Frag::hi(ii)], fr.col(ii))) s[ii] = -INFINITY;
#pragma unroll
      for (int u = 0; u < 2; ++u)
        quad_keep16(drop, ((bh * p.seq + i * 128 + fr.r + 8 * u) * p.seq) + jb * 128, lane, keep[u]);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      delta[u] = s_delta[fr.r + 8 * u];
      xm[u] = row_masked_x(lse2[u], p.neg_log2_seq);
    }
#pragma unroll
    for (int ii = 0; ii < 64; ii += 2) {
      const int u = Frag::hi(ii), c = fr.col(ii);
      float pd[2], ds[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int cc = c + e;
        float x = fmaf(s[ii + e], c2, -lse2[u]);
        if (!kSeg && key_masked<false>(mw, 0, cc)) x = xm[u];   // what score*c2 + (-3.4e38) rounds to (row_masked_x)
        const float pr = ex2_approx(x);
        const bool kp = (keep[u][cc >> 3] >> (cc & 7)) & 1u;
        pd[e] = kp ? pr * drop.scale : 0.f;
        const float dpv = kp ? dp[ii + e] * drop.scale : 0.f;
        ds[e] = pr * (dpv - delta[u]) * p.scale;
      }
      st_pair(sP0, sP1, fr.r + 8 * u, c, pd[0], pd[1]);
      st_pair(sdS, sdS + TILE_BYTES, fr.r + 8 * u, c, ds[0], ds[1]);
    }
    fence_proxy_async_smem();
    __syncthreads();
    float dq[32];
    wgmma_fence();
    {
      // dV[key, d] += sum_q P[q, key] dO[q, d]      (A = P as MN-major: rows = q = K index; this warpgroup's 64 keys
      // are one sub-tile)
      const uint32_t ap = smem_u32(wg ? sP1 : sP0), ado = smem_u32(sdO);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_bf16<64, 1, 1>(dv, make_smem_desc(ap + k * 2048, 8192, 1024), make_smem_desc(ado + k * 2048, 8192, 1024),
                             (i > i0 || k > 0) ? 1u : 0u);
      // dK[key, d] += sum_q dS[q, key] Q[q, d]
      const uint32_t ads = smem_u32(sdS), aq = smem_u32(sQ), ak = smem_u32(sK);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_bf16<64, 1, 1>(dk, make_smem_desc(ads + wg * TILE_BYTES + k * 2048, 8192, 1024),
                             make_smem_desc(aq + k * 2048, 8192, 1024), (i > i0 || k > 0) ? 1u : 0u);
      // dQ[q, d] = sum_key dS[q, key] K[key, d]     (A = dS as K-major)
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_bf16<64, 0, 1>(dq, make_smem_desc(ads + (k >> 2) * TILE_BYTES + wg * 8192 + (k & 3) * 32, 16, 1024),
                             make_smem_desc(ak + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    wgmma_fence_regs(dq);
    if (p.dq_accum == nullptr) {
      // seq == 128: dQ leaves through Q's tile (once both warpgroups' dK products have read it) as a TMA store
      __syncthreads();
#pragma unroll
      for (int e = 0; e < 32; e += 2) {
        (void)pack_bf16_round(dq[e], dq[e + 1]);   // bf16-rounded values (what the GEMMs will read) for the sums
        st_pair(sQ, sQ, fr.r + 8 * Frag::hi(e), fr.col(e), dq[e], dq[e + 1]);
      }
      if (p.dbias != nullptr) frag_colsum64(dq, lane, p.dbias + col_q);
    } else {
#pragma unroll
      for (int e = 0; e < 32; ++e)
        atomicAdd(p.dq_accum + (size_t)(row0 + i * 128 + fr.r + 8 * Frag::hi(e)) * p.hidden + h * 64 + fr.col(e), dq[e]);
    }
    __syncthreads();   // the next query block reuses the tiles
  }

  // dK, dV of this block's keys -> K's and V's tiles -> TMA stores
  __syncthreads();   // every product has read K and V
#pragma unroll
  for (int e = 0; e < 32; e += 2) {
    const int r = fr.r + 8 * Frag::hi(e), c = fr.col(e);
    (void)pack_bf16_round(dk[e], dk[e + 1]);
    (void)pack_bf16_round(dv[e], dv[e + 1]);
    st_pair(sK, sK, r, c, dk[e], dk[e + 1]);
    st_pair(sV, sV, r, c, dv[e], dv[e + 1]);
  }
  if (p.dbias != nullptr) {
    frag_colsum64(dk, lane, p.dbias + col_k);
    frag_colsum64(dv, lane, p.dbias + col_v);
  }
  fence_proxy_async_smem();   // generic-proxy tile writes above -> visible to the TMA engine
  __syncthreads();
  if (tid == 0) {
    if (p.dq_accum == nullptr) tma_store_2d(&tmap_dqkv, sQ, col_q, row0 + (nq - 1) * 128);
    tma_store_2d(&tmap_dqkv, sK, col_k, row0 + jb * 128);
    tma_store_2d(&tmap_dqkv, sV, col_v, row0 + jb * 128);
    tma_store_commit_and_wait();
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward, seq == 128 (the benchmark shape): one query block and one key block per (batch, head) item.  Persistent:
// CTA c takes the items c, c + gridDim.x, ... through two operand buffers of five tiles (K, V, Q, dO, O), the next item's loaded into the
// other buffer once this item's have landed.  Within a buffer, V is dead once dP = dO V^T has completed, so the first
// 64-key half of P lives in V's tile, and the second in O's, which the delta = rowsum(dO * O) pass has read by then
// (two swizzled smem rows per query row, while S and dP are being multiplied).  dQ / dK / dV leave through the Q, K
// and V tiles once the last products have released them, as TMA tile stores that must have read the buffer out
// before it is refilled.  The dS scratch (2 tiles) is shared by the items.
// ------------------------------------------------------------------------------------------------------------
template <bool kSeg>   // kSeg: packed bins (per-row segment mask, p.seg) instead of the key-padding mask
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_bwd128_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_do,
                        const __grid_constant__ CUtensorMap tmap_o, const __grid_constant__ CUtensorMap tmap_dqkv,
                        const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);   // buffer u: tiles [5 u, 5 u + 5) = K, V, Q, dO, O
  uint8_t* sdS = smem + 10 * TILE_BYTES;       // 2 tiles
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(smem + 12 * TILE_BYTES);   // [2], one per buffer
  float* s_delta = reinterpret_cast<float*>(smem + 12 * TILE_BYTES + 64);      // [128]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const Frag fr(warp, lane);
  const int items = p.batch * p.heads;   // item = b * heads + h; the grid never exceeds it
  const int col_q = 0, col_k = p.hidden, col_v = 2 * p.hidden;   // + h * 64

  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    tma_prefetch_desc(&tmap_o);
    tma_prefetch_desc(&tmap_dqkv);
    mbar_init(&bar_load[0], 1);
    mbar_init(&bar_load[1], 1);
    fence_mbar_init();
  }
  pdl_wait();               // PDL: setup above overlapped the predecessor's tail; global reads start below
  pdl_launch_dependents();
  __syncthreads();          // barriers initialised
  // K, V, Q, dO, O of an item -> buffer u
  auto load = [&](int u, int it) {
    uint8_t* t = smem + u * 5 * TILE_BYTES;
    const int h = it % p.heads, row = (it / p.heads) * 128;
    mbar_expect_tx(&bar_load[u], 5 * TILE_BYTES);
    tma_load_2d(t, &tmap_qkv, &bar_load[u], col_k + h * 64, row);
    tma_load_2d(t + TILE_BYTES, &tmap_qkv, &bar_load[u], col_v + h * 64, row);
    tma_load_2d(t + 2 * TILE_BYTES, &tmap_qkv, &bar_load[u], col_q + h * 64, row);
    tma_load_2d(t + 3 * TILE_BYTES, &tmap_do, &bar_load[u], h * 64, row);
    tma_load_2d(t + 4 * TILE_BYTES, &tmap_o, &bar_load[u], h * 64, row);
  };
  if (tid == 0) load(0, blockIdx.x);
  const float c2 = p.scale * kLog2e;
  // the n-th item of this CTA uses buffer n % 2, whose mbarrier then completes its (n / 2)-th phase
  for (int item = blockIdx.x, n = 0; item < items; item += gridDim.x, ++n) {
    const int buf = n & 1;
    const int b = item / p.heads, h = item % p.heads;
    const size_t bh = (size_t)item;
    // read per item: the Philox key would otherwise hold registers through the products
    const DropCtx drop = make_drop_ctx(p.rng, p.rng_site, p.dropout_p);
    uint8_t* sK = smem + buf * 5 * TILE_BYTES;
    uint8_t* sV = sK + TILE_BYTES;          // later: keys 0-63 of P, then dV on its way out
    uint8_t* sQ = sK + 2 * TILE_BYTES;
    uint8_t* sdO = sK + 3 * TILE_BYTES;
    uint8_t* sO = sK + 4 * TILE_BYTES;      // later: keys 64-127 of P
    // mask, segments, log-sum-exp and dropout decisions: read while the operands are in flight
    uint32_t mw[4], masked[2], keep[2];
    mask_words128(p.mask, b, lane, mw);
    float lse2[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const size_t row = bh * 128 + fr.r + 8 * u;
      masked[u] = frag_masked_bits<kSeg>(mw, kSeg ? p.seg[(size_t)b * 128 + fr.r + 8 * u] : 0, fr.t);
      lse2[u] = p.lse[row] * kLog2e;
      unsigned long long kept[2];
      if (p.keep_bits != nullptr) {
        kept[0] = p.keep_bits[row * 2];
        kept[1] = p.keep_bits[row * 2 + 1];
      } else {
        quad_keep128(drop, row * 128, lane, kept);
      }
      keep[u] = frag_keep_bits(kept, fr.t);
    }

    mbar_wait(&bar_load[buf], (n >> 1) & 1);
    float s[64], dp[64];
    wgmma_fence();
    mma_nt_128(s, sQ, sK, wg);
    mma_nt_128(dp, sdO, sV, wg);
    wgmma_commit();
    const int next = item + gridDim.x;
    if (tid == 0 && next < items) {
      // the other buffer last held item - gridDim.x: every thread is past its products (barriers since), and its
      // dQ / dK / dV tiles must have been read out by the TMA stores before the loads overwrite them
      tma_store_wait_read();
      load(buf ^ 1, next);
    }
    // delta = rowsum(dO * O) from the two smem tiles while the products run
    if (tid < 128) {
      float delta = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int off = tid * 128 + ((c ^ (tid & 7)) << 4);
        const uint4 a = *reinterpret_cast<const uint4*>(sO + off);
        const uint4 g = *reinterpret_cast<const uint4*>(sdO + off);
        delta += bf16_lo(a.x) * bf16_lo(g.x) + bf16_hi(a.x) * bf16_hi(g.x) + bf16_lo(a.y) * bf16_lo(g.y) +
                 bf16_hi(a.y) * bf16_hi(g.y) + bf16_lo(a.z) * bf16_lo(g.z) + bf16_hi(a.z) * bf16_hi(g.z) +
                 bf16_lo(a.w) * bf16_lo(g.w) + bf16_hi(a.w) * bf16_hi(g.w);
      }
      s_delta[tid] = delta;
    }
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    __syncthreads();   // delta is in; O has been read and every product has read V: P may overwrite both
    float xm[2], delta[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      delta[u] = s_delta[fr.r + 8 * u];
      xm[u] = row_masked_x(lse2[u], p.neg_log2_seq);
    }
#pragma unroll
    for (int ii = 0; ii < 64; ii += 2) {
      const int u = Frag::hi(ii), c = fr.col(ii);
      float pd[2], ds[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float x = fmaf(s[ii + e], c2, -lse2[u]);
        if ((masked[u] >> frag_bit(ii + e)) & 1u) x = xm[u];   // what score*c2 + (-3.4e38) rounds to (row_masked_x)
        const float pr = ex2_approx(x);
        const bool kp = (keep[u] >> frag_bit(ii + e)) & 1u;
        pd[e] = kp ? pr * drop.scale : 0.f;
        const float dpv = kp ? dp[ii + e] * drop.scale : 0.f;
        ds[e] = pr * (dpv - delta[u]) * p.scale;
      }
      st_pair(sV, sO, fr.r + 8 * u, c, pd[0], pd[1]);
      st_pair(sdS, sdS + TILE_BYTES, fr.r + 8 * u, c, ds[0], ds[1]);
    }
    fence_proxy_async_smem();
    __syncthreads();
    float dv[32], dk[32], dq[32];
    wgmma_fence();
    {
      // dV[key, d] = sum_q P[q, key] dO[q, d]      (A = P as MN-major: rows = q = K index; this warpgroup's 64 keys
      // are one sub-tile)
      const uint32_t ap = smem_u32(wg ? sO : sV), ado = smem_u32(sdO);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_bf16<64, 1, 1>(dv, make_smem_desc(ap + k * 2048, 8192, 1024), make_smem_desc(ado + k * 2048, 8192, 1024),
                             k > 0 ? 1u : 0u);
      // dK[key, d] = sum_q dS[q, key] Q[q, d]
      const uint32_t ads = smem_u32(sdS), aq = smem_u32(sQ), ak = smem_u32(sK);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_bf16<64, 1, 1>(dk, make_smem_desc(ads + wg * TILE_BYTES + k * 2048, 8192, 1024),
                             make_smem_desc(aq + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
      // dQ[q, d] = sum_key dS[q, key] K[key, d]     (A = dS as K-major)
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_bf16<64, 0, 1>(dq, make_smem_desc(ads + (k >> 2) * TILE_BYTES + wg * 8192 + (k & 3) * 32, 16, 1024),
                             make_smem_desc(ak + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    wgmma_fence_regs(dq);
    __syncthreads();   // every product has read Q, K and V (P): dQ, dK, dV may overwrite them
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int r = fr.r + 8 * Frag::hi(e), c = fr.col(e);
      (void)pack_bf16_round(dq[e], dq[e + 1]);   // bf16-rounded values (what the GEMMs will read) for the sums
      (void)pack_bf16_round(dk[e], dk[e + 1]);
      (void)pack_bf16_round(dv[e], dv[e + 1]);
      st_pair(sQ, sQ, r, c, dq[e], dq[e + 1]);
      st_pair(sK, sK, r, c, dk[e], dk[e + 1]);
      st_pair(sV, sV, r, c, dv[e], dv[e + 1]);
    }
    if (p.dbias != nullptr) {
      frag_colsum64(dq, lane, p.dbias + col_q + h * 64);
      frag_colsum64(dk, lane, p.dbias + col_k + h * 64);
      frag_colsum64(dv, lane, p.dbias + col_v + h * 64);
    }
    fence_proxy_async_smem();   // generic-proxy tile writes above -> visible to the TMA engine
    __syncthreads();
    if (tid == 0) {
      tma_store_2d(&tmap_dqkv, sQ, col_q + h * 64, b * 128);
      tma_store_2d(&tmap_dqkv, sK, col_k + h * 64, b * 128);
      tma_store_2d(&tmap_dqkv, sV, col_v + h * 64, b * 128);
      tma_store_commit();
    }
  }
  if (tid == 0) tma_store_wait();
}

// fp32 dQ accumulator [tokens, hidden] -> the Q column block of d_qkv (bf16 [tokens, 3*hidden])
__global__ void dq_convert_kernel(const float* __restrict__ acc, __nv_bfloat16* __restrict__ d_qkv, long long tokens,
                                  int hidden) {
  pdl_wait();
  pdl_launch_dependents();
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= tokens * hidden) return;
  const long long t = i / hidden;
  const int c = (int)(i % hidden);
  const float4 v = *reinterpret_cast<const float4*>(acc + i);
  uint2 o;
  o.x = pack_bf16(v.x, v.y);
  o.y = pack_bf16(v.z, v.w);
  *reinterpret_cast<uint2*>(d_qkv + t * 3 * hidden + c) = o;
}

constexpr int kFwdSmem = 5 * TILE_BYTES + 128 + 1024;
constexpr int kFwd128Smem = 3 * TILE_BYTES + 64 + 1024;
constexpr int kBwdSmem = 8 * TILE_BYTES + 64 + 512 + 1024;
constexpr int kBwd128Smem = 12 * TILE_BYTES + 64 + 512 + 1024;    // two buffers of K, V, Q, dO, O + dS

// Grid of the persistent seq-128 backward: one CTA per resident slot (`per_sm` x the SM count), at most one per (batch,
// head) item.  B2_DEBUG_ATTN_CTAS=n caps it, so that tests can check that results do not depend on how the items are
// spread over the CTAs.
static int32_t persistent_grid(int per_sm, int64_t items, unsigned* grid) {
  B2_REQUIRE(per_sm > 0, "attention: the seq-128 kernel does not fit on an SM");
  B2_REQUIRE(items < (int64_t)1 << 31, "attention: batch * heads = %lld exceeds int", (long long)items);
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    B2_CUDA(cudaGetDevice(&dev));
    B2_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  int64_t n = std::min<int64_t>(items, (int64_t)per_sm * sms);
  if (const char* cap = getenv("B2_DEBUG_ATTN_CTAS")) {
    const long long c = atoll(cap);
    B2_REQUIRE(c > 0, "B2_DEBUG_ATTN_CTAS=%s: expected a positive CTA count", cap);
    n = std::min<int64_t>(n, c);
  }
  *grid = (unsigned)n;
  return 0;
}

static int32_t check_attn_shapes(const char* who, int64_t batch, int64_t seq, int64_t heads, int64_t head_dim) {
  B2_REQUIRE(batch > 0 && seq > 0 && heads > 0, "%s: empty problem (batch=%lld seq=%lld heads=%lld)", who,
             (long long)batch, (long long)seq, (long long)heads);
  B2_REQUIRE(head_dim == 64, "%s: head_dim=%lld (only 64 is on the path)", who, (long long)head_dim);
  B2_REQUIRE(seq % 128 == 0 && seq <= 512, "%s: seq=%lld must be a multiple of 128, at most 512", who,
             (long long)seq);
  B2_REQUIRE(batch <= 65535 && heads <= 65535, "%s: batch/heads exceed grid limits", who);
  return 0;
}

}  // namespace b2

using namespace b2;

static int32_t attention_fwd_impl(const void* qkv, const int64_t* attention_mask, const int32_t* segments,
                                  int64_t batch, int64_t seq, int64_t heads, int64_t head_dim, float dropout_p,
                                  const void* rng_state, uint32_t rng_site, void* ctx, float* lse,
                                  uint64_t* keep_bits, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  B2_REQUIRE(qkv && ctx, "attention_fwd: null pointer");
  int32_t st = check_attn_shapes("attention_fwd", batch, seq, heads, head_dim);
  if (st) return st;
  // also rejects NaN, which would otherwise run without dropout
  B2_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention_fwd: dropout_p out of range");
  B2_REQUIRE(!(dropout_p > 0.f) || rng_state, "attention_fwd: dropout needs rng_state");
  const int64_t hidden = heads * 64, tokens = batch * seq;
  CUtensorMap tm;
  st = get_tensor_map_2d(&tm, qkv, (uint64_t)tokens, (uint64_t)(3 * hidden), (uint64_t)(3 * hidden * 2), 128, 64);
  if (st) return st;
  AttnParams p{};
  p.batch = (int)batch; p.seq = (int)seq; p.heads = (int)heads; p.hidden = (int)hidden;
  p.scale = 0.125f;
  p.dropout_p = dropout_p; p.rng = (const unsigned long long*)rng_state; p.rng_site = rng_site;
  p.mask = (const long long*)attention_mask;
  p.seg = segments;
  p.ctx = (__nv_bfloat16*)ctx; p.lse = lse;
  // the keep-bit cache exists for the seq == 128 kernel pair only (and only when there is dropout to remember)
  p.keep_bits = (seq == 128 && dropout_p > 0.f) ? (unsigned long long*)keep_bits : nullptr;
  static bool attr = false;
  if (!attr) {
    B2_CUDA(cudaFuncSetAttribute(attention_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem));
    B2_CUDA(cudaFuncSetAttribute(attention_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem));
    attr = true;
  }
  CUtensorMap tm_ctx;
  st = get_tensor_map_2d(&tm_ctx, ctx, (uint64_t)tokens, (uint64_t)hidden, (uint64_t)(hidden * 2), 128, 64);
  if (st) return st;
  dim3 grid((unsigned)(seq / 128), (unsigned)heads, (unsigned)batch);
  if (seq == 128) {
    static bool attr128 = false;
    if (!attr128) {
      B2_CUDA(cudaFuncSetAttribute(attention_fwd128_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kFwd128Smem));
      B2_CUDA(cudaFuncSetAttribute(attention_fwd128_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                   cudaSharedmemCarveoutMaxShared));
      B2_CUDA(cudaFuncSetAttribute(attention_fwd128_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kFwd128Smem));
      B2_CUDA(cudaFuncSetAttribute(attention_fwd128_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                   cudaSharedmemCarveoutMaxShared));
      attr128 = true;
    }
    if (segments != nullptr) {
      B2_LAUNCH(attention_fwd128_kernel<true>, grid, ATT_THREADS, kFwd128Smem, stream, tm, tm_ctx, p);
    } else {
      B2_LAUNCH(attention_fwd128_kernel<false>, grid, ATT_THREADS, kFwd128Smem, stream, tm, tm_ctx, p);
    }
    B2_CUDA(cudaGetLastError());
    count_launches(1);
    return 0;
  }
  if (segments != nullptr) {
    B2_LAUNCH(attention_fwd_kernel<true>, grid, ATT_THREADS, kFwdSmem, stream, tm, tm_ctx, p);
  } else {
    B2_LAUNCH(attention_fwd_kernel<false>, grid, ATT_THREADS, kFwdSmem, stream, tm, tm_ctx, p);
  }
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  return 0;
}

extern "C" int32_t b2_attention_fwd(const void* qkv, const int64_t* attention_mask, int64_t batch, int64_t seq,
                                    int64_t heads, int64_t head_dim, float dropout_p, const void* rng_state,
                                    uint32_t rng_site, void* ctx, float* lse, uint64_t* keep_bits, void* stream_) {
  return attention_fwd_impl(qkv, attention_mask, nullptr, batch, seq, heads, head_dim, dropout_p, rng_state, rng_site,
                            ctx, lse, keep_bits, stream_);
}

extern "C" int32_t b2_attention_fwd_packed(const void* qkv, const int32_t* segments, int64_t bins, int64_t heads,
                                           int64_t head_dim, float dropout_p, const void* rng_state,
                                           uint32_t rng_site, void* ctx, float* lse, uint64_t* keep_bits,
                                           void* stream_) {
  B2_REQUIRE(segments != nullptr, "attention_fwd_packed: null segments");
  return attention_fwd_impl(qkv, nullptr, segments, bins, 128, heads, head_dim, dropout_p, rng_state, rng_site, ctx,
                            lse, keep_bits, stream_);
}

extern "C" int32_t b2_attention_fwd_packed_seq(const void* qkv, const int32_t* segments, int64_t bins, int64_t seq,
                                               int64_t heads, int64_t head_dim, float dropout_p, const void* rng_state,
                                               uint32_t rng_site, void* ctx, float* lse, uint64_t* keep_bits,
                                               void* stream_) {
  B2_REQUIRE(segments != nullptr, "attention_fwd_packed_seq: null segments");
  return attention_fwd_impl(qkv, nullptr, segments, bins, seq, heads, head_dim, dropout_p, rng_state, rng_site, ctx,
                            lse, keep_bits, stream_);
}

static int32_t attention_bwd_impl(const void* qkv, const int64_t* attention_mask, const int32_t* segments,
                                  const void* ctx, const void* d_ctx, const float* lse, int64_t batch, int64_t seq,
                                  int64_t heads, int64_t head_dim, float dropout_p, const void* rng_state,
                                  uint32_t rng_site, void* d_qkv, float* dq_accum, float* dbias_accum,
                                  const uint64_t* keep_bits, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  B2_REQUIRE(qkv && ctx && d_ctx && lse && d_qkv, "attention_bwd: null pointer");
  int32_t st = check_attn_shapes("attention_bwd", batch, seq, heads, head_dim);
  if (st) return st;
  B2_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention_bwd: dropout_p out of range");
  B2_REQUIRE(!(dropout_p > 0.f) || rng_state, "attention_bwd: dropout needs rng_state");
  B2_REQUIRE(seq == 128 || dq_accum != nullptr, "attention_bwd: seq > 128 needs the fp32 dq_accum buffer");
  B2_REQUIRE(dbias_accum == nullptr || seq == 128,
             "attention_bwd: the fused QKV bias gradient covers seq == 128 (longer sequences: use b2_colsum)");
  const int64_t hidden = heads * 64, tokens = batch * seq;
  CUtensorMap tm_qkv, tm_do;
  st = get_tensor_map_2d(&tm_qkv, qkv, (uint64_t)tokens, (uint64_t)(3 * hidden), (uint64_t)(3 * hidden * 2), 128, 64);
  if (st) return st;
  st = get_tensor_map_2d(&tm_do, d_ctx, (uint64_t)tokens, (uint64_t)hidden, (uint64_t)(hidden * 2), 128, 64);
  if (st) return st;
  CUtensorMap tm_o, tm_dqkv;
  st = get_tensor_map_2d(&tm_o, ctx, (uint64_t)tokens, (uint64_t)hidden, (uint64_t)(hidden * 2), 128, 64);
  if (st) return st;
  st = get_tensor_map_2d(&tm_dqkv, d_qkv, (uint64_t)tokens, (uint64_t)(3 * hidden), (uint64_t)(3 * hidden * 2), 128, 64);
  if (st) return st;
  AttnParams p{};
  p.batch = (int)batch; p.seq = (int)seq; p.heads = (int)heads; p.hidden = (int)hidden;
  p.scale = 0.125f;
  p.neg_log2_seq = -log2f((float)seq);
  p.dropout_p = dropout_p; p.rng = (const unsigned long long*)rng_state; p.rng_site = rng_site;
  p.mask = (const long long*)attention_mask;
  p.seg = segments;
  p.lse = const_cast<float*>(lse);
  p.ctx_in = (const __nv_bfloat16*)ctx; p.d_ctx = (const __nv_bfloat16*)d_ctx;
  p.d_qkv = (__nv_bfloat16*)d_qkv;
  p.dq_accum = seq > 128 ? dq_accum : nullptr;
  p.dbias = dbias_accum;
  p.keep_bits = (seq == 128 && dropout_p > 0.f) ? (unsigned long long*)keep_bits : nullptr;
  if (p.dq_accum) B2_CUDA(cudaMemsetAsync(p.dq_accum, 0, (size_t)tokens * hidden * 4, stream));
  static int per_sm = 0;   // resident CTAs per SM of attention_bwd128_kernel (1)
  if (per_sm == 0) {
    B2_CUDA(cudaFuncSetAttribute(attention_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmem));
    B2_CUDA(cudaFuncSetAttribute(attention_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmem));
    B2_CUDA(cudaFuncSetAttribute(attention_bwd128_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 kBwd128Smem));
    B2_CUDA(cudaFuncSetAttribute(attention_bwd128_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 cudaSharedmemCarveoutMaxShared));
    B2_CUDA(cudaFuncSetAttribute(attention_bwd128_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 kBwd128Smem));
    B2_CUDA(cudaFuncSetAttribute(attention_bwd128_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 cudaSharedmemCarveoutMaxShared));
    B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, attention_bwd128_kernel<false>, ATT_THREADS,
                                                          kBwd128Smem));
  }
  if (seq == 128) {
    unsigned grid = 0;
    st = persistent_grid(per_sm, batch * heads, &grid);
    if (st) return st;
    if (segments != nullptr) {
      B2_LAUNCH(attention_bwd128_kernel<true>, grid, ATT_THREADS, kBwd128Smem, stream, tm_qkv, tm_do, tm_o, tm_dqkv, p);
    } else {
      B2_LAUNCH(attention_bwd128_kernel<false>, grid, ATT_THREADS, kBwd128Smem, stream, tm_qkv, tm_do, tm_o, tm_dqkv,
                p);
    }
  } else {
    dim3 grid((unsigned)(seq / 128), (unsigned)heads, (unsigned)batch);
    if (segments != nullptr) {
      B2_LAUNCH(attention_bwd_kernel<true>, grid, ATT_THREADS, kBwdSmem, stream, tm_qkv, tm_do, tm_o, tm_dqkv, p);
    } else {
      B2_LAUNCH(attention_bwd_kernel<false>, grid, ATT_THREADS, kBwdSmem, stream, tm_qkv, tm_do, tm_o, tm_dqkv, p);
    }
  }
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  if (p.dq_accum) {
    const long long n4 = tokens * hidden / 4;
    B2_LAUNCH(dq_convert_kernel, (unsigned)((n4 + 255) / 256), 256, 0, stream, p.dq_accum, (__nv_bfloat16*)d_qkv,
              tokens, (int)hidden);
    B2_CUDA(cudaGetLastError());
    count_launches(1);
  }
  return 0;
}

extern "C" int32_t b2_attention_bwd(const void* qkv, const int64_t* attention_mask, const void* ctx, const void* d_ctx,
                                    const float* lse, int64_t batch, int64_t seq, int64_t heads, int64_t head_dim,
                                    float dropout_p, const void* rng_state, uint32_t rng_site, void* d_qkv,
                                    float* dq_accum, float* dbias_accum, const uint64_t* keep_bits, void* stream_) {
  return attention_bwd_impl(qkv, attention_mask, nullptr, ctx, d_ctx, lse, batch, seq, heads, head_dim, dropout_p,
                            rng_state, rng_site, d_qkv, dq_accum, dbias_accum, keep_bits, stream_);
}

extern "C" int32_t b2_attention_bwd_packed(const void* qkv, const int32_t* segments, const void* ctx,
                                           const void* d_ctx, const float* lse, int64_t bins, int64_t heads,
                                           int64_t head_dim, float dropout_p, const void* rng_state, uint32_t rng_site,
                                           void* d_qkv, float* dbias_accum, const uint64_t* keep_bits, void* stream_) {
  B2_REQUIRE(segments != nullptr, "attention_bwd_packed: null segments");
  return attention_bwd_impl(qkv, nullptr, segments, ctx, d_ctx, lse, bins, 128, heads, head_dim, dropout_p, rng_state,
                            rng_site, d_qkv, nullptr, dbias_accum, keep_bits, stream_);
}

extern "C" int32_t b2_attention_bwd_packed_seq(const void* qkv, const int32_t* segments, const void* ctx,
                                               const void* d_ctx, const float* lse, int64_t bins, int64_t seq,
                                               int64_t heads, int64_t head_dim, float dropout_p,
                                               const void* rng_state, uint32_t rng_site, void* d_qkv, float* dq_accum,
                                               float* dbias_accum, const uint64_t* keep_bits, void* stream_) {
  B2_REQUIRE(segments != nullptr, "attention_bwd_packed_seq: null segments");
  return attention_bwd_impl(qkv, nullptr, segments, ctx, d_ctx, lse, bins, seq, heads, head_dim, dropout_p, rng_state,
                            rng_site, d_qkv, dq_accum, dbias_accum, keep_bits, stream_);
}
