// Question-answering span loss (HF BertForQuestionAnswering).  The head itself -- qa_outputs, a Linear(H, 2) on every
// token with no dropout -- is the token head (b2_token_head_fwd / b2_token_head_bwd_split with C = 2, p = 0); what is
// new is its loss, a cross-entropy over the SEQUENCE axis: per sequence one softmax over its own rows for the start
// column and one for the end column, targets clamped and ignored as HF does, and
//   loss = (mean over non-ignored start targets + mean over non-ignored end targets) / 2.
// Every sum runs in a fixed order (thread-strided, then a fixed warp tree, then the warps in index order) with no
// atomics, so the loss and d_logits are bitwise repeatable, with torch.use_deterministic_algorithms on or off.
#include "common.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

constexpr int kQaThreads = 256;      // per-sequence block; a sequence has at most 512 rows (two per thread)
constexpr int kQaMaxSeq = 512;       // the attention kernels' longest sequence
constexpr int kQaMeanThreads = 1024;

namespace {

// online (max, sum of exp) pair: merge (m2, s2) into (m, s); a pair with m = -inf is empty
__device__ __forceinline__ void qa_lse_merge(float& m, float& s, float m2, float s2) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) { m = m2; s = s2; return; }
  if (m2 > m) { s = s * expf(m - m2) + s2; m = m2; }
  else        { s = s + s2 * expf(m2 - m); }
}

// HF's clamp(0, ignored_index)
__device__ __forceinline__ long long qa_clamp(long long p, long long ignored) {
  return p < 0 ? 0 : (p > ignored ? ignored : p);
}

}  // namespace

// d_logits = 0 over every row: the packed form's unused bin rows belong to no sequence
__global__ void qa_zero_kernel(float2* __restrict__ d, long long rows) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (long long)gridDim.x * blockDim.x)
    d[i] = make_float2(0.f, 0.f);
}

// One block per sequence b, rows [row0, row0 + n) of the [rows, 2] logits (row0 = b * ignored, n = ignored when
// first / len are NULL).  Targets ts / te are HF's clamp(0, ignored); a target equal to `ignored` has no loss term and
// a zero gradient column.
//   seq_loss[2b] = lse_start - x[row0 + ts, 0]  (0 when ignored),  seq_loss[2b + 1] likewise for the end column
//   d_logits[row0 + r, c] = (softmax_c(r) - [r == t_c]) * d_loss / (2 n_c)     (0 when t_c is ignored)
// with n_c the number of sequences whose column-c target is not ignored, counted by every block over all sequences.
__global__ void __launch_bounds__(kQaThreads) qa_span_ce_kernel(const float2* __restrict__ logits, long long rows,
                                                                const long long* __restrict__ start_pos,
                                                                const long long* __restrict__ end_pos, int nseq,
                                                                long long ignored, const long long* __restrict__ first,
                                                                const long long* __restrict__ len,
                                                                const float* d_loss, float* __restrict__ seq_loss,
                                                                float2* __restrict__ dlog) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float sm_m[2][kQaThreads / 32], sm_s[2][kQaThreads / 32];
  __shared__ int sm_n[2][kQaThreads / 32];
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const long long row0 = first != nullptr ? first[b] : (long long)b * ignored;
  const long long n = len != nullptr ? len[b] : ignored;
  const long long ts = qa_clamp(start_pos[b], ignored), te = qa_clamp(end_pos[b], ignored);
  if (n < 1 || n > kQaMaxSeq || row0 < 0 || row0 + n > rows) {
    if (t == 0) printf("b2 qa span loss: sequence %d covers rows [%lld, %lld) of %lld (1 to %d rows)\n", b, row0,
                       row0 + n, rows, kQaMaxSeq);
    __trap();
  }
  if ((ts != ignored && ts >= n) || (te != ignored && te >= n)) {
    if (t == 0) printf("b2 qa span loss: sequence %d has %lld tokens, its target (start %lld, end %lld) lies outside "
                       "them and is not the ignored index %lld\n", b, n, ts, te, ignored);
    __trap();
  }
  int cs = 0, ce = 0;
  for (int i = t; i < nseq; i += kQaThreads) {
    cs += qa_clamp(start_pos[i], ignored) != ignored;
    ce += qa_clamp(end_pos[i], ignored) != ignored;
  }
  float m0 = -INFINITY, s0 = 0.f, m1 = -INFINITY, s1 = 0.f;
  for (long long r = t; r < n; r += kQaThreads) {
    const float2 v = logits[row0 + r];
    qa_lse_merge(m0, s0, v.x, 1.f);
    qa_lse_merge(m1, s1, v.y, 1.f);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    qa_lse_merge(m0, s0, __shfl_xor_sync(0xffffffffu, m0, o), __shfl_xor_sync(0xffffffffu, s0, o));
    qa_lse_merge(m1, s1, __shfl_xor_sync(0xffffffffu, m1, o), __shfl_xor_sync(0xffffffffu, s1, o));
    cs += __shfl_xor_sync(0xffffffffu, cs, o);
    ce += __shfl_xor_sync(0xffffffffu, ce, o);
  }
  if (lane == 0) {
    sm_m[0][wid] = m0; sm_s[0][wid] = s0; sm_m[1][wid] = m1; sm_s[1][wid] = s1;
    sm_n[0][wid] = cs; sm_n[1][wid] = ce;
  }
  __syncthreads();
  m0 = sm_m[0][0]; s0 = sm_s[0][0]; m1 = sm_m[1][0]; s1 = sm_s[1][0];
  cs = sm_n[0][0]; ce = sm_n[1][0];
  for (int w = 1; w < kQaThreads / 32; ++w) {     // every thread merges the warps in the same order
    qa_lse_merge(m0, s0, sm_m[0][w], sm_s[0][w]);
    qa_lse_merge(m1, s1, sm_m[1][w], sm_s[1][w]);
    cs += sm_n[0][w];
    ce += sm_n[1][w];
  }
  const float lse0 = m0 + logf(s0), lse1 = m1 + logf(s1);
  if (t == 0) {
    seq_loss[2 * b] = ts == ignored ? 0.f : lse0 - logits[row0 + ts].x;
    seq_loss[2 * b + 1] = te == ignored ? 0.f : lse1 - logits[row0 + te].y;
  }
  if (dlog == nullptr) return;
  const float dl = d_loss != nullptr ? *d_loss : 1.f;
  const float sc0 = ts == ignored ? 0.f : dl * 0.5f / (float)cs;
  const float sc1 = te == ignored ? 0.f : dl * 0.5f / (float)ce;
  for (long long r = t; r < n; r += kQaThreads) {
    const float2 v = logits[row0 + r];
    float2 d;
    d.x = ts == ignored ? 0.f : (expf(v.x - lse0) - (r == ts ? 1.f : 0.f)) * sc0;
    d.y = te == ignored ? 0.f : (expf(v.y - lse1) - (r == te ? 1.f : 0.f)) * sc1;
    dlog[row0 + r] = d;
  }
}

// loss = (sum_b seq_loss[2b] / n_start + sum_b seq_loss[2b + 1] / n_end) / 2, each sum thread-strided then a fixed
// tree; a column whose targets are all ignored gives 0 / 0 = nan, as torch's mean over an all-ignored batch
__global__ void __launch_bounds__(kQaMeanThreads) qa_span_mean_kernel(const float* __restrict__ seq_loss,
                                                                      const long long* __restrict__ start_pos,
                                                                      const long long* __restrict__ end_pos, int nseq,
                                                                      long long ignored, float* loss) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[2][kQaMeanThreads];
  __shared__ int cnt[2][kQaMeanThreads];
  const int t = threadIdx.x;
  float a = 0.f, e = 0.f;
  int na = 0, ne = 0;
  for (int i = t; i < nseq; i += kQaMeanThreads) {
    a += seq_loss[2 * i];
    e += seq_loss[2 * i + 1];
    na += qa_clamp(start_pos[i], ignored) != ignored;
    ne += qa_clamp(end_pos[i], ignored) != ignored;
  }
  red[0][t] = a; red[1][t] = e; cnt[0][t] = na; cnt[1][t] = ne;
  __syncthreads();
  for (int w = kQaMeanThreads / 2; w > 0; w >>= 1) {
    if (t < w) {
      red[0][t] += red[0][t + w];
      red[1][t] += red[1][t + w];
      cnt[0][t] += cnt[0][t + w];
      cnt[1][t] += cnt[1][t + w];
    }
    __syncthreads();
  }
  if (t == 0) *loss = (red[0][0] / (float)cnt[0][0] + red[1][0] / (float)cnt[1][0]) * 0.5f;
}

}  // namespace b2

using namespace b2;

extern "C" int32_t b2_qa_span_loss(const float* logits, int64_t rows, const int64_t* start_positions,
                                   const int64_t* end_positions, int64_t num_seqs, int64_t ignored_index,
                                   const int64_t* seq_first, const int64_t* seq_len, const float* d_loss,
                                   float* seq_loss, float* d_logits, float* loss, void* stream) {
  B2_REQUIRE(logits && start_positions && end_positions && seq_loss, "qa_span_loss: null pointer");
  B2_REQUIRE(((uintptr_t)logits & 7) == 0 && ((uintptr_t)d_logits & 7) == 0,
             "qa_span_loss: logits / d_logits must be 8-byte aligned ([rows, 2] fp32)");
  B2_REQUIRE(rows > 0 && num_seqs > 0 && num_seqs <= rows && num_seqs <= INT_MAX,
             "qa_span_loss: rows=%lld num_seqs=%lld (1 <= num_seqs <= rows)", (long long)rows, (long long)num_seqs);
  B2_REQUIRE(ignored_index >= 1 && ignored_index <= kQaMaxSeq,
             "qa_span_loss: ignored_index=%lld must be the padded sequence length, 1 to %d", (long long)ignored_index,
             kQaMaxSeq);
  B2_REQUIRE((seq_first == nullptr) == (seq_len == nullptr),
             "qa_span_loss: seq_first and seq_len go together (both NULL: padded sequences of ignored_index rows)");
  B2_REQUIRE(seq_first != nullptr || num_seqs * ignored_index == rows,
             "qa_span_loss: padded rows=%lld != num_seqs=%lld x ignored_index=%lld", (long long)rows,
             (long long)num_seqs, (long long)ignored_index);
  if (d_logits != nullptr && seq_first != nullptr) {
    long long g = (rows + 255) / 256;
    if (g > 132 * 8) g = 132 * 8;
    B2_LAUNCH(qa_zero_kernel, (unsigned)g, 256, 0, stream, (float2*)d_logits, (long long)rows);
    B2_CUDA(cudaGetLastError());
    count_launches(1);
  }
  B2_LAUNCH(qa_span_ce_kernel, (unsigned)num_seqs, kQaThreads, 0, stream, (const float2*)logits, (long long)rows,
            (const long long*)start_positions, (const long long*)end_positions, (int)num_seqs,
            (long long)ignored_index, (const long long*)seq_first, (const long long*)seq_len, d_loss, seq_loss,
            (float2*)d_logits);
  B2_CUDA(cudaGetLastError());
  count_launches(1);
  if (loss != nullptr) {
    B2_LAUNCH(qa_span_mean_kernel, 1, kQaMeanThreads, 0, stream, (const float*)seq_loss,
              (const long long*)start_positions, (const long long*)end_positions, (int)num_seqs,
              (long long)ignored_index, loss);
    B2_CUDA(cudaGetLastError());
    count_launches(1);
  }
  return 0;
}
