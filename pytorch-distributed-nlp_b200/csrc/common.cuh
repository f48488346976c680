// Shared device/host helpers for the sm_90a kernels of the DDP BERT fine-tuning step.
// Everything here is written for one target only: H100, compute_90a.
//   - raw PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), clusters / distributed shared memory
//   - wgmma shared-memory descriptors (bit layout documented inline; the MMA wrappers are in wgmma.cuh)
//   - Philox4x32-10 counter RNG for the 38 dropout sites (regenerated, never stored)
//   - bf16 pack/unpack and warp reductions
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdio>
#include "wgmma.cuh"

namespace b2 {

// ----------------------------------------------------------------------------------------------
// error plumbing (host)
// ----------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int32_t check_cuda(cudaError_t e, const char* what);
void count_launches(int n);  // kernels launched by this library (bench.py reports them as gpu_launches)
#define B2_CUDA(expr)                                                   \
  do {                                                                  \
    int32_t _s = ::b2::check_cuda((expr), #expr);                       \
    if (_s != 0) return _s;                                             \
  } while (0)
#define B2_REQUIRE(cond, ...)                                           \
  do {                                                                  \
    if (!(cond)) {                                                      \
      ::b2::set_error(__VA_ARGS__);                                     \
      return -2;                                                        \
    }                                                                   \
  } while (0)

// Encodes (and caches) a 2-D bf16 tensor map: rows x cols, row pitch in bytes, 128B swizzle.
// box_cols is always 64 elements (=128 bytes = one swizzle row).
int32_t get_tensor_map_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                          uint64_t pitch_bytes, uint32_t box_rows, uint32_t box_cols);

#ifdef __CUDACC__
// ----------------------------------------------------------------------------------------------
// kernel launch: cudaLaunchKernelEx with the programmatic-stream-serialization attribute (PDL), so that back-to-back
// kernels of a step (318 per step, captured in one CUDA graph) overlap launch latency with the predecessor's tail
// ----------------------------------------------------------------------------------------------
template <typename... KArgs, typename... Args>
inline void launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                          Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  (void)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);   // errors surface via cudaGetLastError()
}
#define B2_LAUNCH(kernel, grid, block, smem, stream, ...) \
  ::b2::launch_kernel(kernel, dim3(grid), dim3(block), (size_t)(smem), (cudaStream_t)(stream), ##__VA_ARGS__)

// ----------------------------------------------------------------------------------------------
// small device helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
// First 1024-byte boundary inside a dynamic shared-memory window (TMA / wgmma 128-byte-swizzle tiles).  Written as
// `base + offset` -- NOT as a round trip through uintptr_t -- so that every pointer derived from the result is still
// known to the compiler to be SHARED: the cast form degraded each staging-tile access of the epilogues to a generic
// LD.E / ST.E (address-space check, L1 tag stage, and a memory barrier that must wait for them) instead of LDS / STS.
__device__ __forceinline__ uint8_t* smem_align_1024(uint8_t* smem_raw) {
  return smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

// erf-based GELU (transformers' "gelu", activations.py:85-89) and its derivative for the backward epilogue.
// erf via Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, far below bf16 resolution): one rcp.approx + one ex2.approx
// + 5 FMA.  The GELU epilogues are instruction-bound (ncu: ~22 SASS instructions per element before this form), so
// every constant is folded: hq = (1 - erf(|x|/sqrt2)) / 2 = poly_half(t) * t * exp(-x^2/2), t = 1/(1 + p|x|/sqrt2),
// with the 1/2 folded into the polynomial coefficients, and
//   gelu(x)  = max(x, 0) - |x| * hq                      (x >= 0: x(1-hq);  x < 0: x*hq)
//   gelu'(x) = cdf + x * pdf,  cdf = x >= 0 ? 1 - hq : hq,  pdf = exp(-x^2/2) / sqrt(2 pi)
// The same exp(-x^2/2) serves erf and the normal pdf of the derivative.
__device__ __forceinline__ void gelu_hq(float x, float& hq, float& e) {
  float t;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"((x * x) * -0.72134752044448170f));      // exp(-x^2/2)
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(fabsf(x), 0.23164189f, 1.0f)));     // p/sqrt2 = 0.3275911/1.41421356
  float poly = fmaf(0.5307027145f, t, -0.7265760135f);   // A&S 7.1.26 coefficients a5..a1, halved
  poly = fmaf(poly, t, 0.7107068705f);
  poly = fmaf(poly, t, -0.142248368f);
  poly = fmaf(poly, t, 0.127414796f);
  hq = (poly * t) * e;
}
__device__ __forceinline__ float gelu_erf(float x) {
  float hq, e;
  gelu_hq(x, hq, e);
  return fmaf(-fabsf(x), hq, fmaxf(x, 0.f));
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  float hq, e;
  gelu_hq(x, hq, e);
  const float cdf = x >= 0.f ? 1.0f - hq : hq;
  return fmaf(x * 0.3989422804014327f, e, cdf);
}
// 2^x on the SFU without exp2f's denormal-range fix-up (arguments here are <= 0 or already flushed; the masked-key
// bias -3.4e38 gives exactly 0)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// round two fp32 values to bf16 (one F2FP) and hand back both the packed pair and the rounded values as fp32
__device__ __forceinline__ uint32_t pack_bf16_round(float& lo, float& hi) {
  const uint32_t u = pack_bf16(lo, hi);
  lo = bf16_lo(u);
  hi = bf16_hi(u);
  return u;
}

// ----------------------------------------------------------------------------------------------
// Philox4x32-10.  key = (seed_lo, seed_hi); counter = (idx_lo, idx_hi, site, step).
// One call yields 128 random bits = eight 16-bit lanes -> eight dropout decisions.
// keep(element) <=> u16 >= thresh, thresh = round(p * 65536).
// ----------------------------------------------------------------------------------------------
struct Philox4 {
  uint32_t x, y, z, w;
};
__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                 uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  return Philox4{c0, c1, c2, c3};
}

// Dropout state shared by every kernel of one step.  rng[0] = seed, rng[1] = step counter (bumped
// on the device by the optimizer kernel so that CUDA-graph replays draw fresh masks).
struct DropCtx {
  uint32_t k0, k1, step, site, thresh;
  float scale;  // 1/(1-p); p == 0 -> thresh == 0 and every element is kept
};
__device__ __forceinline__ DropCtx make_drop_ctx(const unsigned long long* rng, uint32_t site, float p) {
  DropCtx d;
  unsigned long long seed = rng ? rng[0] : 0ull;
  unsigned long long step = rng ? rng[1] : 0ull;
  d.k0 = (uint32_t)seed; d.k1 = (uint32_t)(seed >> 32);
  d.step = (uint32_t)step; d.site = site;
  d.thresh = (uint32_t)(p * 65536.0f + 0.5f);
  d.scale = (p > 0.f) ? 1.0f / (1.0f - p) : 1.0f;
  return d;
}
// 8 consecutive elements starting at element index `idx` (idx % 8 == 0): bit i of the result is set
// when element idx+i is KEPT.
__device__ __forceinline__ uint32_t dropout_keep8(const DropCtx& d, unsigned long long idx) {
  if (d.thresh == 0) return 0xffu;
  const unsigned long long g = idx >> 3;
  Philox4 r = philox4x32_10((uint32_t)g, (uint32_t)(g >> 32), d.site, d.step, d.k0, d.k1);
  uint32_t m = 0;
  m |= ((r.x & 0xffffu) >= d.thresh) << 0;
  m |= ((r.x >> 16) >= d.thresh) << 1;
  m |= ((r.y & 0xffffu) >= d.thresh) << 2;
  m |= ((r.y >> 16) >= d.thresh) << 3;
  m |= ((r.z & 0xffffu) >= d.thresh) << 4;
  m |= ((r.z >> 16) >= d.thresh) << 5;
  m |= ((r.w & 0xffffu) >= d.thresh) << 6;
  m |= ((r.w >> 16) >= d.thresh) << 7;
  return m;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (-> CUDA error -> RuntimeError on the
// host), never as a hung GPU.  2^24 polls of a suspending try_wait is seconds, far beyond any tile.  (No printf here:
// a function call inside a wgmma mainloop makes ptxas serialise the asynchronous MMAs.)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) __trap();
  }
}

// generic-proxy writes to smem -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load: coordinates are (c0 = innermost/column element index, c1 = row index)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 2-D tile store smem -> global (bulk async-group); rows/columns outside the tensor are clipped by the hardware.
// The smem tile must have been made visible to the async proxy (fence_proxy_async_smem + barrier) beforehand.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
// closes the bulk group of the stores issued by this thread and waits until they have completed (the CTA may then
// exit or reuse the tiles)
__device__ __forceinline__ void tma_store_commit_and_wait() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// clusters and distributed shared memory
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t mapa_u32(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
// 8-byte store into the shared memory of a CTA of the cluster (address from mapa_u32)
__device__ __forceinline__ void st_cluster_f32x2(uint32_t cluster_addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(cluster_addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// barrier over `count` threads (whole warps) of the CTA, ids 1..15 (0 is __syncthreads)
__device__ __forceinline__ void named_barrier_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---- wgmma shared-memory matrix descriptor (64 bit), SWIZZLE_128B ---------------------------------
//   [ 0,14) start address >> 4          [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4 [49,52) base offset (0: swizzle atoms 1024-byte aligned)
//   [62,64) layout type (1 = SWIZZLE_128B)
// K-major operand tile  (rows = M/N index, 64 bf16 = 128 B per row, rows 128 B apart, TMA-swizzled):
//   SBO = 1024 B (8 rows), LBO unused.  Advancing K by 16 elements = +32 B on the start address.
// MN-major operand tile (rows = K index, 64 bf16 of the M/N index per 128 B row; further 64-wide
//   M/N chunks are separate [BK x 128 B] slabs): SBO = 1024 B (8 k-rows), LBO = slab pitch.
//   Advancing K by 16 = +16 rows = +2048 B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fffu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// Programmatic dependent launch (PDL).  Every kernel of the library starts with pdl_wait(): it returns once all
// kernels it depends on have completed and flushed, so whatever precedes it (nothing, by convention) may overlap the
// predecessor's tail; pdl_launch_dependents() then allows the next kernel of the stream to start launching while
// this one runs.  Both are no-ops for launches without the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// vectorised global access helpers
__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void stg16(void* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }
#endif  // __CUDACC__

}  // namespace b2
