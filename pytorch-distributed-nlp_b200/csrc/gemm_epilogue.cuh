// GEMM epilogue: fp32 accumulator tile (shared memory) -> fused element-wise math -> HBM, with COALESCED global traffic.
//
// The mainloop leaves the [128 x BN] fp32 accumulator in shared memory (wgmma fragments written out row-major), and
// every epilogue thread then owns one accumulator ROW.  Storing rows straight from registers would make each
// warp-wide 16-byte store touch 32 different 128-byte lines (one per row).  Here each epilogue warp owns a 4 KB
// shared-memory staging tile (32 rows x 128 B, 16-byte chunks XOR-swizzled by row & 7 so both access patterns are
// bank-conflict free).  Rows go registers -> staging -> global with every warp-wide access covering 4 rows x 128
// contiguous bytes (4 full lines); auxiliary inputs (residual, saved pre-activation) take the same path in reverse.
#pragma once
#include "common.cuh"
#include "../../include/b2_ddp_bert.h"

namespace b2 {

struct GemmKernelParams {
  int M, N, K;
  int tiles_m, tiles_n, splits, kblocks_per_split, kblocks_total;
  int epilogue;
  __nv_bfloat16* D; long long ldd;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* aux_in; long long ld_aux_in;
  __nv_bfloat16* aux_out; long long ld_aux_out;
  float* partial;  // split-K fp32 partials [splits][M][N]
  float dropout_p; const unsigned long long* rng; unsigned rng_site;
  long long* timing;  // unused by the H100 kernels (ABI field)
  float* colsum;      // optional fp32 [N]: += column sums of the bf16 output (bias gradient of the producing layer)
};

constexpr int kEpiStageBytes = 32 * 128;   // per epilogue warp

#ifdef __CUDACC__
// Staging tile of one epilogue warp: 32 rows x CH 16-byte chunks (CH = 8: 128-byte rows = 64 bf16 / 32 fp32 columns;
// CH = 4: 64-byte rows = 32 bf16 columns, two rows sharing one 128-byte line).  Chunks are XOR-swizzled so that both
// access patterns -- a thread walking its own row, and the warp copying 128-byte lines to/from global memory -- are
// free of bank conflicts.
template <int CH>
__device__ __forceinline__ uint4* stage_ptr(uint8_t* stage, int row, int chunk) {
  if (CH == 8) return reinterpret_cast<uint4*>(stage + row * 128 + ((chunk ^ (row & 7)) << 4));
  return reinterpret_cast<uint4*>(stage + (row >> 1) * 128 + (((((row & 1) << 2) | chunk) ^ ((row >> 1) & 7)) << 4));
}
// coalesced copy of a [32 rows x CH*16 bytes] tile between global memory (row pitch in bytes) and the staging tile:
// each warp-wide step moves 512 contiguous-by-row bytes (CH = 8: 4 rows x 128 B, CH = 4: 8 rows x 64 B).
// Rows >= rows_valid are skipped (zero-filled on load).
template <int CH>
__device__ __forceinline__ void tile_s2g(uint8_t* stage, uint8_t* g, long long pitch, int lane, int rows_valid) {
  constexpr int RPS = 32 / CH;   // rows per step
#pragma unroll
  for (int k = 0; k < CH; ++k) {
    const int r = RPS * k + lane / CH, c = lane % CH;
    const uint4 v = *stage_ptr<CH>(stage, r, c);
    if (r < rows_valid) *reinterpret_cast<uint4*>(g + (size_t)r * pitch + c * 16) = v;
  }
}
// same tile walk, but ADDING the fp32 tile into global memory (one 16-byte vector reduction per lane and step)
__device__ __forceinline__ void tile_s2g_red_f32(uint8_t* stage, uint8_t* g, long long pitch, int lane,
                                                 int rows_valid) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int r = 4 * k + (lane >> 3), c = lane & 7;
    const uint4 v = *stage_ptr<8>(stage, r, c);
    if (r < rows_valid)
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(g + (size_t)r * pitch + c * 16),
                   "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
                   "f"(__uint_as_float(v.w))
                   : "memory");
  }
}
// global -> staging, asynchronous (cp.async, no registers held): issue early, tile_async_wait() + __syncwarp() before
// any lane reads the tile
template <int CH>
__device__ __forceinline__ void tile_g2s_async(uint8_t* stage, const uint8_t* g, long long pitch, int lane,
                                               int rows_valid) {
  constexpr int RPS = 32 / CH;
#pragma unroll
  for (int k = 0; k < CH; ++k) {
    const int r = RPS * k + lane / CH, c = lane % CH;
    uint4* dst = stage_ptr<CH>(stage, r, c);
    if (r < rows_valid) {
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(g + (size_t)r * pitch + c * 16)
                   : "memory");
    } else {
      *dst = make_uint4(0u, 0u, 0u, 0u);
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tile_async_wait() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// 32 consecutive fp32 accumulator columns of this thread's row (shared memory, 16-byte aligned)
__device__ __forceinline__ void acc_ld32(const float* a, uint32_t (&v)[32]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint4 t = *reinterpret_cast<const uint4*>(a + 4 * k);
    v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
  }
}

// 32 bf16 columns (4 chunks, starting at chunk c0) of this thread's own row (row == lane) <-> 32 fp32 registers
template <int CH>
__device__ __forceinline__ void row_write32(uint8_t* stage, int lane, int c0, const float (&f)[32]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    uint4 o;
    o.x = pack_bf16(f[8 * c + 0], f[8 * c + 1]); o.y = pack_bf16(f[8 * c + 2], f[8 * c + 3]);
    o.z = pack_bf16(f[8 * c + 4], f[8 * c + 5]); o.w = pack_bf16(f[8 * c + 6], f[8 * c + 7]);
    *stage_ptr<CH>(stage, lane, c0 + c) = o;
  }
}
template <int CH>
__device__ __forceinline__ void row_read32(uint8_t* stage, int lane, int c0, float (&r)[32]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const uint4 t = *stage_ptr<CH>(stage, lane, c0 + c);
    r[8 * c + 0] = bf16_lo(t.x); r[8 * c + 1] = bf16_hi(t.x); r[8 * c + 2] = bf16_lo(t.y); r[8 * c + 3] = bf16_hi(t.y);
    r[8 * c + 4] = bf16_lo(t.z); r[8 * c + 5] = bf16_hi(t.z); r[8 * c + 6] = bf16_lo(t.w); r[8 * c + 7] = bf16_hi(t.w);
  }
}

// The 8 epilogue warps (4 .. 11) drain one [128 rows x BN cols] accumulator: warp -> (row quarter, column half),
// thread -> one row.  All math happens in passes of 32 columns (32 + 32 live registers).
constexpr int kEpiWarps = 8;
template <int BN>
__device__ __forceinline__ void epilogue_tile(const GemmKernelParams& p, const DropCtx& drop, const float* acc,
                                              int acc_ld, int warp, int lane, int m_base, int n0, int split,
                                              uint8_t* stage) {
  static_assert(BN == 128 || BN == 256, "tile widths on the path");
  constexpr int kColsPerWarp = BN / 2;                        // 64 or 128
  constexpr int WT = 64;                                      // bf16 staging-tile width (columns)
  constexpr int CH = WT / 8;                                  // 16-byte chunks per staged bf16 row
  const int quarter = warp & 3;           // row quarter
  const int cgrp = (warp - 4) >> 2;       // column half
  const int row0 = m_base + quarter * 32;
  const int rows_valid = p.M - row0;      // <= 0: nothing to write; >= 32: full tile
  const int m = row0 + lane;
  const int nw = n0 + cgrp * kColsPerWarp;
  const float* arow = acc + (size_t)(quarter * 32 + lane) * acc_ld + cgrp * kColsPerWarp;

  if (p.epilogue == B2_EPI_PARTIAL_F32 || p.epilogue == B2_EPI_RESIDUAL_F32 || p.epilogue == B2_EPI_ACCUM_F32) {
    // ---- fp32 outputs: 32 columns (128 bytes) per group ----
    // ACCUM_F32: D += acc with vector reductions at L2 -- D already holds the residual stream, and split-K slices
    // of one tile simply add into the same place (no partial buffer, no reduce pass)
    const bool accum = p.epilogue == B2_EPI_ACCUM_F32;
    const bool no_aux = p.epilogue != B2_EPI_RESIDUAL_F32;
    const bool to_ws = p.epilogue == B2_EPI_PARTIAL_F32;
    float* dst_base = to_ws ? p.partial + (size_t)split * p.M * p.N : reinterpret_cast<float*>(p.D);
    const long long dst_ld = to_ws ? (long long)p.N : p.ldd;
    // the auxiliary tile (fp32 residual) does not depend on the accumulator: fetch it before waiting for the MMAs,
    // and the next group's while the current one is being combined and stored
    auto prefetch = [&](int c) {
      const int n = nw + c * 32;
      if (!no_aux && n < p.N && rows_valid > 0)
        tile_g2s_async<8>(stage, reinterpret_cast<const uint8_t*>(reinterpret_cast<const float*>(p.aux_in) +
                                                                 (size_t)row0 * p.ld_aux_in + n),
                          p.ld_aux_in * 4, lane, rows_valid);
    };
    prefetch(0);
#pragma unroll 1
    for (int c = 0; c < kColsPerWarp / 32; ++c) {
      const int n = nw + c * 32;
      uint32_t v[32];
      acc_ld32(arow + c * 32, v);
      if (n < p.N && rows_valid > 0) {
        if (!no_aux) {
          if (c > 0) prefetch(c);
          tile_async_wait();
          __syncwarp();
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const uint4 t = *stage_ptr<8>(stage, lane, k);
            v[4 * k + 0] = __float_as_uint(__uint_as_float(v[4 * k + 0]) + __uint_as_float(t.x));
            v[4 * k + 1] = __float_as_uint(__uint_as_float(v[4 * k + 1]) + __uint_as_float(t.y));
            v[4 * k + 2] = __float_as_uint(__uint_as_float(v[4 * k + 2]) + __uint_as_float(t.z));
            v[4 * k + 3] = __float_as_uint(__uint_as_float(v[4 * k + 3]) + __uint_as_float(t.w));
          }
          __syncwarp();
        }
#pragma unroll
        for (int k = 0; k < 8; ++k)
          *stage_ptr<8>(stage, lane, k) = make_uint4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
        __syncwarp();
        uint8_t* gdst = reinterpret_cast<uint8_t*>(dst_base + (size_t)row0 * dst_ld + n);
        if (accum) tile_s2g_red_f32(stage, gdst, dst_ld * 4, lane, rows_valid);
        else       tile_s2g<8>(stage, gdst, dst_ld * 4, lane, rows_valid);
      }
      __syncwarp();
    }
    return;
  }

  // ---- bf16 outputs: staging tiles of WT columns, register passes of 32 columns ----
  const bool has_aux = p.epilogue == B2_EPI_BIAS_DROPOUT_RESIDUAL || p.epilogue == B2_EPI_RESIDUAL ||
                       p.epilogue == B2_EPI_GELU_BWD;
  auto prefetch = [&](int t) {
    const int n = nw + t * WT;
    if (has_aux && n < p.N && rows_valid > 0)
      tile_g2s_async<CH>(stage, reinterpret_cast<const uint8_t*>(p.aux_in + (size_t)row0 * p.ld_aux_in + n),
                         p.ld_aux_in * 2, lane, rows_valid);
  };
  prefetch(0);   // residual / saved pre-activation tile
#pragma unroll 1
  for (int t = 0; t < kColsPerWarp / WT; ++t) {
    const int n = nw + t * WT;
    const bool active = n < p.N && rows_valid > 0;
    if (has_aux && active) {
      if (t > 0) prefetch(t);
      tile_async_wait();
      __syncwarp();
    }
#pragma unroll 1
    for (int h = 0; h < WT / 32; ++h) {
      float f[32];
      {
        uint32_t v[32];
        acc_ld32(arow + t * WT + h * 32, v);
#pragma unroll
        for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]);
      }
      if (!active) continue;
      const int nh = n + h * 32;
      if (p.bias != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          const uint4 b = ldg16(p.bias + nh + j);
          f[j + 0] += bf16_lo(b.x); f[j + 1] += bf16_hi(b.x); f[j + 2] += bf16_lo(b.y); f[j + 3] += bf16_hi(b.y);
          f[j + 4] += bf16_lo(b.z); f[j + 5] += bf16_hi(b.z); f[j + 6] += bf16_lo(b.w); f[j + 7] += bf16_hi(b.w);
        }
      }
      if (has_aux) {
        float r[32];
        row_read32<CH>(stage, lane, 4 * h, r);   // own row of the prefetched tile; overwritten in place below
        if (p.epilogue == B2_EPI_BIAS_DROPOUT_RESIDUAL) {
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            const uint32_t keep = dropout_keep8(drop, (unsigned long long)m * p.N + nh + j);
#pragma unroll
            for (int i = 0; i < 8; ++i) f[j + i] = (((keep >> i) & 1u) ? f[j + i] * drop.scale : 0.f) + r[j + i];
          }
        } else if (p.epilogue == B2_EPI_RESIDUAL) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] += r[j];
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] *= gelu_erf_grad(r[j]);
        }
      }
      row_write32<CH>(stage, lane, 4 * h, f);   // BIAS_GELU: this is the pre-activation u (kept for the backward)
    }
    if (active) {
      __syncwarp();
      if (p.epilogue == B2_EPI_BIAS_GELU) {
        tile_s2g<CH>(stage, reinterpret_cast<uint8_t*>(p.aux_out + (size_t)row0 * p.ld_aux_out + n), p.ld_aux_out * 2,
                     lane, rows_valid);
        __syncwarp();
        // gelu of exactly what was stored: read the bf16-rounded u back from this thread's own staged row
#pragma unroll 1
        for (int h = 0; h < WT / 32; ++h) {
          float f[32];
          row_read32<CH>(stage, lane, 4 * h, f);
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] = gelu_erf(f[j]);
          row_write32<CH>(stage, lane, 4 * h, f);
        }
        __syncwarp();
      }
      if (p.colsum != nullptr) {
        // bias gradient of the layer that produced this tensor: column sums of what was just rounded to bf16, over
        // the 32 staged rows (conflict-free 4-byte reads); WT = 64: lane l owns columns 2l, 2l+1; WT = 32: lanes
        // 0-15 own two columns each
        float s0 = 0.f, s1 = 0.f;
        const int nr = rows_valid < 32 ? rows_valid : 32;
        if (WT == 64 || lane < 16) {
          for (int r = 0; r < nr; ++r) {
            const uint32_t w = *reinterpret_cast<const uint32_t*>(
                reinterpret_cast<const uint8_t*>(stage_ptr<CH>(stage, r, lane >> 2)) + (lane & 3) * 4);
            s0 += bf16_lo(w);
            s1 += bf16_hi(w);
          }
          atomicAdd(p.colsum + n + 2 * lane, s0);
          atomicAdd(p.colsum + n + 2 * lane + 1, s1);
        }
      }
      tile_s2g<CH>(stage, reinterpret_cast<uint8_t*>(p.D + (size_t)row0 * p.ldd + n), p.ldd * 2, lane, rows_valid);
    }
    __syncwarp();
  }
}
#endif  // __CUDACC__

}  // namespace b2
