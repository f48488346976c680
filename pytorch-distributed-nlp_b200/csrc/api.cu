// Library plumbing: thread-local error string, CUDA status conversion, TMA tensor-map encoding (+cache).
#include "common.cuh"
#include "../../include/b2_ddp_bert.h"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <mutex>
#include <unordered_map>

namespace b2 {

static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};
void count_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int32_t check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
  return -1;
}

// cuTensorMapEncodeTiled lives in libcuda; resolve it through the runtime so we never link the driver stub.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;
static std::mutex g_mu;

struct MapKey {
  const void* base; uint64_t rows, cols, pitch; uint32_t box_rows, box_cols;
  bool operator==(const MapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && pitch == o.pitch && box_rows == o.box_rows &&
           box_cols == o.box_cols;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = (size_t)k.base;
    h = h * 1000003u ^ k.rows; h = h * 1000003u ^ k.cols; h = h * 1000003u ^ k.pitch;
    h = h * 1000003u ^ k.box_rows; h = h * 1000003u ^ k.box_cols;
    return h;
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;

int32_t get_tensor_map_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_bytes,
                          uint32_t box_rows, uint32_t box_cols) {
  std::lock_guard<std::mutex> lk(g_mu);
  MapKey key{base, rows, cols, pitch_bytes, box_rows, box_cols};
  auto it = g_maps.find(key);
  if (it != g_maps.end()) {
    *out = it->second;
    return 0;
  }
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
      set_error("cannot resolve cuTensorMapEncodeTiled (cuda error %d, query %d): no CUDA driver?", (int)e,
                (int)qres);
      return -1;
    }
    g_encode = (EncodeTiledFn)fn;
  }
  if (pitch_bytes % 16 != 0 || ((uintptr_t)base % 16) != 0) {
    set_error("tensor map: base/pitch must be 16-byte aligned (base=%p pitch=%llu)", base,
              (unsigned long long)pitch_bytes);
    return -2;
  }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMap m;
  CUresult r = g_encode(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu pitch=%llu box=%ux%u", (int)r,
              (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)pitch_bytes, box_rows, box_cols);
    return -1;
  }
  if (g_maps.size() > 4096) g_maps.clear();
  g_maps.emplace(key, m);
  *out = m;
  return 0;
}

}  // namespace b2

extern "C" const char* b2_last_error(void) { return b2::g_err; }
extern "C" int32_t b2_abi_version(void) { return B2_ABI_VERSION; }
extern "C" int64_t b2_launch_count(void) { return (int64_t)b2::g_launches.load(std::memory_order_relaxed); }
