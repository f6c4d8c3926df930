#include "common.h"

#include <atomic>
#include <mutex>
#include <unordered_map>
#include <string.h>

namespace ab {

static thread_local char g_err[512] = {0};
std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

// Tensor maps are pure functions of (base, shape, pitch, box, type): the engine launches the same ~700 GEMM / attention
// operands every step from persistent buffers, so the encoded descriptors are kept (a plan cache keyed on the operand)
// instead of calling cuTensorMapEncodeTiled three times per launch.
namespace {
struct TmapKey {
  const void* base;
  uint64_t rows, cols, ld;
  uint32_t box_rows, box_cols, fp16;
  bool operator==(const TmapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows &&
           box_cols == o.box_cols && fp16 == o.fp16;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = reinterpret_cast<uintptr_t>(k.base) * 0x9E3779B97F4A7C15ull;
    for (uint64_t v : {k.rows, k.cols, k.ld, static_cast<uint64_t>(k.box_rows) << 32 | k.box_cols, static_cast<uint64_t>(k.fp16)})
      h = (h ^ v) * 0x100000001B3ull + (h >> 29);
    return static_cast<size_t>(h);
  }
};
std::mutex g_tmap_mutex;
std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
constexpr size_t kTmapCacheMax = 16384;
}  // namespace

int make_tmap_16bit_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols, bool fp16) {
  const TmapKey key{base, rows, cols, ld, box_rows, box_cols, fp16 ? 1u : 0u};
  {
    std::lock_guard<std::mutex> lock(g_tmap_mutex);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) {
      *out = it->second;
      return AB_OK;
    }
  }
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is unavailable (no CUDA driver?)");
    return AB_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0 || (ld * 2) % 16 != 0) {
    set_error("TMA operand must be 16-byte aligned with a 16-byte-multiple row pitch (ptr=%p ld=%llu)", base,
              (unsigned long long)ld);
    return AB_ERR_INVALID_ARGUMENT;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 2};  // bytes, dims 1..rank-1
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estride[2] = {1, 1};
  CUresult r = fn(out, fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estride,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d) rows=%llu cols=%llu ld=%llu box=%ux%u", (int)r,
              (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows, box_cols);
    return AB_ERR_CUDA;
  }
  {
    std::lock_guard<std::mutex> lock(g_tmap_mutex);
    if (g_tmap_cache.size() >= kTmapCacheMax) g_tmap_cache.clear();
    g_tmap_cache.emplace(key, *out);
  }
  return AB_OK;
}

}  // namespace ab

extern "C" {

int ab_version(void) { return AB_ABI_VERSION; }

const char* ab_last_error(void) { return ab::g_err; }

unsigned long long ab_launch_count(void) { return ab::g_launches.load(); }

}  // extern "C"
