// Library-level plumbing of the C ABI: thread-local error string, SM count cache and the
// CUtensorMap encoder (driver entry point resolved lazily so the .so loads without libcuda).
#include <cudaTypedefs.h>

#include <atomic>
#include <mutex>
#include <unordered_map>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include "common.cuh"
#include "vjepa_b200.h"

namespace vj {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) in %s", int(e), cudaGetErrorString(e), what);
  return int(e) > 0 ? int(e) : 1;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) return 132;
    n = v;
  }
  return n;
}

// SM budget of the PERSISTENT kernels (GEMM, second-generation attention): data-parallel training reserves a few SMs for
// NCCL's copy / reduce CTAs while gradient buckets are in flight, so that a collective never has to wait for a persistent
// CTA to retire and a persistent grid never queues behind a resident NCCL CTA (jepa_b200/distributed.py).
static std::atomic<int> g_sm_limit{0};
int sm_budget() {
  const int n = num_sms();
  const int lim = g_sm_limit.load(std::memory_order_relaxed);
  return (lim > 0 && lim < n) ? lim : n;
}

static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
  }
  return fn;
}

// Encoded descriptors are cached (SURVEY 8b allows it: "cached CUtensorMaps keyed by (ptr, shape, stride)"): a train step
// encodes ~2000 maps, and the caching allocator hands the same addresses back every step, so after the first step a
// launch costs one hash lookup instead of a driver call per operand.  A map is a pure function of the key.
struct TmapKey {
  const void* ptr;
  uint64_t inner, outer, ld;
  uint32_t box_inner, box_outer;
  int dtype, swizzle;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && inner == o.inner && outer == o.outer && ld == o.ld && box_inner == o.box_inner &&
           box_outer == o.box_outer && dtype == o.dtype && swizzle == o.swizzle;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = reinterpret_cast<uint64_t>(k.ptr) * 0x9E3779B97F4A7C15ull;
    auto mix = [&](uint64_t v) { h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); };
    mix(k.inner); mix(k.outer); mix(k.ld); mix((uint64_t(k.box_inner) << 32) | k.box_outer);
    mix((uint64_t(uint32_t(k.dtype)) << 32) | uint32_t(k.swizzle));
    return size_t(h);
  }
};
static std::mutex g_tmap_mu;
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
static std::atomic<long long> g_tmap_hits{0}, g_tmap_misses{0};

static int encode_tmap_2d(CUtensorMap* out, const void* ptr, int dtype, uint64_t inner, uint64_t outer, uint64_t ld_bytes,
                          uint32_t box_inner, uint32_t box_outer, int swizzle);

int make_tmap_2d(CUtensorMap* out, const void* ptr, int dtype, uint64_t inner, uint64_t outer,
                 uint64_t ld_bytes, uint32_t box_inner, uint32_t box_outer, int swizzle) {
  const TmapKey key{ptr, inner, outer, ld_bytes, box_inner, box_outer, dtype, swizzle};
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) {
      *out = it->second;
      g_tmap_hits.fetch_add(1, std::memory_order_relaxed);
      return 0;
    }
  }
  const int rc = encode_tmap_2d(out, ptr, dtype, inner, outer, ld_bytes, box_inner, box_outer, swizzle);
  if (rc) return rc;
  g_tmap_misses.fetch_add(1, std::memory_order_relaxed);
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  if (g_tmap_cache.size() >= 16384) g_tmap_cache.clear();   // shapes changing every step (dynamic masks): bounded memory
  g_tmap_cache.emplace(key, *out);
  return 0;
}

static int encode_tmap_2d(CUtensorMap* out, const void* ptr, int dtype, uint64_t inner, uint64_t outer, uint64_t ld_bytes,
                          uint32_t box_inner, uint32_t box_outer, int swizzle) {
  auto enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return 1;
  }
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstride[1] = {ld_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapSwizzle sw = swizzle == 3   ? CU_TENSOR_MAP_SWIZZLE_128B
                          : swizzle == 2 ? CU_TENSOR_MAP_SWIZZLE_64B
                          : swizzle == 1 ? CU_TENSOR_MAP_SWIZZLE_32B
                                         : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = enc(out, dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                   const_cast<void*>(ptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): ptr=%p inner=%llu outer=%llu ld=%llu box=%ux%u sw=%d",
              int(r), ptr, (unsigned long long)inner, (unsigned long long)outer,
              (unsigned long long)ld_bytes, box_inner, box_outer, swizzle);
    return 1;
  }
  return 0;
}

}  // namespace vj

extern "C" const char* vj_last_error_string(void) { return vj::g_err; }
extern "C" int vj_version(void) { return VJ_VERSION; }
extern "C" long long vj_launch_count(void) { return vj::g_launches.load(std::memory_order_relaxed); }
extern "C" int vj_set_sm_limit(int n) {
  vj::g_sm_limit.store(n < 0 ? 0 : n, std::memory_order_relaxed);
  return 0;
}
extern "C" long long vj_tmap_cache_stats(int which) {
  return which == 0 ? vj::g_tmap_hits.load(std::memory_order_relaxed) : vj::g_tmap_misses.load(std::memory_order_relaxed);
}
