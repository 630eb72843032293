#include "host.h"

#include <cudaTypedefs.h>
#include <stdarg.h>
#include <stdio.h>

#include <string.h>

#include <atomic>
#include <mutex>
#include <unordered_map>

namespace b200 {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// cuTensorMapEncodeTiled is a driver entry point; resolve it through the runtime so the
// library has no link-time dependency on libcuda (the CPU build box has no driver).
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
  });
  return fn;
}

// A tensor map is a pure function of (base, dtype, rank, dims, strides, box, swizzle), and a training step presents
// the same few hundred combinations every step (flat parameter store, persistent workspaces, the allocator's recurring
// activation addresses): keep the encoded descriptors, so the per-launch host cost is a hash lookup instead of a
// driver call (~300 encodes per C2 step otherwise).
namespace {
struct MapKey {
  uint64_t w[16];
  bool operator==(const MapKey& o) const { return memcmp(w, o.w, sizeof(w)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = 0x9E3779B97F4A7C15ull;
    for (uint64_t x : k.w) h = (h ^ x) * 0xFF51AFD7ED558CCDull + (h >> 29);
    return (size_t)h;
  }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
std::atomic<unsigned long long> g_map_hits{0}, g_map_misses{0};
constexpr size_t kMapCacheCap = 8192;
}  // namespace

int make_tensor_map(CUtensorMap* out, const void* base, CUtensorMapDataType dtype, int elem_bytes,
                    int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, bool swizzle128) {
  MapKey key{};
  const bool cacheable = rank >= 1 && rank <= 5;
  if (cacheable) {
    key.w[0] = reinterpret_cast<uintptr_t>(base);
    key.w[1] = ((uint64_t)dtype << 32) | ((uint64_t)rank << 8) | (swizzle128 ? 1u : 0u) | ((uint64_t)elem_bytes << 16);
    for (int i = 0; i < rank; ++i) {
      key.w[2 + i] = dims[i];
      key.w[7 + i] = box[i];
      if (i + 1 < rank) key.w[12 + i] = strides_bytes[i];
    }
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) {
      *out = it->second;
      g_map_hits.fetch_add(1, std::memory_order_relaxed);
      return B200_OK;
    }
  }
  g_map_misses.fetch_add(1, std::memory_order_relaxed);
  auto encode = get_encode();
  if (!encode) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return B200_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0) {
    set_error("TMA base address %p is not 16-byte aligned", base);
    return B200_ERR_ARG;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (strides_bytes[i] % 16 != 0) {
      set_error("TMA stride[%d]=%llu bytes is not a multiple of 16", i,
                (unsigned long long)strides_bytes[i]);
      return B200_ERR_ARG;
    }
  }
  if (swizzle128 && box[0] * (uint32_t)elem_bytes > 128) {
    set_error("TMA inner box %u x %d B exceeds the 128-byte swizzle span", box[0], elem_bytes);
    return B200_ERR_ARG;
  }
  cuuint64_t gdims[5];
  cuuint64_t gstrides[4];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
    if (i + 1 < rank) gstrides[i] = strides_bytes[i];
  }
  CUresult r = encode(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdims, gstrides, gbox,
                      estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)",
              (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              box[0], rank > 1 ? box[1] : 0);
    return B200_ERR_CUDA;
  }
  if (cacheable) {
    std::lock_guard<std::mutex> lk(g_map_mu);
    if (g_maps.size() >= kMapCacheCap) g_maps.clear();   // addresses churned (e.g. a new model): start over
    g_maps.emplace(key, *out);
  }
  return B200_OK;
}

static std::atomic<unsigned long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 148;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 148;
  }
  return n;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_version(void) { return 4; }
const char* b200_last_error(void) { return g_err; }

unsigned long long b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
void b200_tensor_map_cache_stats(unsigned long long* hits, unsigned long long* misses) {
  if (hits) *hits = g_map_hits.load(std::memory_order_relaxed);
  if (misses) *misses = g_map_misses.load(std::memory_order_relaxed);
}

int b200_device_ok(void) {
  int dev = 0, major = 0, minor = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
  return (major == 9 && minor == 0) ? 1 : 0;  // the library holds sm_90a code only
}

}  // extern "C"
