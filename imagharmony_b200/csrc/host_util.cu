// Error reporting, tensor-map cache and misc C-ABI entry points (ih_last_error, ih_version, launch counter).
#include "host_util.h"

#include <cudaTypedefs.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <string>
#include <unordered_map>

#include "../../include/ih_api.h"

namespace ih {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

static PFN_cuTensorMapEncodeTiled get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled>(p);
  }();
  return fn;
}

struct TmapKey {
  const void* base;
  uint64_t dims[5];
  uint64_t strides[4];
  uint32_t box[5];
  int rank;
  int swz;
};

static std::mutex g_tmap_mu;
static std::unordered_map<std::string, CUtensorMap> g_tmap_cache;

int get_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int swizzle_bytes) {
  if (swizzle_bytes != 128 && swizzle_bytes != 64) return set_error(IH_ERR_ARG, "unsupported swizzle %d", swizzle_bytes);
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base;
  key.rank = rank;
  key.swz = swizzle_bytes;
  for (int i = 0; i < rank; ++i) {
    key.dims[i] = dims[i];
    key.box[i] = box[i];
    if (i + 1 < rank) key.strides[i] = strides_bytes[i];
  }
  std::string k(reinterpret_cast<const char*>(&key), sizeof(key));
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    auto it = g_tmap_cache.find(k);
    if (it != g_tmap_cache.end()) {
      *out = it->second;
      return 0;
    }
  }
  PFN_cuTensorMapEncodeTiled enc = get_encode_fn();
  if (!enc) return set_error(IH_ERR_TMAP, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error(IH_ERR_ALIGN, "tensor base not 16B aligned");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i + 1 < rank) {
      gstr[i] = strides_bytes[i];
      if (gstr[i] % 16 != 0) return set_error(IH_ERR_ALIGN, "tensor stride %llu not a multiple of 16 bytes",
                                              (unsigned long long)gstr[i]);
    }
  }
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstr, bx, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(IH_ERR_TMAP, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d)", (int)r, rank);
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    if (g_tmap_cache.size() > 65536) g_tmap_cache.clear();
    g_tmap_cache.emplace(std::move(k), m);
  }
  *out = m;
  return 0;
}

int num_sms() {
  static int n = [] {
    int dev = 0, v = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v > 0 ? v : 132;
  }();
  return n;
}

bool pdl_enabled() {
  static bool on = [] {
    const char* e = getenv("IH_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

bool first_launch_of(const void* kern) {
  static std::mutex mu;
  static std::unordered_map<const void*, bool> seen;
  std::lock_guard<std::mutex> lk(mu);
  return seen.emplace(kern, true).second;
}

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

}  // namespace ih

extern "C" {
const char* ih_last_error(void) { return ih::g_err; }
int ih_version(void) { return IH_API_VERSION; }
long long ih_launch_count(void) { return ih::g_launches.load(); }
void ih_launch_count_reset(void) { ih::g_launches.store(0); }
}
