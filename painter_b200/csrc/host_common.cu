#include "host_common.h"

#include <stdarg.h>
#include <stdlib.h>
#include <mutex>

#include "../../include/painter_b200.h"

namespace pk {

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static std::atomic<int> g_sm_budget{0};

// SM count of the CURRENT device (cached per device ordinal), capped by pk_set_sm_budget.  Without a device (host-only
// schedule queries) the H100 SXM's 132 SMs.
int sm_count() {
  static std::atomic<int> cache[64];
  int dev = 0;
  cudaGetDevice(&dev);
  int n = (dev >= 0 && dev < 64) ? cache[dev].load(std::memory_order_relaxed) : 0;
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
    if (dev >= 0 && dev < 64) cache[dev].store(n, std::memory_order_relaxed);
  }
  const int b = g_sm_budget.load(std::memory_order_relaxed);
  if (b > 0 && b < n) n = b;
  return n < 1 ? 1 : n;
}

static std::atomic<int> g_pdl{-1};
bool pdl_enabled() {
  int v = g_pdl.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("PK_PDL");
    v = (e != nullptr && e[0] == '0') ? 0 : 1;
    g_pdl.store(v, std::memory_order_relaxed);
  }
  return v != 0;
}
int set_pdl(int on) { return g_pdl.exchange(on ? 1 : 0); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

bool make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return false;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank),
                   const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,..] stride0 %llu box [%u,%u,..] base %p",
              static_cast<int>(r), rank, (unsigned long long)dims[0],
              (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 1 ? strides_bytes[0] : 0), box[0], rank > 1 ? box[1] : 0,
              base);
    return false;
  }
  return true;
}

}  // namespace pk

extern "C" {
int pk_version(void) { return 100; }
const char* pk_last_error(void) { return pk::g_err; }
long long pk_launch_count(void) { return pk::g_launches.load(); }
int pk_set_sm_budget(int n) { return pk::g_sm_budget.exchange(n < 0 ? 0 : n); }
int pk_set_pdl(int on) { return pk::set_pdl(on); }
}
