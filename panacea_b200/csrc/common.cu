#include "common.cuh"
#include "../../include/panacea_b200.h"

#include <cstdarg>
#include <mutex>
#include <unordered_map>

namespace pn {

static thread_local std::string g_last_error;

void set_last_error(const std::string& msg) { g_last_error = msg; }

int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
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

static std::mutex g_tmap32_mu;
struct Tmap32Key {
  const void* ptr; uint64_t cols, rows, ld; uint32_t box_rows, pad;
  bool operator==(const Tmap32Key& o) const { return std::memcmp(this, &o, sizeof(Tmap32Key)) == 0; }
};
struct Tmap32Hash {
  size_t operator()(const Tmap32Key& k) const {
    const unsigned char* w = reinterpret_cast<const unsigned char*>(&k);
    size_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(Tmap32Key); ++i) h = (h ^ w[i]) * 1099511628211ull;
    return h;
  }
};
static std::unordered_map<Tmap32Key, CUtensorMap, Tmap32Hash> g_tmap32_cache;

int cached_tmap_f32_2d(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t ld_elems, uint32_t box_rows) {
  Tmap32Key key;
  std::memset(&key, 0, sizeof(key));
  key.ptr = base; key.cols = cols; key.rows = rows; key.ld = ld_elems; key.box_rows = box_rows;
  {
    std::lock_guard<std::mutex> lk(g_tmap32_mu);
    auto it = g_tmap32_cache.find(key);
    if (it != g_tmap32_cache.end()) { *out = it->second; return PN_OK; }
  }
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return fail(PN_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld_elems * 4};
  cuuint32_t bdim[2] = {32u, box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstr, bdim, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(PN_ERR_CUDA, "cuTensorMapEncodeTiled(fp32) failed (%d): cols=%llu rows=%llu ld=%llu", (int)r,
                (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)ld_elems);
  std::lock_guard<std::mutex> lk(g_tmap32_mu);
  if (g_tmap32_cache.size() > 65536) g_tmap32_cache.clear();
  g_tmap32_cache.emplace(key, *out);
  return PN_OK;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_elems, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return fail(PN_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  if (rank < 1 || rank > 5) return fail(PN_ERR_INVALID, "tensor map rank %d out of range", rank);
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_elems[i] * 2;  // bytes
  CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
  if (swizzle_bytes == 32) sw = CU_TENSOR_MAP_SWIZZLE_32B;
  else if (swizzle_bytes == 64) sw = CU_TENSOR_MAP_SWIZZLE_64B;
  else if (swizzle_bytes == 128) sw = CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return fail(PN_ERR_CUDA,
                "cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u,%u] "
                "stride0=%llu",
                (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
                (unsigned long long)(rank > 4 ? dims[4] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0,
                rank > 3 ? box[3] : 0, rank > 4 ? box[4] : 0, (unsigned long long)(rank > 1 ? strides_elems[0] : 0));
  }
  return PN_OK;
}

struct TmapKey {
  const void* ptr;
  uint64_t d[5], s[4];
  uint32_t b[5];
  int rank, swizzle;
  bool operator==(const TmapKey& o) const { return std::memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    const unsigned char* w = reinterpret_cast<const unsigned char*>(&k);
    size_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(TmapKey); ++i) h = (h ^ w[i]) * 1099511628211ull;
    return h;
  }
};
static std::mutex g_tmap_mu;
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;

// Tensor maps are pure functions of (pointer, geometry); encoding costs microseconds on the host, so they
// are memoised. Buffers of the denoising loop are allocated once, so the cache stays small.
int cached_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_elems, const uint32_t* box, int swizzle_bytes) {
  TmapKey key;
  std::memset(&key, 0, sizeof(key));
  key.ptr = base;
  key.rank = rank;
  key.swizzle = swizzle_bytes;
  for (int i = 0; i < rank; ++i) { key.d[i] = dims[i]; key.b[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) key.s[i] = strides_elems[i];
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) { *out = it->second; return PN_OK; }
  }
  int rc = make_tmap_bf16(out, base, rank, dims, strides_elems, box, swizzle_bytes);
  if (rc != PN_OK) return rc;
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  if (g_tmap_cache.size() > 65536) g_tmap_cache.clear();
  g_tmap_cache.emplace(key, *out);
  return PN_OK;
}

// Per-device caches: the SM count and the opt-in dynamic shared-memory limit of a kernel are properties of the
// CURRENT device / context, so both are keyed by the device ordinal (a process may drive several GPUs).
static std::mutex g_dev_mu;
static int g_sm_count[64];
static std::unordered_map<unsigned long long, size_t> g_smem_attr;   // (func address ^ device << 56) -> bytes set

int sm_count() {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  std::lock_guard<std::mutex> lk(g_dev_mu);
  if (g_sm_count[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    g_sm_count[dev] = n > 0 ? n : 132;
  }
  return g_sm_count[dev];
}

int stride_grid(size_t total, int threads) {
  size_t g = (total + threads - 1) / threads;
  const size_t cap = (size_t)16 * sm_count();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

int ensure_dyn_smem(const void* func, size_t bytes, bool max_carveout) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long key = (unsigned long long)reinterpret_cast<uintptr_t>(func) ^ ((unsigned long long)(dev & 0xff) << 56);
  std::lock_guard<std::mutex> lk(g_dev_mu);
  auto it = g_smem_attr.find(key);
  if (it != g_smem_attr.end() && it->second >= bytes) return PN_OK;
  PN_CHECK_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  if (max_carveout)
    PN_CHECK_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
  g_smem_attr[key] = bytes;
  return PN_OK;
}

}  // namespace pn

extern "C" const char* pn_last_error(void) { return pn::g_last_error.c_str(); }
extern "C" int pn_abi_version(void) { return PN_ABI_VERSION; }
