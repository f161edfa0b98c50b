// Host-side helpers shared by all translation units: error reporting across the C ABI and TMA
// tensor-map construction (driver entry point resolved at run time, so the library links without libcuda).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <cuda.h>
#include <cuda_runtime.h>

namespace pn {

// Error codes returned over the C ABI (see include/panacea_b200.h).
enum : int { PN_OK = 0, PN_ERR_INVALID = -1, PN_ERR_CUDA = -2, PN_ERR_UNSUPPORTED = -3 };

void set_last_error(const std::string& msg);
int fail(int code, const char* fmt, ...);

#define PN_CHECK_CUDA(expr)                                                                       \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return ::pn::fail(::pn::PN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                        __FILE__, __LINE__);                                                      \
  } while (0)

#define PN_REQUIRE(cond, ...)                                    \
  do {                                                           \
    if (!(cond)) return ::pn::fail(::pn::PN_ERR_INVALID, __VA_ARGS__); \
  } while (0)

// Encode a tiled bf16 tensor map. dims/strides are innermost-first; strides in ELEMENTS for dims 1..rank-1
// (dim 0 is contiguous). box is innermost-first. swizzle_bytes in {0,32,64,128}.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_elems, const uint32_t* box, int swizzle_bytes);

// fp32 2-D [rows, ld] map with a {32 floats, box_rows} box, 128B swizzle (streaming GEMM epilogue)
int cached_tmap_f32_2d(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t ld_elems, uint32_t box_rows);

int cached_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_elems, const uint32_t* box, int swizzle_bytes);

int sm_count();                                          // of the current device
// opt in to `bytes` of dynamic shared memory for `func` on the current device (once per device and size);
// `max_carveout` also asks for the largest shared-memory carveout, for kernels that plan on several CTAs per SM
int ensure_dyn_smem(const void* func, size_t bytes, bool max_carveout = false);

// PN_PDL=1 enables programmatic dependent launch (off by default: measured no gain on the captured graph)
bool pdl_enabled();

// Launch with programmatic stream serialization (and optionally a thread-block cluster): the kernel must call
// pdl_prologue_done() (ptx.cuh) before its first global-memory access.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x,
                                 Args&&... args) {
  cudaLaunchConfig_t cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[n].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  ++n;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = (unsigned)cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace pn
