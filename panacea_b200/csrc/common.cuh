// Host-side helpers shared by all translation units: error reporting across the C ABI and TMA
// tensor-map construction (driver entry point resolved at run time, so the library links without libcuda).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <cuda.h>
#include <cuda_runtime.h>

struct pn_attn_args;      // include/panacea_b200.h

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
// blocks of `threads` for a grid-stride loop over `total` items: one item per thread, at most 16 blocks per SM
int stride_grid(size_t total, int threads = 256);
// opt in to `bytes` of dynamic shared memory for `func` on the current device (once per device and size);
// `max_carveout` also asks for the largest shared-memory carveout, for kernels that plan on several CTAs per SM
int ensure_dyn_smem(const void* func, size_t bytes, bool max_carveout = false);

// Parity-mode attention (attn_f32.cu): fp32 q/k/v, fp32 math on CUDA cores, the output written as the operand of the
// to_out GEMM in operand_mode. pn_attention / pn_attention_temporal / pn_attention_causal call these for the fp32 modes.
int attention_f32(const pn_attn_args* a, int operand_mode, void* stream);
int attention_temporal_f32(const float* q, const float* k, const float* v, void* out, int64_t batch, int64_t T, int64_t pixels,
                           int32_t heads, int32_t head_dim, int64_t ld, int64_t out_ld, float scale, int operand_mode,
                           void* stream);
int attention_causal_f32(const float* q, const float* k, const float* v, void* out, int64_t batch, int64_t L, int32_t heads,
                         int32_t head_dim, int64_t ld, int64_t out_ld, float scale, int operand_mode, void* stream);

}  // namespace pn
