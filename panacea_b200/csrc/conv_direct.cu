// Direct 3x3 convolution on CUDA cores for the layers whose channel counts cannot feed a 64-wide wgmma K block:
// the UNet/ControlNet stems (8 -> 320, openaimodel.py:977), the output head (320 -> 4, openaimodel.py:1251) and the
// BEV hint stem (19 -> 16 -> 16 -> 32 -> 32 -> 96 -> 96 -> 256 -> 320 with strides 1,1,2,1,2,1,2,1,
// controlmodel.py:43-59). The hint stem is step-invariant and runs once per sample; stem and head are <0.02 % of
// the step's FLOPs.
//
// Channels-last fp32 in, fp32 (or bf16) out. One thread = one output pixel x 16 output channels; the weight
// slice of the current tap ([Cin][16]) is staged in shared memory and broadcast.
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

constexpr int CD_COUT_TILE = 16;
constexpr int CD_THREADS = 128;

template <typename TIn>
__device__ __forceinline__ float4 load4(const TIn* p);
template <>
__device__ __forceinline__ float4 load4<float>(const float* p) { return *reinterpret_cast<const float4*>(p); }
template <>
__device__ __forceinline__ float4 load4<__nv_bfloat16>(const __nv_bfloat16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

// weights: fp32 [9][Cin][Cout_pad] (tap-major, cout innermost, Cout_pad multiple of 16)
template <typename TIn>
__global__ void __launch_bounds__(CD_THREADS) conv3x3_direct_kernel(const TIn* __restrict__ x, const float* __restrict__ w,
                                                                    const float* __restrict__ bias, const float* __restrict__ addend,
                                                                    float* __restrict__ y_f32, __nv_bfloat16* __restrict__ y_bf16,
                                                                    int F, int H, int W, int Cin, int Cout, int Cout_pad, int Ho,
                                                                    int Wo, int stride, int act_silu) {
  extern __shared__ float sw[];  // [Cin][16]
  const int co0 = blockIdx.y * CD_COUT_TILE;
  const size_t pix = (size_t)blockIdx.x * CD_THREADS + threadIdx.x;
  const size_t npix = (size_t)F * Ho * Wo;
  const bool active = pix < npix;
  int f = 0, oy = 0, ox = 0;
  if (active) {
    ox = (int)(pix % Wo);
    oy = (int)((pix / Wo) % Ho);
    f = (int)(pix / ((size_t)Wo * Ho));
  }
  float acc[CD_COUT_TILE];
#pragma unroll
  for (int j = 0; j < CD_COUT_TILE; ++j) acc[j] = 0.f;
  for (int tap = 0; tap < 9; ++tap) {
    __syncthreads();
    for (int i = threadIdx.x; i < Cin * CD_COUT_TILE; i += CD_THREADS) {
      const int ci = i / CD_COUT_TILE, j = i - ci * CD_COUT_TILE;
      sw[i] = w[((size_t)tap * Cin + ci) * Cout_pad + co0 + j];
    }
    __syncthreads();
    const int iy = oy * stride - 1 + tap / 3, ix = ox * stride - 1 + tap % 3;
    if (active && iy >= 0 && iy < H && ix >= 0 && ix < W) {
      const TIn* src = x + (((size_t)f * H + iy) * W + ix) * Cin;
      for (int ci = 0; ci < Cin; ci += 4) {
        const float4 v = load4<TIn>(src + ci);
        const float xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float4* wr = reinterpret_cast<const float4*>(sw + (ci + k) * CD_COUT_TILE);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 ww = wr[q];
            acc[q * 4 + 0] += xv[k] * ww.x;
            acc[q * 4 + 1] += xv[k] * ww.y;
            acc[q * 4 + 2] += xv[k] * ww.z;
            acc[q * 4 + 3] += xv[k] * ww.w;
          }
        }
      }
    }
  }
  if (!active) return;
  const size_t obase = pix * Cout + co0;
#pragma unroll
  for (int j = 0; j < CD_COUT_TILE; ++j) {
    if (co0 + j < Cout) {
      float v = acc[j] + (bias ? bias[co0 + j] : 0.f);
      if (act_silu) v = silu(v);
      if (addend) v += addend[obase + j];
      if (y_f32) y_f32[obase + j] = v;
      if (y_bf16) y_bf16[obase + j] = __float2bfloat16(v);
    }
  }
}

}  // namespace pn

using namespace pn;

extern "C" int pn_conv3x3_direct(const void* x, int x_is_bf16, const float* w_packed, const float* bias,
                                 const float* addend, float* y_f32, void* y_bf16, int64_t frames, int64_t H, int64_t W,
                                 int64_t Cin, int64_t Cout, int64_t Cout_pad, int stride, int act_silu, void* stream_v) {
  PN_REQUIRE(x && w_packed && (y_f32 || y_bf16), "pn_conv3x3_direct: null pointer");
  PN_REQUIRE(Cin > 0 && Cin % 4 == 0 && Cout > 0 && Cout_pad % CD_COUT_TILE == 0 && Cout_pad >= Cout,
             "pn_conv3x3_direct: Cin=%lld (must be %%4) Cout=%lld Cout_pad=%lld", (long long)Cin, (long long)Cout,
             (long long)Cout_pad);
  PN_REQUIRE(stride == 1 || stride == 2, "pn_conv3x3_direct: stride must be 1 or 2");
  PN_REQUIRE(frames > 0 && H > 0 && W > 0, "pn_conv3x3_direct: empty input");
  const int Ho = (int)((H + 2 - 3) / stride + 1), Wo = (int)((W + 2 - 3) / stride + 1);
  const size_t npix = (size_t)frames * Ho * Wo;
  dim3 grid((unsigned)((npix + CD_THREADS - 1) / CD_THREADS), (unsigned)(Cout_pad / CD_COUT_TILE));
  const size_t smem = (size_t)Cin * CD_COUT_TILE * sizeof(float);
  PN_REQUIRE(smem <= 48 * 1024, "pn_conv3x3_direct: Cin=%lld too large for the direct path", (long long)Cin);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (x_is_bf16)
    conv3x3_direct_kernel<__nv_bfloat16><<<grid, CD_THREADS, smem, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(x), w_packed, bias, addend, y_f32, reinterpret_cast<__nv_bfloat16*>(y_bf16),
        (int)frames, (int)H, (int)W, (int)Cin, (int)Cout, (int)Cout_pad, Ho, Wo, stride, act_silu);
  else
    conv3x3_direct_kernel<float><<<grid, CD_THREADS, smem, st>>>(
        reinterpret_cast<const float*>(x), w_packed, bias, addend, y_f32, reinterpret_cast<__nv_bfloat16*>(y_bf16),
        (int)frames, (int)H, (int)W, (int)Cin, (int)Cout, (int)Cout_pad, Ho, Wo, stride, act_silu);
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}
