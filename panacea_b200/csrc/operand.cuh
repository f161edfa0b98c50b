// How a producer kernel writes the A operand of the GEMM that follows it.
//
//  PN_OP_BF16   : bf16 [rows, C]                     (the fast path: bf16 products, fp32 accumulation)
//  PN_OP_SPLIT3 : bf16 [rows, 3C] = [hi | lo | hi]   (parity mode) with hi = bf16(v), lo = bf16(v - hi).
//                 Against weights packed as [W_hi | W_hi | W_lo] per tap the SAME wgmma GEMM kernel computes
//                 hi*W_hi + lo*W_hi + hi*W_lo = v*W up to the dropped lo*W_lo term (2^-18 relative): fp32-class
//                 products on the bf16 tensor pipe by K-concatenation, no kernel change.
//  PN_OP_F32    : fp32 [rows, C]                     (consumers that are CUDA-core kernels in parity mode)
//  PN_OP_SPLIT3_B: bf16 [rows, 3C] = [hi | hi | lo]  (parity mode, the WEIGHT form of ops.split3 made on the device: the
//                 B operand of a GEMM whose two factors are both activations, the VAE mid-block attention's S = q k^T
//                 and O = P v). Only pn_cast_operand writes it; PN_DISPATCH_OP does not instantiate it.
#pragma once
#include "ptx.cuh"

namespace pn {

enum : int { PN_OP_BF16 = 0, PN_OP_SPLIT3 = 1, PN_OP_F32 = 2, PN_OP_SPLIT3_B = 3 };

__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat16 ha = __float2bfloat16_rn(a), hb = __float2bfloat16_rn(b);
  const float ra = a - __bfloat162float(ha), rb = b - __bfloat162float(hb);      // exact in fp32
  hi = (uint32_t)__bfloat16_as_ushort(ha) | ((uint32_t)__bfloat16_as_ushort(hb) << 16);
  lo = pack_bf16x2(ra, rb);
}

// element size of the stored operand row in units of its own dtype
template <int OP>
__device__ __forceinline__ constexpr int op_row_mult() { return OP == PN_OP_SPLIT3 || OP == PN_OP_SPLIT3_B ? 3 : 1; }

// 8 consecutive channels [col, col+8) of row `row` of a [rows, C] operand
template <int OP>
__device__ __forceinline__ void store_op8(void* base, size_t row, int C, int col, const float (&v)[8]) {
  if (OP == PN_OP_F32) {
    float* p = reinterpret_cast<float*>(base) + row * (size_t)C + col;
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
  } else if (OP == PN_OP_BF16) {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)C + col;
    *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                                              pack_bf16x2(v[6], v[7]));
  } else if (OP == PN_OP_SPLIT3_B) {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)(3 * C) + col;
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) split_bf16x2(v[2 * i], v[2 * i + 1], h[i], l[i]);
    const uint4 hv = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(p) = hv;
    *reinterpret_cast<uint4*>(p + C) = hv;
    *reinterpret_cast<uint4*>(p + 2 * C) = make_uint4(l[0], l[1], l[2], l[3]);
  } else {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)(3 * C) + col;
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) split_bf16x2(v[2 * i], v[2 * i + 1], h[i], l[i]);
    const uint4 hv = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(p) = hv;
    *reinterpret_cast<uint4*>(p + C) = make_uint4(l[0], l[1], l[2], l[3]);
    *reinterpret_cast<uint4*>(p + 2 * C) = hv;
  }
}

template <int OP>
__device__ __forceinline__ void store_op4(void* base, size_t row, int C, int col, const float (&v)[4]) {
  if (OP == PN_OP_F32) {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + row * (size_t)C + col) = make_float4(v[0], v[1], v[2], v[3]);
  } else if (OP == PN_OP_BF16) {
    *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)C + col) =
        make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]));
  } else if (OP == PN_OP_SPLIT3_B) {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)(3 * C) + col;
    uint32_t h0, h1, l0, l1;
    split_bf16x2(v[0], v[1], h0, l0);
    split_bf16x2(v[2], v[3], h1, l1);
    *reinterpret_cast<uint2*>(p) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(p + C) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(p + 2 * C) = make_uint2(l0, l1);
  } else {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)(3 * C) + col;
    uint32_t h0, h1, l0, l1;
    split_bf16x2(v[0], v[1], h0, l0);
    split_bf16x2(v[2], v[3], h1, l1);
    *reinterpret_cast<uint2*>(p) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(p + C) = make_uint2(l0, l1);
    *reinterpret_cast<uint2*>(p + 2 * C) = make_uint2(h0, h1);
  }
}

template <int OP>
__device__ __forceinline__ void store_op2(void* base, size_t row, int C, int col, float a, float b) {
  if (OP == PN_OP_F32) {
    *reinterpret_cast<float2*>(reinterpret_cast<float*>(base) + row * (size_t)C + col) = make_float2(a, b);
  } else if (OP == PN_OP_BF16) {
    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)C + col) = pack_bf16x2(a, b);
  } else if (OP == PN_OP_SPLIT3_B) {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)(3 * C) + col;
    uint32_t h, l;
    split_bf16x2(a, b, h, l);
    *reinterpret_cast<uint32_t*>(p) = h;
    *reinterpret_cast<uint32_t*>(p + C) = h;
    *reinterpret_cast<uint32_t*>(p + 2 * C) = l;
  } else {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)(3 * C) + col;
    uint32_t h, l;
    split_bf16x2(a, b, h, l);
    *reinterpret_cast<uint32_t*>(p) = h;
    *reinterpret_cast<uint32_t*>(p + C) = l;
    *reinterpret_cast<uint32_t*>(p + 2 * C) = h;
  }
}

// dispatch a kernel launch expression on a run-time operand mode (BF16 / SPLIT3 / F32). Any other mode, SPLIT3_B
// included, makes the enclosing entry point return an error: a producer that forgets its own operand_mode check still
// never writes an operand of the wrong size.
#define PN_DISPATCH_OP(mode, ...)                                                           \
  do {                                                                                      \
    if ((mode) == ::pn::PN_OP_BF16) { constexpr int OP = ::pn::PN_OP_BF16; __VA_ARGS__; }   \
    else if ((mode) == ::pn::PN_OP_SPLIT3) { constexpr int OP = ::pn::PN_OP_SPLIT3; __VA_ARGS__; } \
    else if ((mode) == ::pn::PN_OP_F32) { constexpr int OP = ::pn::PN_OP_F32; __VA_ARGS__; } \
    else return ::pn::fail(::pn::PN_ERR_INVALID, "operand_mode %d is not a producer store mode", (int)(mode)); \
  } while (0)

}  // namespace pn
