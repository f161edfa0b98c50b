// How a producer kernel writes the A operand of the GEMM that follows it: in one of the layouts of pn_operand_mode
// (include/panacea_b200.h), chosen by the kernel's OP template argument. In the split forms the GEMM drops the
// lo*W_lo term of (hi + lo)(W_hi + W_lo): it is 2^-18 of the product, below fp32-class accuracy.
#pragma once
#include <type_traits>
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat16 ha = __float2bfloat16_rn(a), hb = __float2bfloat16_rn(b);
  const float ra = a - __bfloat162float(ha), rb = b - __bfloat162float(hb);      // exact in fp32
  hi = (uint32_t)__bfloat16_as_ushort(ha) | ((uint32_t)__bfloat16_as_ushort(hb) << 16);
  lo = pack_bf16x2(ra, rb);
}

// N consecutive channels as one vector access: the bf16 vector of N values (`pack`, or `words` from N / 2 packed pairs),
// and the fp32 vector (N <= 4; 8 channels are two float4 accesses). split() makes the hi and lo words of the split
// forms; it is a loop for 8 channels and written out for 2 and 4 because the compiler schedules the callers differently
// for the two forms, and these are the ones the producers' SASS was tuned with.
template <int N> struct op_vec;
template <> struct op_vec<2> {
  using bf16 = uint32_t;
  using f32 = float2;
  static __device__ __forceinline__ bf16 words(const uint32_t* w) { return w[0]; }
  static __device__ __forceinline__ bf16 pack(const float* v) { return pack_bf16x2(v[0], v[1]); }
  static __device__ __forceinline__ f32 floats(const float* v) { return make_float2(v[0], v[1]); }
  static __device__ __forceinline__ void split(const float* v, uint32_t* hi, uint32_t* lo) {
    split_bf16x2(v[0], v[1], hi[0], lo[0]);
  }
};
template <> struct op_vec<4> {
  using bf16 = uint2;
  using f32 = float4;
  static __device__ __forceinline__ bf16 words(const uint32_t* w) { return make_uint2(w[0], w[1]); }
  static __device__ __forceinline__ bf16 pack(const float* v) {
    return make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]));
  }
  static __device__ __forceinline__ f32 floats(const float* v) { return make_float4(v[0], v[1], v[2], v[3]); }
  static __device__ __forceinline__ void split(const float* v, uint32_t* hi, uint32_t* lo) {
    split_bf16x2(v[0], v[1], hi[0], lo[0]);
    split_bf16x2(v[2], v[3], hi[1], lo[1]);
  }
};
template <> struct op_vec<8> {
  using bf16 = uint4;
  static __device__ __forceinline__ bf16 words(const uint32_t* w) { return make_uint4(w[0], w[1], w[2], w[3]); }
  static __device__ __forceinline__ bf16 pack(const float* v) {
    return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
  }
  static __device__ __forceinline__ void split(const float* v, uint32_t* hi, uint32_t* lo) {
#pragma unroll
    for (int i = 0; i < 4; ++i) split_bf16x2(v[2 * i], v[2 * i + 1], hi[i], lo[i]);
  }
};

// N = 2, 4 or 8 consecutive channels [col, col + N) of row `row` of a [rows, C] operand
template <int OP, int N>
__device__ __forceinline__ void store_op(void* base, size_t row, int C, int col, const float (&v)[N]) {
  using V = op_vec<N>;
  using B = typename V::bf16;
  if constexpr (OP == PN_OPERAND_BF16) {
    *reinterpret_cast<B*>(reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)C + col) = V::pack(v);
  } else if constexpr (OP == PN_OPERAND_F32) {
    using F = op_vec<N < 4 ? N : 4>;
    using T = typename F::f32;
    *reinterpret_cast<T*>(reinterpret_cast<float*>(base) + row * (size_t)C + col) = F::floats(v);
    if constexpr (N == 8) *reinterpret_cast<T*>(reinterpret_cast<float*>(base) + row * (size_t)C + col + 4) = F::floats(v + 4);
  } else {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + row * (size_t)(3 * C) + col;
    uint32_t hi[N / 2], lo[N / 2];
    V::split(v, hi, lo);
    constexpr bool a_form = OP == PN_OPERAND_SPLIT3;
    *reinterpret_cast<B*>(p) = V::words(hi);
    *reinterpret_cast<B*>(p + C) = V::words(a_form ? lo : hi);
    *reinterpret_cast<B*>(p + 2 * C) = V::words(a_form ? hi : lo);
  }
}

// The operand modes an entry point accepts. PN_OPERAND_MODES(Name, mode, "entry", modes...) declares them as the type
// Name and returns PN_ERR_INVALID for any other mode; an entry point states it before it does any work.
// PN_DISPATCH_OP(Name, mode, launch) then instantiates the launch expression, which names the mode OP, for exactly
// these modes and runs the one that matches.
template <int... MODES>
struct OperandModes {
  static constexpr bool has(int mode) { return ((mode == MODES) || ...); }
  template <typename F>
  static void dispatch(int mode, F&& launch) {
    ((mode == MODES ? launch(std::integral_constant<int, MODES>{}) : void()), ...);
  }
};

#define PN_OPERAND_MODES(Name, mode, entry, ...)    \
  using Name = ::pn::OperandModes<__VA_ARGS__>;     \
  PN_REQUIRE(Name::has(mode), entry ": operand_mode %d unsupported", (int)(mode))

#define PN_DISPATCH_OP(MODES, mode, ...) \
  MODES::dispatch((mode), [&](auto op_) { constexpr int OP = decltype(op_)::value; __VA_ARGS__; })

}  // namespace pn
