// Parameters and per-element epilogue arithmetic shared by the two wgmma GEMM kernels (gemm_tc.cu, gemm_ws.cu). Both
// kernels call these helpers for every output element, so an element sees the same operations in the same order on
// either path: bias or the folded LayerNorm, then the row vector, the residual, the second residual (each `epi_add`);
// GEGLU through geglu_f32; the per-half row statistics summed in column-block order and reduced over the quad.
#pragma once
#include "ptx.cuh"

namespace pn {

struct GemmParams {
  CUtensorMap mapA;
  CUtensorMap mapB;
  // geometry of the A tensor / output rows
  int NB, H, W;
  int tw, th, tn;             // tile box extents, tw*th*tn == 128
  int tiles_w, tiles_h, tiles_n, tiles_col;
  int kc_per_tap;             // C / 64
  int taps_h, taps_w, pad_h, pad_w;
  int N;                      // GEMM N (weight rows)
  // epilogue
  void* out;
  const float* bias;
  const float* rowvec;
  const void* residual;
  const float* residual2;
  long long ldo, ldr, ldr2, ldv;
  int rows_per_group, n_groups;
  // LayerNorm folded into the GEMMs around the bf16 token stream (attention.py:726-747: x + attn(norm(x))):
  //  * a PRODUCER of the stream also emits per-row partial sums (sum, sum of squares) of the values it stores:
  //    ln_stats_out[row][tile_col * 2 + half][2] (ln_parts_out = 2 * tiles_col, half = which half of the tile's columns);
  //  * a CONSUMER multiplies the UN-normalised stream by W' = W diag(gamma) and finishes the LayerNorm in its
  //    epilogue: out = rstd_m * (acc - mean_m * s_n) + t_n, s_n = sum_k W'[n,k], t_n = sum_k beta_k W[n,k] (+ bias,
  //    passed as `bias`), mean/rstd from the ln_parts_in partial sums of row m.
  const float* ln_stats_in;
  const float* ln_colsum;
  float* ln_stats_out;
  int ln_parts_in, ln_parts_out;
  float ln_inv_dim, ln_eps;
  int res_bf16;                // the residual is bf16 (bf16 token stream of the transformer blocks), bf16 output only
};

// gemm_ws.cu: the persistent weight-stationary kernel for a 1x1 GEMM over `rows` dense rows (row stride `row_stride`
// elements) with C <= 320 and N % 160 == 0; `p` holds mapB (160-row boxes) and the epilogue fields.
int launch_gemm_ws(GemmParams& p, int mode, const void* A, long long rows, long long row_stride, int C, cudaStream_t stream);

// Folded LayerNorm of output row `row`: out = a * acc + b * s_n + t_n, from the row's ln_parts_in partial sums.
__device__ __forceinline__ void ln_row_coeffs(const GemmParams& p, long long row, float& a, float& b) {
  float sm = 0.f, sq = 0.f;
  const float2* st = reinterpret_cast<const float2*>(p.ln_stats_in) + row * p.ln_parts_in;
  for (int q = 0; q < p.ln_parts_in; ++q) { const float2 t2 = __ldg(st + q); sm += t2.x; sq += t2.y; }
  const float mu = sm * p.ln_inv_dim;
  const float rstd = rsqrtf(fmaxf(sq * p.ln_inv_dim - mu * mu, 0.f) + p.ln_eps);
  a = rstd;
  b = -rstd * mu;
}

// The first term of a pair of adjacent outputs: the folded LayerNorm (a, b of the row, s2 = column sums, b2 = bias)
// when `ln`, else the bias b2 (zeros without a bias).
__device__ __forceinline__ void epi_bias(float& v0, float& v1, float2 b2, float2 s2, bool ln, float a, float b) {
  if (ln) {
    v0 = fmaf(a, v0, fmaf(b, s2.x, b2.x));
    v1 = fmaf(a, v1, fmaf(b, s2.y, b2.y));
  } else {
    v0 += b2.x; v1 += b2.y;
  }
}

// every later term (row vector, residual, second residual) of a pair of adjacent outputs
__device__ __forceinline__ void epi_add(float& v0, float& v1, float2 t) { v0 += t.x; v1 += t.y; }

// row statistics of the fp32 values of a bf16 output pair (their bf16 rounding, which the consumer's MMA reads,
// perturbs mean / variance by < 2^-9 / sqrt(C))
__device__ __forceinline__ void row_stats_add(float& s, float& q, float v0, float v1) {
  s += v0 + v1;
  q = fmaf(v0, v0, fmaf(v1, v1, q));
}

// sum over the four lanes of a quad, which hold the columns of one accumulator row
__device__ __forceinline__ float quad_sum(float s) {
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  return s;
}

}  // namespace pn
