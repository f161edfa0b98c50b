// Parameters and epilogue arithmetic shared by the two wgmma GEMM kernels (gemm_tc.cu, gemm_ws.cu). Both kernels call
// these helpers for every output element, so an element sees the same operations in the same order on either path: bias
// or the folded LayerNorm, then the row vector, the residual, the second residual (each `epi_add`); GEGLU through
// geglu_add and geglu_out; the per-half row statistics summed in column-block order and reduced over the quad.
#pragma once
#include "ptx.cuh"

namespace pn {

// the epilogue of a kernel instantiation: MODE of gemm_tc_kernel / gemm_ws_kernel (an int, so symbol names keep 0/1/2)
enum EpiMode : int {
  EPI_F32 = 0,     // fp32 store (+ fp32 residual, + second fp32 residual)
  EPI_BF16 = 1,    // bf16 store (+ fp32 or bf16 residual, LayerNorm fold / row statistics)
  EPI_GEGLU = 2    // bf16 store of N/2 columns: value * gelu_erf(gate)
};

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
int launch_gemm_ws(GemmParams& p, EpiMode mode, const void* A, long long rows, long long row_stride, int C, cudaStream_t stream);

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

// rv[h] = the row vector of row grow[h]'s group from column n_base on (p.rowvec without one or for grow[h] < 0)
__device__ __forceinline__ void rowvec_rows(const GemmParams& p, const long long (&grow)[2], int n_base, const float* (&rv)[2]) {
  rv[0] = rv[1] = p.rowvec;
  if (p.rowvec == nullptr) return;
#pragma unroll
  for (int h = 0; h < 2; ++h)
    if (grow[h] >= 0) rv[h] += (long long)((grow[h] / p.rows_per_group) % p.n_groups) * p.ldv + n_base;
}

// GEGLU: each 32 columns hold the values of 16 outputs in blocks j, j + 1 (j % 4 == 0) and their gates in j + 2, j + 3
// (ops.geglu_pack). Adds one term (bias, then row vector) to value block j (j % 4 < 2) of row h and gate block j + 2.
__device__ __forceinline__ void geglu_add(float* acc, int j, int h, float2 value, float2 gate) {
  epi_add(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], value);
  epi_add(acc[4 * (j + 2) + 2 * h], acc[4 * (j + 2) + 2 * h + 1], gate);
}

// the bf16 output pair of value block j of row h: value * gelu_erf(gate) (reference GEGLU: attention.py:97-99)
__device__ __forceinline__ uint32_t geglu_out(const float* acc, int j, int h) {
  return pack_bf16x2(geglu_f32(acc[4 * j + 2 * h], acc[4 * (j + 2) + 2 * h]),
                     geglu_f32(acc[4 * j + 2 * h + 1], acc[4 * (j + 2) + 2 * h + 1]));
}

// the first of the two output columns of value block j (j % 4 < 2), within the tile's BN / 2 output columns
__device__ __forceinline__ int geglu_out_col(int j, int quad) { return (j >> 2) * 16 + (j & 1) * 8 + 2 * quad; }

// Row statistics of a bf16 output tile of NJ column blocks: s[h][half], q[h][half] sum the stored fp32 values of row h
// and their squares over each half of the columns (their bf16 rounding perturbs mean / variance by < 2^-9 / sqrt(C)).
template <int NJ>
__device__ __forceinline__ void row_stats_add(float (&s)[2][2], float (&q)[2][2], int h, int j, float v0, float v1) {
  const int hf = j < NJ / 2 ? 0 : 1;
  s[h][hf] += v0 + v1;
  q[h][hf] = fmaf(v0, v0, fmaf(v1, v1, q[h][hf]));
}

// sum over the four lanes of a quad, which hold the columns of one accumulator row
__device__ __forceinline__ float quad_sum(float s) {
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  return s;
}

// sums a thread's row statistics over the quad and stores those of rows grow[h] >= 0: ln_stats_out[row][col * 2 + half]
__device__ __forceinline__ void row_stats_store(const GemmParams& p, const float (&s)[2][2], const float (&q)[2][2],
                                                const long long (&grow)[2], int col, int quad) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const float sh = quad_sum(s[h][hf]), qh = quad_sum(q[h][hf]);
      if (quad == 0 && grow[h] >= 0)
        reinterpret_cast<float2*>(p.ln_stats_out)[grow[h] * p.ln_parts_out + col * 2 + hf] = make_float2(sh, qh);
    }
}

}  // namespace pn
