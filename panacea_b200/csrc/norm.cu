// Normalisation kernels (HBM-bound): they read the fp32 residual stream once and emit the bf16 MMA operand
// of the GEMM/conv that follows, with the affine transform and SiLU fused in.
//
//  * spatial GroupNorm(32)  — statistics over (C/32 channels x all H x Wtot pixels of one frame), i.e. over
//    ALL SIX VIEWS jointly (reference: util.py:276-283 eps 1e-5 in ResBlock3D, attention.py:129-132 eps 1e-6
//    in SpatialTemporalTransformer);
//  * pixel-wise GroupNorm(32) over (C/32 channels x T frames) per pixel (reference: openaimodel.py:509-515,
//    534-539: GroupNorm applied to the [(b h w), C, T] rearrangement) — here computed in place on the
//    [b, T, P, C] layout, no rearrange copies;
//  * LayerNorm(C) per token (attention.py:699-701, eps 1e-5).
#include <cstdlib>
#include "common.cuh"
#include "ptx.cuh"
#include "operand.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

constexpr int GN_GROUPS = 32;
constexpr int GN_THREADS = 512;
constexpr int GN_MAX_FRAMES = 1024;
constexpr size_t GN_WAVE_BYTES = 56ull << 20;   // frames processed together: their fp32 input stays resident in L2

// ---------------------------------------------------------------- spatial GN (+SiLU) -> bf16, ONE launch
// The statistics of a frame need every pixel of it before the first output can be written, so the input is read
// twice; done as two kernels over the whole tensor the second read comes from HBM again (220 MB at level 0). Here the
// frames are processed in waves small enough to stay in L2: `cpf` co-resident CTAs share one frame, each
//   1. accumulates (sum, sumsq) per group over its pixel range (fixed order: bit-reproducible, no float atomics),
//   2. publishes them and waits for the other CTAs of the frame (one integer atomic per CTA),
//   3. combines all partials of the frame in double precision (every CTA does the same sum in the same order),
//   4. normalises ITS OWN pixel range again (L2 hits) -> y = act(x * rstd * gamma + beta - mean * rstd * gamma).
// Thread layout in both passes: (pixel lane, 8-channel column), so scale/shift live in registers in pass 4.
// partial: [frames][cpf][32 groups][2] floats; arrive: [frames] counters, both in the PER-CALL workspace (the counters
// are zeroed by a memset node in front of the launch), so concurrent launches on other streams, other devices or an
// aborted earlier launch cannot disturb the barrier.
// PHASE 0: fused, launched COOPERATIVELY (the runtime guarantees the co-residency the barrier needs or refuses the
// launch); PHASE 1 / 2: the same work as two ordinary launches (statistics, then normalise) for devices/contexts that
// cannot hold the whole grid (MPS active-thread percentage, green contexts, SM partitioning).
// OP: how the operand is stored (operand.cuh): bf16, split3 (parity mode) or fp32.
template <int OP, int PHASE>
__global__ void __launch_bounds__(GN_THREADS, 1)
gn_fused_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                void* __restrict__ y, void* __restrict__ raw, float* __restrict__ partial, unsigned int* __restrict__ arrive,
                int P, int C, int F, int wave, int cpf, float eps, int act_silu) {
  extern __shared__ float gn_smem[];
  const int c8n = C / 8;
  const int cols = c8n < GN_THREADS ? c8n : GN_THREADS;
  const int PL = GN_THREADS / cols;                 // pixel lanes
  float* colacc = gn_smem;                          // [PL][2][C]
  float* s_scale = gn_smem + (size_t)PL * 2 * C;    // [C]
  float* s_shift = s_scale + C;                     // [C]
  __shared__ double s_part[8][GN_GROUPS * 2];
  __shared__ float s_mean[GN_GROUPS], s_rstd[GN_GROUPS];
  const int cpg = C / GN_GROUPS;
  const int pl = threadIdx.x / cols;
  const int col0 = threadIdx.x - pl * cols;
  const int fi = blockIdx.x / cpf, r = blockIdx.x - fi * cpf;
  if (fi >= wave) return;
  const int ppc = (P + cpf - 1) / cpf;              // pixels per CTA
  const int p0 = r * ppc, p1 = min(P, p0 + ppc);

  for (int f = fi; f < F; f += wave) {
    const float* xb = x + (size_t)f * P * C;
    // ---- pass 1: per-thread column sums over this CTA's pixels
    if (PHASE != 2 && pl < PL) {
      for (int c8 = col0; c8 < c8n; c8 += cols) {
        float s[8], q[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { s[j] = 0.f; q[j] = 0.f; }
        int p = p0 + pl;
        for (; p + 3 * PL < p1; p += 4 * PL) {      // four pixels in flight per thread
          float4 a[4], b[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float* src = xb + (size_t)(p + u * PL) * C + (size_t)c8 * 8;
            a[u] = *reinterpret_cast<const float4*>(src);
            b[u] = *reinterpret_cast<const float4*>(src + 4);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            s[0] += a[u].x; q[0] += a[u].x * a[u].x; s[1] += a[u].y; q[1] += a[u].y * a[u].y;
            s[2] += a[u].z; q[2] += a[u].z * a[u].z; s[3] += a[u].w; q[3] += a[u].w * a[u].w;
            s[4] += b[u].x; q[4] += b[u].x * b[u].x; s[5] += b[u].y; q[5] += b[u].y * b[u].y;
            s[6] += b[u].z; q[6] += b[u].z * b[u].z; s[7] += b[u].w; q[7] += b[u].w * b[u].w;
          }
        }
        for (; p < p1; p += PL) {
          const float* src = xb + (size_t)p * C + (size_t)c8 * 8;
          const float4 a = *reinterpret_cast<const float4*>(src);
          const float4 b = *reinterpret_cast<const float4*>(src + 4);
          s[0] += a.x; q[0] += a.x * a.x; s[1] += a.y; q[1] += a.y * a.y; s[2] += a.z; q[2] += a.z * a.z;
          s[3] += a.w; q[3] += a.w * a.w; s[4] += b.x; q[4] += b.x * b.x; s[5] += b.y; q[5] += b.y * b.y;
          s[6] += b.z; q[6] += b.z * b.z; s[7] += b.w; q[7] += b.w * b.w;
        }
        float* dst = colacc + (size_t)pl * 2 * C + (size_t)c8 * 8;
        *reinterpret_cast<float4*>(dst) = make_float4(s[0], s[1], s[2], s[3]);
        *reinterpret_cast<float4*>(dst + 4) = make_float4(s[4], s[5], s[6], s[7]);
        *reinterpret_cast<float4*>(dst + C) = make_float4(q[0], q[1], q[2], q[3]);
        *reinterpret_cast<float4*>(dst + C + 4) = make_float4(q[4], q[5], q[6], q[7]);
      }
    }
    __syncthreads();
    float* my_partial = partial + ((size_t)f * cpf + r) * GN_GROUPS * 2;
    if (PHASE != 2 && threadIdx.x < GN_GROUPS * 2) {
      const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
      float acc = 0.f;
      for (int l = 0; l < PL; ++l) {
        const float* src = colacc + (size_t)l * 2 * C + which * C + g * cpg;
        for (int j = 0; j < cpg; ++j) acc += src[j];
      }
      my_partial[threadIdx.x] = acc;
      __threadfence();
    }
    __syncthreads();
    if (PHASE == 1) continue;
    // ---- frame barrier among the cpf CTAs of this frame (each frame's counter is used exactly once per launch)
    if (PHASE == 0) {
      if (threadIdx.x == 0) {
        atomicAdd(&arrive[f], 1u);
        while (*reinterpret_cast<volatile unsigned int*>(&arrive[f]) < (unsigned int)cpf) __nanosleep(64);
        __threadfence();
      }
      __syncthreads();
    }
    // ---- combine all partials of the frame (double precision, fixed order, identical in every CTA)
    {
      const int slot = threadIdx.x & 63, part = threadIdx.x >> 6;      // 8 interleaved partial sums per slot
      double acc = 0.0;
      const float* pp = partial + (size_t)f * cpf * GN_GROUPS * 2 + slot;
      for (int k = part; k < cpf; k += GN_THREADS / 64) acc += (double)__ldcg(pp + (size_t)k * GN_GROUPS * 2);
      s_part[part][slot] = acc;
    }
    __syncthreads();
    if (threadIdx.x < GN_GROUPS) {
      const int g = threadIdx.x;
      double sm = 0.0, sq = 0.0;
#pragma unroll
      for (int k = 0; k < 8; ++k) { sm += s_part[k][2 * g]; sq += s_part[k][2 * g + 1]; }
      const double n = (double)P * cpg;
      const double mean = sm / n;
      double var = sq / n - mean * mean;
      if (var < 0.0) var = 0.0;
      s_mean[g] = (float)mean;
      s_rstd[g] = (float)(1.0 / sqrt(var + (double)eps));
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += GN_THREADS) {
      const int g = c / cpg;
      const float sc = s_rstd[g] * gamma[c];
      s_scale[c] = sc;
      s_shift[c] = beta[c] - s_mean[g] * sc;
    }
    __syncthreads();
    // ---- pass 2: normalise this CTA's pixel range (second read of x: L2)
    const size_t row0 = (size_t)f * P;
    if (pl < PL) {
      for (int c8 = col0; c8 < c8n; c8 += cols) {
        float sc[8], sh[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { sc[j] = s_scale[c8 * 8 + j]; sh[j] = s_shift[c8 * 8 + j]; }
        auto emit = [&](size_t off, const float4& a, const float4& b) {
          float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
          const size_t row = row0 + off / (size_t)C;
          if (raw) store_op<OP>(raw, row, C, c8 * 8, v);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float t = v[j] * sc[j] + sh[j];
            v[j] = act_silu ? silu(t) : t;
          }
          store_op<OP>(y, row, C, c8 * 8, v);
        };
        int p = p0 + pl;
        for (; p + 3 * PL < p1; p += 4 * PL) {      // four pixels in flight per thread
          float4 a[4], b[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float* src = xb + (size_t)(p + u * PL) * C + (size_t)c8 * 8;
            a[u] = *reinterpret_cast<const float4*>(src);
            b[u] = *reinterpret_cast<const float4*>(src + 4);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) emit((size_t)(p + u * PL) * C + (size_t)c8 * 8, a[u], b[u]);
        }
        for (; p < p1; p += PL) {
          const size_t off = (size_t)p * C + (size_t)c8 * 8;
          emit(off, *reinterpret_cast<const float4*>(xb + off), *reinterpret_cast<const float4*>(xb + off + 4));
        }
      }
    }
    __syncthreads();      // colacc / s_scale are rewritten by the next frame of this CTA
  }
}

// ---------------------------------------------------------------- pixel-wise temporal GN (+SiLU) -> bf16
// x: fp32 [b, T, P, C]. One block per (b, p); thread (t, g) = (warp, lane) owns the cpg channels of group g at frame t
// and keeps them in registers: a single pass over HBM, exact two-pass statistics (mean, then centred sum of squares)
// combined across the T warps through shared memory. Lanes read adjacent cpg-float runs, i.e. whole rows coalesced.
template <int CPG, int OP>
__global__ void __launch_bounds__(512) gn_pixel_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, void* __restrict__ y,
                                                       int T, int P, int C, float eps, int act_silu) {
  __shared__ float red[16][32];
  const int t = threadIdx.x >> 5, g = threadIdx.x & 31;
  const int b = blockIdx.x / P, p = blockIdx.x - b * P;
  const size_t off = (((size_t)b * T + t) * P + p) * C + (size_t)g * CPG;
  float v[CPG];
  const float2* src = reinterpret_cast<const float2*>(x + off);
#pragma unroll
  for (int j = 0; j < CPG / 2; ++j) {
    const float2 a = src[j];
    v[2 * j] = a.x;
    v[2 * j + 1] = a.y;
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < CPG; ++j) s += v[j];
  red[t][g] = s;
  __syncthreads();
  float tot = 0.f;
  for (int k = 0; k < T; ++k) tot += red[k][g];
  const float n = (float)(T * CPG);
  const float mean = tot / n;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < CPG; ++j) {
    const float d = v[j] - mean;
    q += d * d;
  }
  __syncthreads();
  red[t][g] = q;
  __syncthreads();
  float qt = 0.f;
  for (int k = 0; k < T; ++k) qt += red[k][g];
  const float rstd = rsqrtf(qt / n + eps);
  const size_t row = ((size_t)b * T + t) * P + p;
  const float2* g2 = reinterpret_cast<const float2*>(gamma + g * CPG);
  const float2* b2 = reinterpret_cast<const float2*>(beta + g * CPG);
#pragma unroll
  for (int j = 0; j < CPG / 2; ++j) {
    const float2 gm = g2[j], bt = b2[j];
    float a0 = (v[2 * j] - mean) * rstd * gm.x + bt.x;
    float a1 = (v[2 * j + 1] - mean) * rstd * gm.y + bt.y;
    if (act_silu) { a0 = silu(a0); a1 = silu(a1); }
    const float o[2] = {a0, a1};
    store_op<OP>(y, row, C, g * CPG + 2 * j, o);
  }
}

// ---------------------------------------------------------------- LayerNorm per token -> bf16
// one warp per row; the row (C <= 2048 floats) lives in registers between the two passes.
__device__ __forceinline__ float4 ln_load4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ln_load4(const __nv_bfloat16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

// TIn: fp32 residual stream, or the bf16 token stream of the transformer blocks (fast path)
template <int MAXV, int OP, typename TIn>
__global__ void __launch_bounds__(256) layernorm_kernel(const TIn* __restrict__ x, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, void* __restrict__ y,
                                                        long long rows, int C, float eps) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const TIn* xr = x + row * C;
  const int n4 = C / 4;
  float4 v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + i * 32;
    if (j < n4) {
      v[i] = ln_load4(xr + 4 * j);
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + i * 32;
    if (j < n4) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += a * a + b * b + c * c + d * d;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int j = lane + i * 32;
    if (j < n4) {
      const float4 g = g4[j], bb = b4[j];
      const float o0 = (v[i].x - mean) * rstd * g.x + bb.x;
      const float o1 = (v[i].y - mean) * rstd * g.y + bb.y;
      const float o2 = (v[i].z - mean) * rstd * g.z + bb.z;
      const float o3 = (v[i].w - mean) * rstd * g.w + bb.w;
      const float o[4] = {o0, o1, o2, o3};
      store_op<OP>(y, (size_t)row, C, j * 4, o);
    }
  }
}

// bf16 token stream -> bf16 operand, the LayerNorm of the fast path (norm3 of every block, all three at C = 1280):
// LPR lanes per row, NV 16-byte loads (8 channels each) per lane all in flight at once, ONE shuffle reduction of
// (sum, sum of squares) over the LPR lanes — the warp-per-row two-reduction kernel above was latency-bound at 37 % of the
// HBM bandwidth for this 2-bytes-in / 2-bytes-out shape.
template <int LPR, int NV>
__global__ void __launch_bounds__(256) layernorm_bf16_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, __nv_bfloat16* __restrict__ y,
                                                             long long rows, int C, float eps) {
  constexpr int RPW = 32 / LPR;                                  // rows per warp and pass
  const int lane = threadIdx.x & 31, sub = lane % LPR;
  // the affine parameters are staged in shared memory once per CTA (re-reading them from global per row cost four times
  // the row's own bytes in L1 traffic); each CTA then walks many rows
  extern __shared__ float ln_gb[];                               // [2][C]
  for (int i = threadIdx.x; i < C / 4; i += blockDim.x) {
    reinterpret_cast<float4*>(ln_gb)[i] = reinterpret_cast<const float4*>(gamma)[i];
    reinterpret_cast<float4*>(ln_gb + C)[i] = reinterpret_cast<const float4*>(beta)[i];
  }
  __syncthreads();
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float inv_c = 1.f / (float)C;
  for (long long base = warp0 * RPW; base < rows; base += nwarps * RPW) {
    const long long row = base + lane / LPR;
    const bool ok = row < rows;
    const __nv_bfloat16* xr = x + (ok ? row : base) * C;
    uint4 raw[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) raw[i] = *reinterpret_cast<const uint4*>(xr + (sub + i * LPR) * 8);
    float v[NV][8];
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        v[i][2 * e] = __uint_as_float(w[e] << 16);
        v[i][2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u);
        s += v[i][2 * e] + v[i][2 * e + 1];
        q = fmaf(v[i][2 * e], v[i][2 * e], fmaf(v[i][2 * e + 1], v[i][2 * e + 1], q));
      }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    const float mean = s * inv_c;
    const float rstd = rsqrtf(fmaxf(q * inv_c - mean * mean, 0.f) + eps);
    if (ok) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c0 = (sub + i * LPR) * 8;
        const float4 g0 = *reinterpret_cast<const float4*>(ln_gb + c0), g1 = *reinterpret_cast<const float4*>(ln_gb + c0 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(ln_gb + C + c0), b1 = *reinterpret_cast<const float4*>(ln_gb + C + c0 + 4);
        const float gq[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, bq[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mean) * rstd * gq[e] + bq[e];
        *reinterpret_cast<uint4*>(y + row * C + (sub + i * LPR) * 8) =
            make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
      }
    }
  }
}

}  // namespace pn

using namespace pn;

// wave = frames processed concurrently (their input fits L2), cpf = CTAs per frame; wave * cpf <= SM count
static void gn_geometry(int64_t frames, int64_t pixels, int64_t channels, int* wave, int* cpf) {
  const size_t frame_bytes = (size_t)pixels * channels * sizeof(float);
  int w = (int)(GN_WAVE_BYTES / (frame_bytes ? frame_bytes : 1));
  if (w < 1) w = 1;
  if (w > frames) w = (int)frames;
  const int sms = sm_count();
  if (w > sms) w = sms;
  for (int d = w; 2 * d > w; --d)                 // prefer a wave that divides the frame count (no idle last wave)
    if (frames % d == 0) { w = d; break; }
  int c = sms / w;
  const int max_c = (int)((pixels + 7) / 8);      // at least 8 pixels per CTA
  if (c > max_c) c = max_c < 1 ? 1 : max_c;
  *wave = w;
  *cpf = c;
}

extern "C" int64_t pn_groupnorm_workspace_floats(int64_t frames, int64_t pixels, int64_t channels) {
  int wave, cpf;
  gn_geometry(frames, pixels, channels, &wave, &cpf);
  return frames * cpf * GN_GROUPS * 2 + frames;      // partial sums + one arrival counter per frame
}

extern "C" int64_t pn_groupnorm_ctas_per_frame(int64_t frames, int64_t pixels, int64_t channels) {
  int wave, cpf;
  gn_geometry(frames, pixels, channels, &wave, &cpf);
  return cpf;
}

template <int OP, int PHASE>
static int gn_launch(bool cooperative, int grid, size_t smem, cudaStream_t st, const float* x, const float* gamma, const float* beta,
                     void* y, void* raw, float* partial, unsigned int* arrive, int P, int C, int F, int wave, int cpf, float eps,
                     int act_silu) {
  const int rc = ensure_dyn_smem(reinterpret_cast<const void*>(&gn_fused_kernel<OP, PHASE>), smem);
  if (rc != PN_OK) return rc;
  cudaLaunchConfig_t cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(GN_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = cooperative ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  PN_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gn_fused_kernel<OP, PHASE>, x, gamma, beta, y, raw, partial, arrive, P, C, F, wave, cpf,
                                   eps, act_silu));
  return PN_OK;
}

extern "C" int pn_groupnorm_silu(const float* x, const float* gamma, const float* beta, void* y, void* raw,
                                 float* workspace, int64_t frames, int64_t pixels, int64_t channels, float eps,
                                 int act_silu, int operand_mode, void* stream_v) {
  PN_OPERAND_MODES(Modes, operand_mode, "pn_groupnorm_silu", PN_OPERAND_BF16, PN_OPERAND_SPLIT3, PN_OPERAND_F32);
  PN_REQUIRE(x && gamma && beta && y && workspace, "pn_groupnorm_silu: null pointer");
  PN_REQUIRE(channels % 32 == 0 && channels % 8 == 0 && channels <= 8192, "pn_groupnorm_silu: C=%lld unsupported",
             (long long)channels);
  PN_REQUIRE(frames > 0 && pixels > 0, "pn_groupnorm_silu: empty input");
  PN_REQUIRE(frames <= GN_MAX_FRAMES, "pn_groupnorm_silu: more than %d frames", GN_MAX_FRAMES);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  const int P = (int)pixels, C = (int)channels, F = (int)frames;
  int wave, cpf;
  gn_geometry(frames, pixels, channels, &wave, &cpf);
  const int c8n = C / 8;
  const int cols = c8n < GN_THREADS ? c8n : GN_THREADS;
  const int PL = GN_THREADS / cols;
  const size_t smem = ((size_t)PL * 2 * C + 2 * (size_t)C) * sizeof(float);
  float* partial = workspace;
  unsigned int* arrive = reinterpret_cast<unsigned int*>(workspace + (size_t)F * cpf * GN_GROUPS * 2);
  const int grid = wave * cpf;
  // The fused form needs all wave * cpf CTAs resident at once. The grid never exceeds the SM count the device
  // reports and the kernel takes one CTA per SM; the cooperative launch makes the runtime check that against what the
  // context can really hold. PN_GN_TWO_PHASE=1 (or a single CTA per frame) selects the barrier-free two-launch form.
  static const bool force_two_phase = [] { const char* e = std::getenv("PN_GN_TWO_PHASE"); return e && std::atoi(e) != 0; }();
  if (force_two_phase) {
    int rc = PN_OK;
    PN_DISPATCH_OP(Modes, operand_mode, rc = gn_launch<OP, 1>(false, grid, smem, st, x, gamma, beta, y, raw, partial, arrive, P, C, F,
                                                               wave, cpf, eps, act_silu));
    if (rc != PN_OK) return rc;
    PN_DISPATCH_OP(Modes, operand_mode, rc = gn_launch<OP, 2>(false, grid, smem, st, x, gamma, beta, y, raw, partial, arrive, P, C, F,
                                                               wave, cpf, eps, act_silu));
    return rc;
  }
  PN_CHECK_CUDA(cudaMemsetAsync(arrive, 0, sizeof(unsigned int) * (size_t)F, st));
  int rc = PN_OK;
  PN_DISPATCH_OP(Modes, operand_mode, rc = gn_launch<OP, 0>(true, grid, smem, st, x, gamma, beta, y, raw, partial, arrive, P, C, F,
                                                             wave, cpf, eps, act_silu));
  return rc;
}

extern "C" int pn_groupnorm_pixel_silu(const float* x, const float* gamma, const float* beta, void* y,
                                       int64_t batch, int64_t frames_per_seq, int64_t pixels, int64_t channels,
                                       float eps, int act_silu, int operand_mode, void* stream_v) {
  PN_OPERAND_MODES(Modes, operand_mode, "pn_groupnorm_pixel_silu", PN_OPERAND_BF16, PN_OPERAND_SPLIT3, PN_OPERAND_F32);
  PN_REQUIRE(x && gamma && beta && y, "pn_groupnorm_pixel_silu: null pointer");
  PN_REQUIRE(channels % 64 == 0, "pn_groupnorm_pixel_silu: C=%lld must be a multiple of 64", (long long)channels);
  PN_REQUIRE(batch > 0 && frames_per_seq > 0 && pixels > 0, "pn_groupnorm_pixel_silu: empty input");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  PN_REQUIRE(frames_per_seq <= 16, "pn_groupnorm_pixel_silu: T=%lld > 16 unsupported", (long long)frames_per_seq);
  const long long blocks = batch * pixels;
  PN_REQUIRE(blocks < (1ll << 31), "pn_groupnorm_pixel_silu: grid too large");
  const int threads = (int)frames_per_seq * 32;
  const int T = (int)frames_per_seq, P = (int)pixels, C = (int)channels;
  switch (C / 32) {
#define PN_GNP_CASE(CPG) case CPG: PN_DISPATCH_OP(Modes, operand_mode, gn_pixel_kernel<CPG, OP><<<(unsigned)blocks, threads, 0, st>>>(x, gamma, beta, y, T, P, C, eps, act_silu)); break;
    PN_GNP_CASE(2) PN_GNP_CASE(4) PN_GNP_CASE(6) PN_GNP_CASE(8) PN_GNP_CASE(10) PN_GNP_CASE(12) PN_GNP_CASE(16) PN_GNP_CASE(20)
    PN_GNP_CASE(24) PN_GNP_CASE(30) PN_GNP_CASE(32) PN_GNP_CASE(40) PN_GNP_CASE(60) PN_GNP_CASE(80)
#undef PN_GNP_CASE
    default:
      return fail(PN_ERR_UNSUPPORTED, "pn_groupnorm_pixel_silu: C=%lld (C/32=%lld channels per group) is not instantiated",
                  (long long)channels, (long long)(channels / 32));
  }
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}

extern "C" int pn_layernorm(const void* x, int x_is_bf16, const float* gamma, const float* beta, void* y, int64_t rows,
                            int64_t channels, float eps, int operand_mode, void* stream_v) {
  PN_OPERAND_MODES(Modes, operand_mode, "pn_layernorm", PN_OPERAND_BF16, PN_OPERAND_SPLIT3, PN_OPERAND_F32);
  PN_REQUIRE(x && gamma && beta && y, "pn_layernorm: null pointer");
  PN_REQUIRE(channels % 4 == 0 && channels <= 2048 && channels > 0, "pn_layernorm: C=%lld unsupported", (long long)channels);
  PN_REQUIRE(rows > 0, "pn_layernorm: empty input");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  const int C = (int)channels;
  if (x_is_bf16 && operand_mode == PN_OPERAND_BF16 && C % 64 == 0) {
    // fast path: LPR lanes per row, NV = C / (8 LPR) loads per lane (5 for C = 320 / 640 / 1280)
#define PN_LNB(LPR, NV)                                                                                                            \
    do {                                                                                                                           \
      const long long rows_per_block = 8 * (32 / LPR);                                                                             \
      long long nb = (rows + rows_per_block - 1) / rows_per_block;                                                                 \
      if (nb > 6ll * sm_count()) nb = 6ll * sm_count();          /* grid-stride over the rows: affine parameters staged once per CTA */ \
      layernorm_bf16_kernel<LPR, NV><<<(unsigned)nb, 256, (size_t)C * 8, st>>>(reinterpret_cast<const __nv_bfloat16*>(x),          \
          gamma, beta, reinterpret_cast<__nv_bfloat16*>(y), (long long)rows, C, eps);                                              \
      PN_CHECK_CUDA(cudaGetLastError());                                                                                           \
      return PN_OK;                                                                                                                \
    } while (0)
    for (int lpr = 8; lpr <= 32; lpr *= 2) {
      if (C % (8 * lpr) != 0) continue;
      const int nv = C / (8 * lpr);
      if (nv < 1 || nv > 8) continue;
      if (lpr == 8) { switch (nv) { case 1: PN_LNB(8, 1); case 2: PN_LNB(8, 2); case 3: PN_LNB(8, 3); case 4: PN_LNB(8, 4); case 5: PN_LNB(8, 5); case 6: PN_LNB(8, 6); case 7: PN_LNB(8, 7); default: PN_LNB(8, 8); } }
      if (lpr == 16) { switch (nv) { case 1: PN_LNB(16, 1); case 2: PN_LNB(16, 2); case 3: PN_LNB(16, 3); case 4: PN_LNB(16, 4); case 5: PN_LNB(16, 5); case 6: PN_LNB(16, 6); case 7: PN_LNB(16, 7); default: PN_LNB(16, 8); } }
      switch (nv) { case 1: PN_LNB(32, 1); case 2: PN_LNB(32, 2); case 3: PN_LNB(32, 3); case 4: PN_LNB(32, 4); case 5: PN_LNB(32, 5); case 6: PN_LNB(32, 6); case 7: PN_LNB(32, 7); default: PN_LNB(32, 8); }
    }
#undef PN_LNB
  }
  const long long blocks = (rows * 32 + 255) / 256;
#define PN_LN(MAXV)                                                                                                          \
  do {                                                                                                                       \
    if (x_is_bf16)                                                                                                           \
      PN_DISPATCH_OP(Modes, operand_mode, layernorm_kernel<MAXV, OP, __nv_bfloat16><<<(unsigned)blocks, 256, 0, st>>>(       \
          reinterpret_cast<const __nv_bfloat16*>(x), gamma, beta, y, rows, C, eps));                                         \
    else                                                                                                                     \
      PN_DISPATCH_OP(Modes, operand_mode, layernorm_kernel<MAXV, OP, float><<<(unsigned)blocks, 256, 0, st>>>(               \
          reinterpret_cast<const float*>(x), gamma, beta, y, rows, C, eps));                                                 \
  } while (0)
  if (C <= 512) PN_LN(4);
  else if (C <= 1024) PN_LN(8);
  else PN_LN(16);
#undef PN_LN
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}
