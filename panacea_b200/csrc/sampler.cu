// The sampler's per-evaluation step: one grid-stride fp32 elementwise kernel that turns the network output of one
// evaluation into the next sampler state and the next network input. It restates, in the reference's fp32 operation
// order, the denoiser scalings (denoiser.py:22-28 with EpsScaling), the guidance combine (guiders.py:25-29,
// sampling_utils.py:7-9) and the solver updates of sampling.py:85-365 (see pn_sampler_mode in the header).
#include "common.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

// ---------------------------------------------------------------- Philox4x32-10 (Salmon et al., SC'11) + Box-Muller
__host__ __device__ __forceinline__ void philox_round(uint32_t (&c)[4], const uint32_t (&k)[2]) {
  const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
  const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
  c[0] = hi1 ^ c[1] ^ k[0];
  c[1] = lo1;
  c[2] = hi0 ^ c[3] ^ k[1];
  c[3] = lo0;
}

__host__ __device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  uint32_t k[2] = {k0, k1};
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k);
    k[0] += 0x9E3779B9u;
    k[1] += 0xBB67AE85u;
  }
}

// Standard normal for element e of draw `draw` under `seed`: Philox block (e / 4, draw) with key `seed`; words
// (0,1) and (2,3) are two Box-Muller pairs, u1 = (w + 1) 2^-32 in (0, 1], u2 = w 2^-32 in [0, 1); the even element of
// a pair takes the cosine, the odd one the sine. Evaluated in fp64 and rounded once, so a value depends only on
// (seed, draw, e) and the host restatement (tests/test_sampler_philox_cpu.py) reproduces it bit for bit.
__device__ __forceinline__ float philox_normal(uint64_t seed, uint64_t draw, uint64_t e) {
  const uint64_t blk = e >> 2;
  uint32_t c[4] = {(uint32_t)blk, (uint32_t)(blk >> 32), (uint32_t)draw, (uint32_t)(draw >> 32)};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const int pair = (int)((e >> 1) & 1);
  const uint32_t a = pair ? c[2] : c[0], b = pair ? c[3] : c[1];
  const double u1 = ((double)a + 1.0) * 2.3283064365386963e-10;
  const double u2 = (double)b * 2.3283064365386963e-10;
  const double r = sqrt(-2.0 * log(u1));
  const double th = 6.283185307179586 * u2;
  return (float)((e & 1) ? r * sin(th) : r * cos(th));
}

// ---------------------------------------------------------------- the step kernel
// KNOWN = false takes an empty second argument, so those instantiations compile to the plain step kernel.
template <bool KNOWN> struct KnownArgs {};
template <> struct KnownArgs<true> : pn_sampler_known_args {};

template <int MODE, bool KNOWN>
__global__ void sampler_step_kernel(pn_sampler_step_args a, KnownArgs<KNOWN> k) {
  const size_t n = (size_t)a.n;
  float* out = a.out ? a.out : a.x;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    float o;
    if (MODE == PN_SAMPLER_SCALE) {
      o = a.x[e] * a.coef[0];
    } else {
      const float xe = a.x_eval ? a.x_eval[e] : a.x[e];
      // denoiser.py:28 with EpsScaling: denoised = net * c_out + x * c_skip, c_out = -sigma_q, c_skip = 1
      float den = a.net_is_denoised ? a.net[e] : a.net[e] * (-a.sigma_q) + xe;
      if (a.halves == 2) {              // VanillaCFG: x_u + scale (x_c - x_u), unconditional half first
        const float den_c = a.net_is_denoised ? a.net[n + e] : a.net[n + e] * (-a.sigma_q) + xe;
        den = den + a.cfg_scale * (den_c - den);
      }
      if (MODE == PN_SAMPLER_EULER) {   // sampling_utils.py:39-40 to_d; sampling.py:81-82 x + dt d
        const float d = (xe - den) / a.sigma;
        o = xe + a.dt * d;
        if (a.hist_write >= 0) a.hist[(size_t)a.hist_write * n + e] = d;
      } else if (MODE == PN_SAMPLER_HEUN) {   // sampling.py:229-235
        const float d_new = (xe - den) / a.sigma;
        const float d_prime = (a.hist[(size_t)a.hist_read[0] * n + e] + d_new) / 2.0f;
        o = a.x[e] + d_prime * a.dt;
      } else if (MODE == PN_SAMPLER_LMS) {    // sampling.py:200-209: x + sum_j c_j d_{i-j}
        const float d = (xe - den) / a.sigma;
        float acc = a.coef[0] * d;
#pragma unroll
        for (int j = 0; j < 3; ++j)
          if (a.hist_read[j] >= 0) acc = acc + a.coef[j + 1] * a.hist[(size_t)a.hist_read[j] * n + e];
        o = a.x[e] + acc;
        if (a.hist_write >= 0) a.hist[(size_t)a.hist_write * n + e] = d;
      } else if (MODE == PN_SAMPLER_DPM) {    // sampling.py:279,281,332: m0 x - m1 D
        o = a.coef[0] * a.x[e] - a.coef[1] * den;
        if (a.hist_write >= 0) a.hist[(size_t)a.hist_write * n + e] = den;
      } else {                                // PN_SAMPLER_DPM_2M, sampling.py:337-338
        const float den_d = a.coef[2] * den - a.coef[3] * a.hist[(size_t)a.hist_read[0] * n + e];
        o = a.coef[0] * a.x[e] - a.coef[1] * den_d;
        if (a.hist_write >= 0) a.hist[(size_t)a.hist_write * n + e] = den;
      }
    }
    if (a.noise_amp != 0.f) {           // sampling.py:99-100 (churn), :151-155 (ancestral): x + (xi s_noise) amp
      const float xi = a.noise ? a.noise[e] : philox_normal(a.seed, a.draw, e);
      o = o + xi * a.noise_scale * a.noise_amp;
    }
    if constexpr (KNOWN) {              // blend toward the known latent (pn_sampler_step_known)
      const float m = k.mask[(e / ((size_t)k.channels * k.plane)) * k.plane + e % k.plane];
      if (m != 1.f) {
        float kn = k.known[e];
        if (k.sigma != 0.f) kn = __fadd_rn(kn, __fmul_rn(k.sigma, philox_normal(k.seed, k.draw, e)));
        o = m == 0.f ? kn : m * o + (1.f - m) * kn;
      }
    }
    out[e] = o;
    if (a.x_in_next) {                  // next network input: x * c_in, duplicated for CFG
      const float v = o * a.c_in_next;
      for (int h = 0; h < a.halves; ++h) a.x_in_next[(size_t)h * n + e] = v;
    }
  }
}

}  // namespace pn

using namespace pn;

template <bool KNOWN>
static int launch_sampler_step(const pn_sampler_step_args* a, KnownArgs<KNOWN> k, void* stream_v) {
  PN_REQUIRE(a && a->x && a->n > 0, "pn_sampler_step: bad arguments");
  PN_REQUIRE(a->mode >= PN_SAMPLER_EULER && a->mode <= PN_SAMPLER_SCALE, "pn_sampler_step: mode %d", a->mode);
  PN_REQUIRE(a->halves == 1 || a->halves == 2, "pn_sampler_step: halves %d", a->halves);
  const bool net_mode = a->mode != PN_SAMPLER_SCALE;
  PN_REQUIRE(!net_mode || a->net, "pn_sampler_step: net is NULL");
  PN_REQUIRE(!(a->mode == PN_SAMPLER_EULER || a->mode == PN_SAMPLER_HEUN || a->mode == PN_SAMPLER_LMS) || a->sigma > 0.f,
             "pn_sampler_step: sigma must be > 0");
  const bool reads_hist = a->mode == PN_SAMPLER_HEUN || a->mode == PN_SAMPLER_DPM_2M ||
                          (a->mode == PN_SAMPLER_LMS && (a->hist_read[0] >= 0 || a->hist_read[1] >= 0 || a->hist_read[2] >= 0));
  PN_REQUIRE(!(reads_hist || a->hist_write >= 0) || a->hist, "pn_sampler_step: hist is NULL");
  PN_REQUIRE(!reads_hist || a->mode == PN_SAMPLER_LMS || a->hist_read[0] >= 0, "pn_sampler_step: hist_read[0] missing");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  const dim3 grid(stride_grid((size_t)a->n)), block(256);
  switch (a->mode) {
    case PN_SAMPLER_EULER: sampler_step_kernel<PN_SAMPLER_EULER, KNOWN><<<grid, block, 0, st>>>(*a, k); break;
    case PN_SAMPLER_HEUN: sampler_step_kernel<PN_SAMPLER_HEUN, KNOWN><<<grid, block, 0, st>>>(*a, k); break;
    case PN_SAMPLER_LMS: sampler_step_kernel<PN_SAMPLER_LMS, KNOWN><<<grid, block, 0, st>>>(*a, k); break;
    case PN_SAMPLER_DPM: sampler_step_kernel<PN_SAMPLER_DPM, KNOWN><<<grid, block, 0, st>>>(*a, k); break;
    case PN_SAMPLER_DPM_2M: sampler_step_kernel<PN_SAMPLER_DPM_2M, KNOWN><<<grid, block, 0, st>>>(*a, k); break;
    default: sampler_step_kernel<PN_SAMPLER_SCALE, KNOWN><<<grid, block, 0, st>>>(*a, k); break;
  }
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}

extern "C" int pn_sampler_step(const pn_sampler_step_args* a, void* stream_v) {
  return launch_sampler_step(a, KnownArgs<false>{}, stream_v);
}

extern "C" int pn_sampler_step_known(const pn_sampler_step_args* a, const pn_sampler_known_args* k, void* stream_v) {
  PN_REQUIRE(a && k && k->known && k->mask, "pn_sampler_step_known: bad arguments");
  PN_REQUIRE(k->channels > 0 && k->plane > 0 && a->n % ((int64_t)k->channels * k->plane) == 0,
             "pn_sampler_step_known: n = %lld is not a whole number of frames of %d x %lld", (long long)a->n,
             k->channels, (long long)k->plane);
  KnownArgs<true> kk;
  static_cast<pn_sampler_known_args&>(kk) = *k;
  return launch_sampler_step(a, kk, stream_v);
}

