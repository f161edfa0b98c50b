// fp32 attention on CUDA cores — the attention of the PARITY mode (fp32-class arithmetic end to end, see operand.cuh).
//
// Same token geometry and view tables as the wgmma kernel (attn_fa.cu, pn_attn_args), but q/k/v are fp32, the
// products, the softmax (exp2f, not the MUFU approximation) and the PV accumulation are fp32 FMAs, and the output is
// written as the operand of the to_out GEMM (split3 in parity mode). It also covers head_dim 80 (BASELINE config 5).
// Throughput is irrelevant here (a full-size eps-eval spends ~30 ms in it); exactness against the reference's
// xformers / SDPA semantics softmax(q k^T * scale) v (attention.py:469-471, 590-592, 279-283) is the point.
//
//   view kernel    : one thread per query row, 128 queries per CTA; keys/values of the visited views are staged
//                    through shared memory 32 tokens at a time and broadcast to all threads; online softmax.
//   temporal kernel: one thread per (pixel, head, query frame); T <= 16 keys read straight from global/L1.
#include "common.cuh"
#include "ptx.cuh"
#include "operand.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

constexpr int AF_QTILE = 128;
constexpr int AF_KTILE = 32;

struct AfParams {
  const float* q; const float* k; const float* v;
  void* out;
  long long q_ld, kv_ld;
  int out_C;                    // channels of the output operand (heads * head_dim)
  int F, H, V, W, Hk, Vk, Wk, kv_frame_div, heads;
  int kv_views[8][2];
  int kv_view_count[8];
  float scale_log2;
};

template <int D, int OP>
__global__ void __launch_bounds__(AF_QTILE) attn_f32_view_kernel(const AfParams p) {
  __shared__ __align__(16) float sK[AF_KTILE][D];
  __shared__ __align__(16) float sV[AF_KTILE][D];
  const int tiles = (p.H * p.W + AF_QTILE - 1) / AF_QTILE;
  int item = blockIdx.x;
  const int tile = item % tiles; item /= tiles;
  const int head = item % p.heads; item /= p.heads;
  const int view = item % p.V; item /= p.V;
  const int frame = item;
  const int qi = tile * AF_QTILE + threadIdx.x;
  const bool active = qi < p.H * p.W;
  const int qy = active ? qi / p.W : 0, qx = active ? qi - (qi / p.W) * p.W : 0;
  const long long qtok = (((long long)frame * p.H + qy) * p.V + view) * p.W + qx;
  float q[D], o[D];
  {
    const float* qp = p.q + qtok * p.q_ld + head * D;
#pragma unroll
    for (int d = 0; d < D; d += 4) {
      const float4 t = active ? *reinterpret_cast<const float4*>(qp + d) : make_float4(0.f, 0.f, 0.f, 0.f);
      q[d] = t.x * p.scale_log2; q[d + 1] = t.y * p.scale_log2; q[d + 2] = t.z * p.scale_log2; q[d + 3] = t.w * p.scale_log2;
    }
#pragma unroll
    for (int d = 0; d < D; ++d) o[d] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  const int kv_frame = frame / p.kv_frame_div;
  const int keys_per_view = p.Hk * p.Wk;
  for (int vi = 0; vi < p.kv_view_count[view]; ++vi) {
    const int kvv = p.kv_views[view][vi];
    for (int k0 = 0; k0 < keys_per_view; k0 += AF_KTILE) {
      const int nk = min(AF_KTILE, keys_per_view - k0);
      __syncthreads();
      for (int e = threadIdx.x; e < AF_KTILE * (D / 4); e += AF_QTILE) {
        const int j = e / (D / 4), d4 = e - j * (D / 4);
        float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
        if (j < nk) {
          const int ki = k0 + j;
          const int ky = ki / p.Wk, kx = ki - ky * p.Wk;
          const long long ktok = (((long long)kv_frame * p.Hk + ky) * p.Vk + kvv) * p.Wk + kx;
          kk = *reinterpret_cast<const float4*>(p.k + ktok * p.kv_ld + head * D + d4 * 4);
          vv = *reinterpret_cast<const float4*>(p.v + ktok * p.kv_ld + head * D + d4 * 4);
        }
        *reinterpret_cast<float4*>(&sK[j][d4 * 4]) = kk;
        *reinterpret_cast<float4*>(&sV[j][d4 * 4]) = vv;
      }
      __syncthreads();
      float s[AF_KTILE];
      float mx = m;
#pragma unroll
      for (int j = 0; j < AF_KTILE; ++j) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
        for (int d = 0; d < D; d += 4) {
          const float4 kk = *reinterpret_cast<const float4*>(&sK[j][d]);
          a0 = fmaf(q[d], kk.x, a0); a1 = fmaf(q[d + 1], kk.y, a1); a2 = fmaf(q[d + 2], kk.z, a2); a3 = fmaf(q[d + 3], kk.w, a3);
        }
        s[j] = j < nk ? (a0 + a1) + (a2 + a3) : -INFINITY;
        mx = fmaxf(mx, s[j]);
      }
      const float alpha = exp2f(m - mx);          // first tile: exp2(-inf) = 0
      m = mx;
      l *= alpha;
#pragma unroll
      for (int d = 0; d < D; ++d) o[d] *= alpha;
#pragma unroll
      for (int j = 0; j < AF_KTILE; ++j) {
        const float pj = exp2f(s[j] - m);         // masked keys: exp2(-inf) = 0
        l += pj;
#pragma unroll
        for (int d = 0; d < D; d += 4) {
          const float4 vv = *reinterpret_cast<const float4*>(&sV[j][d]);
          o[d] = fmaf(pj, vv.x, o[d]); o[d + 1] = fmaf(pj, vv.y, o[d + 1]); o[d + 2] = fmaf(pj, vv.z, o[d + 2]); o[d + 3] = fmaf(pj, vv.w, o[d + 3]);
        }
      }
    }
  }
  if (active) {
    const float inv = 1.f / l;
#pragma unroll
    for (int d = 0; d < D; d += 8) {
      const float v8[8] = {o[d] * inv, o[d + 1] * inv, o[d + 2] * inv, o[d + 3] * inv,
                           o[d + 4] * inv, o[d + 5] * inv, o[d + 6] * inv, o[d + 7] * inv};
      store_op<OP>(p.out, (size_t)qtok, p.out_C, head * D + d, v8);
    }
  }
}

// q/k/v fp32 [batch, T, pixels, ld] -> out operand [batch*T*pixels, heads*D]
template <int D, int OP>
__global__ void __launch_bounds__(128) attn_f32_temporal_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                const float* __restrict__ v, void* __restrict__ out, int batch,
                                                                int T, int P, int heads, long long ld, float scale_log2) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)batch * T * P * heads;
  if (idx >= total) return;
  const int head = (int)(idx % heads);
  long long r = idx / heads;
  const int pix = (int)(r % P); r /= P;
  const int tq = (int)(r % T);
  const int b = (int)(r / T);
  const long long qtok = ((long long)b * T + tq) * P + pix;
  float qq[D], o[D];
  const float* qp = q + qtok * ld + head * D;
#pragma unroll
  for (int d = 0; d < D; d += 4) {
    const float4 t = *reinterpret_cast<const float4*>(qp + d);
    qq[d] = t.x * scale_log2; qq[d + 1] = t.y * scale_log2; qq[d + 2] = t.z * scale_log2; qq[d + 3] = t.w * scale_log2;
  }
  float s[16];
  float m = -INFINITY;
  for (int t = 0; t < T; ++t) {
    const float* kp = k + (((long long)b * T + t) * P + pix) * ld + head * D;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int d = 0; d < D; d += 4) {
      const float4 kk = *reinterpret_cast<const float4*>(kp + d);
      a0 = fmaf(qq[d], kk.x, a0); a1 = fmaf(qq[d + 1], kk.y, a1); a2 = fmaf(qq[d + 2], kk.z, a2); a3 = fmaf(qq[d + 3], kk.w, a3);
    }
    s[t] = (a0 + a1) + (a2 + a3);
    m = fmaxf(m, s[t]);
  }
#pragma unroll
  for (int d = 0; d < D; ++d) o[d] = 0.f;
  float l = 0.f;
  for (int t = 0; t < T; ++t) {
    const float pj = exp2f(s[t] - m);
    l += pj;
    const float* vp = v + (((long long)b * T + t) * P + pix) * ld + head * D;
#pragma unroll
    for (int d = 0; d < D; d += 4) {
      const float4 vv = *reinterpret_cast<const float4*>(vp + d);
      o[d] = fmaf(pj, vv.x, o[d]); o[d + 1] = fmaf(pj, vv.y, o[d + 1]); o[d + 2] = fmaf(pj, vv.z, o[d + 2]); o[d + 3] = fmaf(pj, vv.w, o[d + 3]);
    }
  }
  const float inv = 1.f / l;
#pragma unroll
  for (int d = 0; d < D; d += 8) {
    const float v8[8] = {o[d] * inv, o[d + 1] * inv, o[d + 2] * inv, o[d + 3] * inv,
                         o[d + 4] * inv, o[d + 5] * inv, o[d + 6] * inv, o[d + 7] * inv};
    store_op<OP>(out, (size_t)qtok, heads * D, head * D + d, v8);
  }
}

// Causal self-attention (the OpenCLIP text transformer) in fp32: one thread per (batch, head, query i) visits keys
// j <= i of its sequence, read from global/L1. Two passes over the keys (row maximum, then exp2 and P V) keep the
// scores out of registers for L up to 128.
// q/k/v fp32 [batch, L, ld] -> out operand [batch*L, heads*64]
template <int OP>
__global__ void __launch_bounds__(128) attn_f32_causal_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                              const float* __restrict__ v, void* __restrict__ out, int batch,
                                                              int L, int heads, long long ld, float scale_log2) {
  constexpr int D = 64;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)batch * heads * L;
  if (idx >= total) return;
  const int qi = (int)(idx % L);
  long long r = idx / L;
  const int head = (int)(r % heads);
  const int b = (int)(r / heads);
  const long long row0 = (long long)b * L;
  float qq[D], o[D];
  const float* qp = q + (row0 + qi) * ld + head * D;
#pragma unroll
  for (int d = 0; d < D; d += 4) {
    const float4 t = *reinterpret_cast<const float4*>(qp + d);
    qq[d] = t.x * scale_log2; qq[d + 1] = t.y * scale_log2; qq[d + 2] = t.z * scale_log2; qq[d + 3] = t.w * scale_log2;
  }
  auto score = [&](int j) {
    const float* kp = k + (row0 + j) * ld + head * D;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int d = 0; d < D; d += 4) {
      const float4 kk = *reinterpret_cast<const float4*>(kp + d);
      a0 = fmaf(qq[d], kk.x, a0); a1 = fmaf(qq[d + 1], kk.y, a1); a2 = fmaf(qq[d + 2], kk.z, a2); a3 = fmaf(qq[d + 3], kk.w, a3);
    }
    return (a0 + a1) + (a2 + a3);
  };
  float m = -INFINITY;
  for (int j = 0; j <= qi; ++j) m = fmaxf(m, score(j));
#pragma unroll
  for (int d = 0; d < D; ++d) o[d] = 0.f;
  float l = 0.f;
  for (int j = 0; j <= qi; ++j) {
    const float pj = exp2f(score(j) - m);
    l += pj;
    const float* vp = v + (row0 + j) * ld + head * D;
#pragma unroll
    for (int d = 0; d < D; d += 4) {
      const float4 vv = *reinterpret_cast<const float4*>(vp + d);
      o[d] = fmaf(pj, vv.x, o[d]); o[d + 1] = fmaf(pj, vv.y, o[d + 1]); o[d + 2] = fmaf(pj, vv.z, o[d + 2]); o[d + 3] = fmaf(pj, vv.w, o[d + 3]);
    }
  }
  const float inv = 1.f / l;
#pragma unroll
  for (int d = 0; d < D; d += 8) {
    const float v8[8] = {o[d] * inv, o[d + 1] * inv, o[d + 2] * inv, o[d + 3] * inv,
                         o[d + 4] * inv, o[d + 5] * inv, o[d + 6] * inv, o[d + 7] * inv};
    store_op<OP>(out, (size_t)(row0 + qi), heads * D, head * D + d, v8);
  }
}

// The parity-mode launchers behind pn_attention / pn_attention_temporal / pn_attention_causal (declared in common.cuh):
// those entry points check operand_mode and call them for the two modes below.
using F32Modes = OperandModes<PN_OPERAND_SPLIT3, PN_OPERAND_F32>;

int attention_causal_f32(const float* q, const float* k, const float* v, void* out, int64_t batch, int64_t L, int32_t heads,
                         int32_t head_dim, int64_t ld, int64_t out_ld, float scale, int operand_mode, void* stream_v) {
  PN_REQUIRE(q && k && v && out, "pn_attention_causal: null pointer");
  PN_REQUIRE(head_dim == 64, "pn_attention_causal: head_dim %d unsupported (64)", head_dim);
  PN_REQUIRE(batch > 0 && L >= 1 && L <= 128 && heads > 0, "pn_attention_causal: bad geometry (1 <= L <= 128)");
  PN_REQUIRE(ld % 4 == 0 && ld >= (int64_t)heads * head_dim, "pn_attention_causal: bad token stride");
  PN_REQUIRE(out_ld == (int64_t)heads * head_dim, "pn_attention_causal: out_ld must equal heads*head_dim (dense operand)");
  const long long total = batch * heads * L;
  const long long blocks = (total + 127) / 128;
  PN_REQUIRE(blocks < (1ll << 31), "pn_attention_causal: grid too large");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  PN_DISPATCH_OP(F32Modes, operand_mode, attn_f32_causal_kernel<OP><<<(unsigned)blocks, 128, 0, st>>>(q, k, v, out, (int)batch, (int)L, heads, ld,
                                                                                         scale * 1.4426950408889634f));
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}

int attention_f32(const pn_attn_args* a, int operand_mode, void* stream_v) {
  if (a == nullptr) return fail(PN_ERR_INVALID, "pn_attention: null args");
  PN_REQUIRE(a->q && a->k && a->v && a->out, "pn_attention: null tensor pointer");
  PN_REQUIRE(a->head_dim == 64 || a->head_dim == 80, "pn_attention: head_dim %d unsupported (64 or 80)", a->head_dim);
  PN_REQUIRE(a->heads > 0 && a->F > 0 && a->H > 0 && a->V > 0 && a->V <= 8 && a->W > 0, "pn_attention: bad query geometry");
  PN_REQUIRE(a->Hk > 0 && a->Vk > 0 && a->Vk <= 8 && a->Wk > 0 && a->kv_frame_div > 0, "pn_attention: bad key geometry");
  PN_REQUIRE(a->q_ld % 4 == 0 && a->kv_ld % 4 == 0, "pn_attention: fp32 token strides must be multiples of 4 floats");
  PN_REQUIRE(a->out_ld == (int64_t)a->heads * a->head_dim, "pn_attention: out_ld must equal heads*head_dim (dense operand)");
  AfParams p;
  std::memset(&p, 0, sizeof(p));
  p.q = reinterpret_cast<const float*>(a->q); p.k = reinterpret_cast<const float*>(a->k); p.v = reinterpret_cast<const float*>(a->v);
  p.out = a->out;
  p.q_ld = a->q_ld; p.kv_ld = a->kv_ld; p.out_C = (int)a->out_ld;
  p.F = (int)a->F; p.H = (int)a->H; p.V = (int)a->V; p.W = (int)a->W;
  p.Hk = (int)a->Hk; p.Vk = (int)a->Vk; p.Wk = (int)a->Wk;
  p.kv_frame_div = a->kv_frame_div; p.heads = a->heads;
  for (int v = 0; v < a->V; ++v) {
    const int cnt = a->kv_view_count[v];
    PN_REQUIRE(cnt >= 1 && cnt <= 2, "pn_attention: kv_view_count[%d]=%d must be 1 or 2", v, cnt);
    p.kv_view_count[v] = cnt;
    for (int i = 0; i < cnt; ++i) {
      PN_REQUIRE(a->kv_views[v][i] >= 0 && a->kv_views[v][i] < a->Vk, "pn_attention: kv view out of range");
      p.kv_views[v][i] = a->kv_views[v][i];
    }
  }
  p.scale_log2 = a->scale * 1.4426950408889634f;
  const long long tiles = (a->H * a->W + AF_QTILE - 1) / AF_QTILE;
  const long long blocks = tiles * a->heads * a->V * a->F;
  PN_REQUIRE(blocks > 0 && blocks < (1ll << 31), "pn_attention: grid too large");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  if (a->head_dim == 64) PN_DISPATCH_OP(F32Modes, operand_mode, attn_f32_view_kernel<64, OP><<<(unsigned)blocks, AF_QTILE, 0, st>>>(p));
  else PN_DISPATCH_OP(F32Modes, operand_mode, attn_f32_view_kernel<80, OP><<<(unsigned)blocks, AF_QTILE, 0, st>>>(p));
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}

int attention_temporal_f32(const float* q, const float* k, const float* v, void* out, int64_t batch, int64_t T, int64_t pixels,
                           int32_t heads, int32_t head_dim, int64_t ld, int64_t out_ld, float scale, int operand_mode,
                           void* stream_v) {
  PN_REQUIRE(q && k && v && out, "pn_attention_temporal: null pointer");
  PN_REQUIRE(head_dim == 64 || head_dim == 80, "pn_attention_temporal: head_dim %d unsupported (64 or 80)", head_dim);
  PN_REQUIRE(batch > 0 && T > 0 && T <= 16 && pixels > 0 && heads > 0, "pn_attention_temporal: bad geometry (T <= 16)");
  PN_REQUIRE(ld % 4 == 0 && ld >= (int64_t)heads * head_dim, "pn_attention_temporal: bad token stride");
  PN_REQUIRE(out_ld == (int64_t)heads * head_dim, "pn_attention_temporal: out_ld must equal heads*head_dim (dense operand)");
  const long long total = batch * T * pixels * heads;
  const long long blocks = (total + 127) / 128;
  PN_REQUIRE(blocks < (1ll << 31), "pn_attention_temporal: grid too large");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  const float sl2 = scale * 1.4426950408889634f;
  if (head_dim == 64)
    PN_DISPATCH_OP(F32Modes, operand_mode, attn_f32_temporal_kernel<64, OP><<<(unsigned)blocks, 128, 0, st>>>(q, k, v, out, (int)batch, (int)T, (int)pixels, heads, ld, sl2));
  else
    PN_DISPATCH_OP(F32Modes, operand_mode, attn_f32_temporal_kernel<80, OP><<<(unsigned)blocks, 128, 0, st>>>(q, k, v, out, (int)batch, (int)T, (int)pixels, heads, ld, sl2));
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}

}  // namespace pn
