// Cross-frame (temporal) self-attention: every pixel attends over its T <= 16 frames (attention.py:1116-1125 feeding
// CrossAttention.forward :229-291 with context=None). Sequences this short cannot fill a 64-row wgmma tile (wgmma needs
// M = 64 rows of ONE problem), so each warp runs one (sequence b, pixel p, head) problem on the warp-level tensor path:
// S = Q K^T as m16n8k16 bf16 MMAs (4 per 8 keys), fp32 softmax on the accumulator fragment, O = P V as 8 more MMAs with
// the S fragment re-used as the A operand. The op is HBM-bound (reads q,k,v once, writes o once); the scalar version of
// this kernel spent ~800 instructions per problem and ran at a third of that roofline.
//
// Layout: qkv bf16 [b, T, P, ld] with q/k/v at channel offsets given by the three base pointers; the
// "(b t)(h w) c -> (b h w) t c" rearrangement of the reference is just this indexing — nothing is copied.
#include "common.cuh"
#include "ptx.cuh"
#include "operand.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

constexpr int TA_MAXT = 16;
constexpr int TA_WARPS = 4;
// row pitch D + 8 elements (144 B for head_dim 64, 176 B for 80): 16-B aligned, 8 consecutive rows start in 8 different
// 4-bank groups (conflict-free ldmatrix)

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x2(uint32_t (&r)[2], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t (&r)[2], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(smem_u32(p)));
}
// D (16x8 fp32) += A (16x16 bf16, row) * B (16x8 bf16, col)
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int D>
__global__ void __launch_bounds__(TA_WARPS * 32) attn_temporal_kernel(const __nv_bfloat16* __restrict__ q,
                                                                      const __nv_bfloat16* __restrict__ k,
                                                                      const __nv_bfloat16* __restrict__ v,
                                                                      __nv_bfloat16* __restrict__ out, int nb, int T, int P,
                                                                      int heads, long long ld, long long out_ld, float scale) {
  constexpr int TA_PITCH = D + 8;
  constexpr int RCH = D / 8;            // 16-byte chunks per row
  __shared__ __align__(16) __nv_bfloat16 sq[TA_WARPS][TA_MAXT][TA_PITCH];   // Q rows, later the output rows
  __shared__ __align__(16) __nv_bfloat16 sk[TA_WARPS][TA_MAXT][TA_PITCH];
  __shared__ __align__(16) __nv_bfloat16 sv[TA_WARPS][TA_MAXT][TA_PITCH];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long item = (long long)blockIdx.x * TA_WARPS + w;
  const long long total = (long long)nb * P * heads;
  if (item >= total) return;   // whole warp exits together
  const int head = (int)(item % heads);
  const long long bp = item / heads;
  const int pix = (int)(bp % P);
  const int b = (int)(bp / P);
  // rows T..15 are MMA padding: they must be finite (0 * NaN would poison the valid rows of P V)
  for (int i = lane; i < (TA_MAXT - T) * RCH; i += 32) {
    const int t = T + i / RCH, ch = i % RCH;
    *reinterpret_cast<uint4*>(&sq[w][t][ch * 8]) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(&sk[w][t][ch * 8]) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(&sv[w][t][ch * 8]) = make_uint4(0, 0, 0, 0);
  }
  // stage q,k,v rows: each row is D bf16 = RCH x 16 B; consecutive lanes take consecutive chunks
  for (int i = lane; i < T * RCH; i += 32) {
    const int t = i / RCH, ch = i % RCH;
    const long long tok = ((long long)(b * T + t) * P + pix);
    const long long off = tok * ld + head * D + ch * 8;
    *reinterpret_cast<uint4*>(&sq[w][t][ch * 8]) = *reinterpret_cast<const uint4*>(q + off);
    *reinterpret_cast<uint4*>(&sk[w][t][ch * 8]) = *reinterpret_cast<const uint4*>(k + off);
    *reinterpret_cast<uint4*>(&sv[w][t][ch * 8]) = *reinterpret_cast<const uint4*>(v + off);
  }
  __syncwarp();
  const int ntile = T > 8 ? 2 : 1;             // key tiles of 8
  const int r0 = lane >> 2, cq = (lane & 3) * 2;   // accumulator fragment: rows r0, r0+8; columns cq, cq+1 of a tile

  // ---- S = Q K^T (16 x 8*ntile), fp32
  float sacc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk) {
    uint32_t aq[4];
    ldmatrix_x4(aq, &sq[w][lane & 15][kk * 16 + (lane >> 4) * 8]);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      if (nt < ntile) {
        uint32_t bk[2];
        ldmatrix_x2(bk, &sk[w][nt * 8 + (lane & 7)][kk * 16 + ((lane >> 3) & 1) * 8]);
        mma_16816(sacc[nt], aq, bk);
      }
    }
  }
  // ---- softmax over the keys of each query row (rows r0 and r0+8 of this lane; a row lives in the 4 lanes of a quad)
  const float c = scale * 1.4426950408889634f;
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool ok = nt < ntile && nt * 8 + cq + e < T;
      if (!ok) { sacc[nt][e] = -INFINITY; sacc[nt][2 + e] = -INFINITY; }
      mx0 = fmaxf(mx0, sacc[nt][e]);
      mx1 = fmaxf(mx1, sacc[nt][2 + e]);
    }
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      sacc[nt][e] = ex2_approx((sacc[nt][e] - mx0) * c);            // exp2(-inf) = 0 for the masked keys
      sacc[nt][2 + e] = ex2_approx((sacc[nt][2 + e] - mx1) * c);
      sum0 += sacc[nt][e];
      sum1 += sacc[nt][2 + e];
    }
  }
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
  const float inv0 = 1.f / sum0, inv1 = 1.f / sum1;
  // the S accumulator fragment IS the A fragment of P (16 queries x 16 keys)
  uint32_t ap[4] = {pack_bf16x2(sacc[0][0], sacc[0][1]), pack_bf16x2(sacc[0][2], sacc[0][3]),
                    pack_bf16x2(sacc[1][0], sacc[1][1]), pack_bf16x2(sacc[1][2], sacc[1][3])};
  __syncwarp();                                 // every lane has read its Q fragments: sq becomes the output staging
  // ---- O = P V (16 x D): D/8 channel tiles of 8, V rows (keys) x channels read transposed
#pragma unroll
  for (int nd = 0; nd < D / 8; ++nd) {
    uint32_t bv[2];
    ldmatrix_x2_trans(bv, &sv[w][lane & 15][nd * 8]);
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    mma_16816(o, ap, bv);
    *reinterpret_cast<uint32_t*>(&sq[w][r0][nd * 8 + cq]) = pack_bf16x2(o[0] * inv0, o[1] * inv0);
    *reinterpret_cast<uint32_t*>(&sq[w][r0 + 8][nd * 8 + cq]) = pack_bf16x2(o[2] * inv1, o[3] * inv1);
  }
  __syncwarp();
  for (int i = lane; i < T * RCH; i += 32) {
    const int t = i / RCH, ch = i % RCH;
    const long long tok = ((long long)(b * T + t) * P + pix);
    *reinterpret_cast<uint4*>(out + tok * out_ld + head * D + ch * 8) = *reinterpret_cast<const uint4*>(&sq[w][t][ch * 8]);
  }
}

// Causal self-attention over one short sequence per (batch, head): the text transformer of the OpenCLIP embedder
// (open_clip ResidualAttentionBlock with attn_mask = -inf above the diagonal, L = 77). One CTA per (batch, head) stages
// the L <= 128 rows of q, k and v once in shared memory; warp w owns query rows [16 w, 16 w + 16) and only visits the
// key tiles its rows can see (keys <= its last row). S = Q K^T, the masked fp32 softmax and O = P V follow the
// temporal kernel above, with P fed back as the A operand in chunks of 16 keys.
constexpr int CA_MAXL = 128;
constexpr int CA_D = 64;
constexpr int CA_PITCH = CA_D + 8;

__global__ void __launch_bounds__((CA_MAXL / 16) * 32) attn_causal_kernel(const __nv_bfloat16* __restrict__ q,
                                                                          const __nv_bfloat16* __restrict__ k,
                                                                          const __nv_bfloat16* __restrict__ v,
                                                                          __nv_bfloat16* __restrict__ out, int L, int heads,
                                                                          long long ld, long long out_ld, float scale) {
  constexpr int RCH = CA_D / 8;
  extern __shared__ __align__(16) unsigned char ca_smem[];
  const int Lp = (L + 15) & ~15;
  __nv_bfloat16 (*sq)[CA_PITCH] = reinterpret_cast<__nv_bfloat16 (*)[CA_PITCH]>(ca_smem);   // Q rows, later the output
  __nv_bfloat16 (*sk)[CA_PITCH] = sq + Lp;
  __nv_bfloat16 (*sv)[CA_PITCH] = sk + Lp;
  const int head = blockIdx.x % heads, b = blockIdx.x / heads;
  const long long row0 = (long long)b * L;
  // rows L..Lp-1 are MMA padding: they must be finite (0 * NaN would poison the valid rows of P V)
  for (int i = threadIdx.x; i < Lp * RCH; i += blockDim.x) {
    const int t = i / RCH, ch = i % RCH;
    uint4 zq = make_uint4(0, 0, 0, 0), zk = zq, zv = zq;
    if (t < L) {
      const long long off = (row0 + t) * ld + head * CA_D + ch * 8;
      zq = *reinterpret_cast<const uint4*>(q + off);
      zk = *reinterpret_cast<const uint4*>(k + off);
      zv = *reinterpret_cast<const uint4*>(v + off);
    }
    *reinterpret_cast<uint4*>(&sq[t][ch * 8]) = zq;
    *reinterpret_cast<uint4*>(&sk[t][ch * 8]) = zk;
    *reinterpret_cast<uint4*>(&sv[t][ch * 8]) = zv;
  }
  __syncthreads();
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qb = w * 16;                                    // first query row of this warp
  const int ntile = min((L + 7) / 8, (qb + 16) / 8);        // key tiles of 8 that hold a key some row here may see
  const int r0 = qb + (lane >> 2), cq = (lane & 3) * 2;     // accumulator fragment: rows r0, r0+8; columns cq, cq+1

  // ---- S = Q K^T (16 x 8*ntile), fp32
  float sacc[CA_MAXL / 8][4];
#pragma unroll
  for (int nt = 0; nt < CA_MAXL / 8; ++nt) sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < CA_D / 16; ++kk) {
    uint32_t aq[4];
    ldmatrix_x4(aq, &sq[qb + (lane & 15)][kk * 16 + (lane >> 4) * 8]);
#pragma unroll
    for (int nt = 0; nt < CA_MAXL / 8; ++nt) {
      if (nt < ntile) {
        uint32_t bk[2];
        ldmatrix_x2(bk, &sk[nt * 8 + (lane & 7)][kk * 16 + ((lane >> 3) & 1) * 8]);
        mma_16816(sacc[nt], aq, bk);
      }
    }
  }
  // ---- causal mask (key > query, key >= L, unvisited tiles) and softmax on the fragment
  const float c = scale * 1.4426950408889634f;
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int nt = 0; nt < CA_MAXL / 8; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int key = nt * 8 + cq + e;
      const bool vis = nt < ntile && key < L;
      if (!(vis && key <= r0)) sacc[nt][e] = -INFINITY;
      if (!(vis && key <= r0 + 8)) sacc[nt][2 + e] = -INFINITY;
      mx0 = fmaxf(mx0, sacc[nt][e]);
      mx1 = fmaxf(mx1, sacc[nt][2 + e]);
    }
  }
  // every row sees key 0, so both maxima are finite
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
  for (int nt = 0; nt < CA_MAXL / 8; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      sacc[nt][e] = ex2_approx((sacc[nt][e] - mx0) * c);            // exp2(-inf) = 0 for the masked keys
      sacc[nt][2 + e] = ex2_approx((sacc[nt][2 + e] - mx1) * c);
      sum0 += sacc[nt][e];
      sum1 += sacc[nt][2 + e];
    }
  }
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
  const float inv0 = 1.f / sum0, inv1 = 1.f / sum1;
  // ---- O = P V (16 x 64): chunks of 16 keys, the S fragments of two key tiles form the A fragment of P
  float o[CA_D / 8][4];
#pragma unroll
  for (int nd = 0; nd < CA_D / 8; ++nd) o[nd][0] = o[nd][1] = o[nd][2] = o[nd][3] = 0.f;
  const int nchunk = (ntile + 1) / 2;
#pragma unroll
  for (int kc = 0; kc < CA_MAXL / 16; ++kc) {
    if (kc < nchunk) {
      const uint32_t ap[4] = {pack_bf16x2(sacc[2 * kc][0], sacc[2 * kc][1]), pack_bf16x2(sacc[2 * kc][2], sacc[2 * kc][3]),
                              pack_bf16x2(sacc[2 * kc + 1][0], sacc[2 * kc + 1][1]),
                              pack_bf16x2(sacc[2 * kc + 1][2], sacc[2 * kc + 1][3])};
#pragma unroll
      for (int nd = 0; nd < CA_D / 8; ++nd) {
        uint32_t bv[2];
        ldmatrix_x2_trans(bv, &sv[kc * 16 + (lane & 15)][nd * 8]);
        mma_16816(o[nd], ap, bv);
      }
    }
  }
  __syncwarp();                                 // every lane has read its Q fragments: its 16 sq rows become the output
#pragma unroll
  for (int nd = 0; nd < CA_D / 8; ++nd) {
    *reinterpret_cast<uint32_t*>(&sq[r0][nd * 8 + cq]) = pack_bf16x2(o[nd][0] * inv0, o[nd][1] * inv0);
    *reinterpret_cast<uint32_t*>(&sq[r0 + 8][nd * 8 + cq]) = pack_bf16x2(o[nd][2] * inv1, o[nd][3] * inv1);
  }
  __syncwarp();
  for (int i = lane; i < 16 * RCH; i += 32) {
    const int t = qb + i / RCH, ch = i % RCH;
    if (t < L)
      *reinterpret_cast<uint4*>(out + (row0 + t) * out_ld + head * CA_D + ch * 8) = *reinterpret_cast<const uint4*>(&sq[t][ch * 8]);
  }
}

}  // namespace pn

using namespace pn;

extern "C" int pn_attention_causal(const void* q, const void* k, const void* v, void* out, int64_t batch, int64_t L,
                                   int32_t heads, int32_t head_dim, int64_t ld, int64_t out_ld, float scale, int operand_mode,
                                   void* stream_v) {
  PN_OPERAND_MODES(Modes, operand_mode, "pn_attention_causal", PN_OPERAND_BF16, PN_OPERAND_SPLIT3, PN_OPERAND_F32);
  if (operand_mode != PN_OPERAND_BF16)
    return attention_causal_f32(reinterpret_cast<const float*>(q), reinterpret_cast<const float*>(k),
                                reinterpret_cast<const float*>(v), out, batch, L, heads, head_dim, ld, out_ld, scale, operand_mode,
                                stream_v);
  PN_REQUIRE(q && k && v && out, "pn_attention_causal: null pointer");
  PN_REQUIRE(head_dim == CA_D, "pn_attention_causal: head_dim %d unsupported (64)", head_dim);
  PN_REQUIRE(L >= 1 && L <= CA_MAXL, "pn_attention_causal: L=%lld out of range 1..128", (long long)L);
  PN_REQUIRE(batch > 0 && heads > 0 && ld % 8 == 0 && out_ld % 8 == 0 && ld >= (int64_t)heads * head_dim &&
                 out_ld >= (int64_t)heads * head_dim,
             "pn_attention_causal: bad arguments (ld and out_ld multiples of 8, >= heads*64)");
  PN_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
               reinterpret_cast<uintptr_t>(out)) & 15) == 0, "pn_attention_causal: pointers must be 16-byte aligned");
  const long long blocks = batch * heads;
  PN_REQUIRE(blocks < (1ll << 31), "pn_attention_causal: grid too large");
  const int Lp = (int)((L + 15) & ~15);
  const size_t smem = (size_t)3 * Lp * CA_PITCH * sizeof(__nv_bfloat16);
  const int rc = ensure_dyn_smem(reinterpret_cast<const void*>(&attn_causal_kernel), smem);
  if (rc != PN_OK) return rc;
  attn_causal_kernel<<<(unsigned)blocks, (Lp / 16) * 32, smem, reinterpret_cast<cudaStream_t>(stream_v)>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k),
      reinterpret_cast<const __nv_bfloat16*>(v), reinterpret_cast<__nv_bfloat16*>(out), (int)L, heads, ld, out_ld, scale);
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}

extern "C" int pn_attention_temporal(const void* q, const void* k, const void* v, void* out, int64_t batch, int64_t T,
                                     int64_t pixels, int32_t heads, int32_t head_dim, int64_t ld, int64_t out_ld,
                                     float scale, int operand_mode, void* stream_v) {
  PN_OPERAND_MODES(Modes, operand_mode, "pn_attention_temporal", PN_OPERAND_BF16, PN_OPERAND_SPLIT3, PN_OPERAND_F32);
  if (operand_mode != PN_OPERAND_BF16)
    return attention_temporal_f32(reinterpret_cast<const float*>(q), reinterpret_cast<const float*>(k),
                                  reinterpret_cast<const float*>(v), out, batch, T, pixels, heads, head_dim, ld, out_ld, scale,
                                  operand_mode, stream_v);
  PN_REQUIRE(q && k && v && out, "pn_attention_temporal: null pointer");
  PN_REQUIRE(head_dim == 64 || head_dim == 80, "pn_attention_temporal: head_dim %d unsupported (64 or 80)", head_dim);
  PN_REQUIRE(T >= 1 && T <= TA_MAXT, "pn_attention_temporal: T=%lld out of range 1..16", (long long)T);
  PN_REQUIRE(batch > 0 && pixels > 0 && heads > 0 && ld % 8 == 0 && out_ld % 2 == 0, "pn_attention_temporal: bad arguments");
  PN_REQUIRE(out_ld % 8 == 0, "pn_attention_temporal: out_ld must be a multiple of 8");
  const long long total = batch * pixels * heads;
  const long long blocks = (total + TA_WARPS - 1) / TA_WARPS;
  PN_REQUIRE(blocks < (1ll << 31), "pn_attention_temporal: grid too large");
  if (head_dim == 64)
    attn_temporal_kernel<64><<<(unsigned)blocks, TA_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream_v)>>>(
        reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k),
        reinterpret_cast<const __nv_bfloat16*>(v), reinterpret_cast<__nv_bfloat16*>(out), (int)batch, (int)T, (int)pixels, heads,
        ld, out_ld, scale);
  else
    attn_temporal_kernel<80><<<(unsigned)blocks, TA_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream_v)>>>(
        reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k),
        reinterpret_cast<const __nv_bfloat16*>(v), reinterpret_cast<__nv_bfloat16*>(out), (int)batch, (int)T, (int)pixels, heads,
        ld, out_ld, scale);
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}
