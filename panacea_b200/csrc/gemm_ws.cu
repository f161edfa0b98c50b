// Persistent, weight-stationary wgmma GEMM for 1x1 GEMMs over dense rows with K = C <= 320 and N % 160 == 0 (the
// level-0 transformer linears and zero convs). pn_gemm (gemm_tc.cu) selects it from the call's shape.
//
// At K <= 320 a tile's MMAs are short and its epilogue (residual read, output write) is most of its time, so
// gemm_tc_kernel's one-tile CTAs spend it re-reading the same weight tile, re-filling their ring and running the
// epilogue in the warps that issue the MMAs. Here:
//   * one CTA per SM owns one 160-column tile of W, loads it once (up to 5 [160, 64] boxes, 100 KB) and keeps it while
//     it walks 64-row tiles. CTA c takes column c % tiles_col and row tiles g, g + G, g + 2G, ... (g = c / tiles_col,
//     G = grid / tiles_col), so all column tiles work on the same window of rows at the same time and A is read from
//     HBM about once. The grid is G * tiles_col with G = SMs / tiles_col: when tiles_col does not divide the SM count
//     the remaining SMs stay idle (4 of 132 for tiles_col = 16, none for 2 and 6);
//   * warpgroup 2 produces: one thread issues the A boxes of each row tile into a 5-stage ring, another the tile's
//     residual into the staging buffer of the warpgroup that will run its epilogue, and a warp computes the folded
//     LayerNorm's row coefficients into shared memory;
//   * warpgroups 0 and 1 take alternate row tiles: while one runs its epilogue the other issues its MMAs (m64n160k16,
//     A from the ring, B the resident W). The epilogue reads the residual from shared memory, writes the result back
//     into the same staging buffer and stores it with TMA, so the tile's HBM traffic is in flight as bulk copies
//     instead of register loads. A tile's residual is read before its store and no other tile touches its rows, so
//     `out == residual` stays exact.
// The per-element arithmetic is gemm_epilogue.cuh's, in the same order as gemm_tc_kernel's, and an output element's
// MMAs are the same k-ordered m64n160k16 chain, so both kernels give bitwise identical results.
#include <algorithm>

#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

namespace {
constexpr int WS_BN = 160, WS_BM = 64, WS_BK = 64;
constexpr int WS_MAX_KB = 5;                        // C <= 320
// One row tile of A at C = 320. Ten stages (two tiles, with 20 KB bf16 staging buffers) measured slower.
constexpr int WS_STAGES = 5;
// Two consumer warpgroups and a producer warpgroup of which two threads and a warp work: three warps on each SM sub-partition, so
// a thread may hold 168 registers (16,384 / (3 * 32)), which the 80-float accumulator and the epilogue fit unspilled.
constexpr int WS_THREADS = 384;
constexpr int W_BOX = WS_BN * WS_BK * 2;            // 20 KB
constexpr int A_BOX = WS_BM * WS_BK * 2;            // 8 KB
constexpr int STAGING = WS_BM * WS_BN * 4;          // one fp32 64 x 160 tile
constexpr int OFF_A = WS_MAX_KB * W_BOX;
constexpr int OFF_STAGING = OFF_A + WS_STAGES * A_BOX;
constexpr int OFF_BAR = OFF_STAGING + 2 * STAGING;
constexpr int OFF_VEC = OFF_BAR + 32 * 8;           // bias and LayerNorm column sums of the CTA's 160 columns
constexpr int OFF_COEF = OFF_VEC + 2 * WS_BN * 4;   // LayerNorm (a, b) of the 64 rows of each warpgroup's tile
constexpr int WS_SMEM = OFF_COEF + 2 * WS_BM * 8 + 1024;   // + alignment slack of the dynamic window
static_assert(WS_SMEM <= 227 * 1024, "the weight tile, the A ring and two staging tiles must fit one SM");

// Staging tiles are TMA boxes of 64 rows x R bytes (R = 128 / 64 / 32 with the matching 128B / 64B / 32B swizzle),
// side by side. Byte `b` of tile row r sits in box b / R; the swizzle XORs its 16-byte chunk with address bits 7 and up,
// which spreads a warp's 8 rows over the banks.
template <int R>
__device__ __forceinline__ int stage_off(int r, int b) {
  const int w = b % R;
  return (b / R) * (WS_BM * R) + r * R + ((((w >> 4) ^ ((r * R) >> 7)) & (R / 16 - 1)) << 4) + (w & 15);
}
}  // namespace

struct GemmWsParams {
  GemmParams p;                  // mapA: 2-D [rows, C] with [64, 64] boxes; mapB, epilogue fields as for gemm_tc_kernel
  CUtensorMap mapOut, mapRes;    // [rows, ldo] / [rows, ldr] with 32-column boxes (16 for GEGLU's output)
  int M, row_tiles, groups, kc;
};

template <int MODE>    // MODE: an EpiMode
__global__ void __launch_bounds__(WS_THREADS, 1) gemm_ws_kernel(const __grid_constant__ GemmWsParams q) {
  const GemmParams& p = q.p;
  constexpr int NJ = WS_BN / 8;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* full = w_full + 1;
  uint64_t* empty = full + WS_STAGES;
  uint64_t* res_full = empty + WS_STAGES;
  uint64_t* res_empty = res_full + 2;
  uint64_t* mma_turn = res_empty + 2;
  uint64_t* coef_full = mma_turn + 2;
  uint64_t* coef_empty = coef_full + 2;
  float* s_bias = reinterpret_cast<float*>(smem + OFF_VEC);
  float* s_colsum = s_bias + WS_BN;
  float2* s_coef = reinterpret_cast<float2*>(smem + OFF_COEF);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int col = blockIdx.x % p.tiles_col;
  const int grp = blockIdx.x / p.tiles_col;
  const bool has_res = MODE != EPI_GEGLU && p.residual != nullptr;
  const bool res_bf16 = MODE == EPI_BF16 && p.res_bf16;
  const bool ln = MODE == EPI_BF16 && p.ln_stats_in != nullptr;

  // The column vectors are the same for every row tile of the CTA. Read in the epilogue straight from global memory,
  // under the kernel's own HBM traffic, they cost a memory round trip per tile.
  if (threadIdx.x < WS_BN) {
    s_bias[threadIdx.x] = p.bias != nullptr ? p.bias[col * WS_BN + threadIdx.x] : 0.f;
    s_colsum[threadIdx.x] = ln ? p.ln_colsum[col * WS_BN + threadIdx.x] : 0.f;
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.mapA);
    tma_prefetch_desc(&p.mapB);
    tma_prefetch_desc(&q.mapOut);
    if (has_res) tma_prefetch_desc(&q.mapRes);
    mbar_init(w_full, 1);
    for (int i = 0; i < WS_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
    for (int i = 0; i < 2; ++i) { mbar_init(&res_full[i], 1); mbar_init(&res_empty[i], 1); mbar_init(&mma_turn[i], 1);
      mbar_init(&coef_full[i], 1); mbar_init(&coef_empty[i], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // ===================== producers: one thread of warp 8 (W, A) and one of warp 9 (residuals) =====================
  // Two independent threads: a residual waits for its staging buffer (the warpgroup's previous store), and that wait
  // must not hold back the A boxes of the tiles in between.
  if (warp >= 8) {
    if (warp == 8 && lane == 0) {
      mbar_arrive_expect_tx(w_full, q.kc * W_BOX);
      for (int kb = 0; kb < q.kc; ++kb) tma_load_2d(smem + kb * W_BOX, &p.mapB, w_full, kb * WS_BK, col * WS_BN);
      int stage = 0;
      uint32_t phase = 0;
      for (int t = 0;; ++t) {
        const int rt = grp + t * q.groups;
        if (rt >= q.row_tiles) break;
        for (int kb = 0; kb < q.kc; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], A_BOX);
          tma_load_2d(smem + OFF_A + stage * A_BOX, &p.mapA, &full[stage], kb * WS_BK, rt * WS_BM);
          if (++stage == WS_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (warp == 9 && lane == 0 && has_res) {
      const int res_bytes = res_bf16 ? WS_BM * WS_BN * 2 : WS_BM * WS_BN * 4;
      const int box = res_bf16 ? WS_BM * 64 : WS_BM * 128;
      for (int t = 0;; ++t) {
        const int rt = grp + t * q.groups;
        if (rt >= q.row_tiles) break;
        const int wg = t & 1;
        const uint32_t use = t >> 1;
        uint8_t* stg = smem + OFF_STAGING + wg * STAGING;
        mbar_wait(&res_empty[wg], (use & 1) ^ 1);
        mbar_arrive_expect_tx(&res_full[wg], res_bytes);
        for (int b = 0; b < WS_BN / 32; ++b)
          tma_load_2d(stg + b * box, &q.mapRes, &res_full[wg], col * WS_BN + 32 * b, rt * WS_BM);
      }
    } else if (warp == 10 && ln) {
      // the folded LayerNorm's row coefficients of each tile, ahead of its epilogue (their partial sums are another
      // dependent global round trip per row)
      for (int t = 0;; ++t) {
        const int rt = grp + t * q.groups;
        if (rt >= q.row_tiles) break;
        const int wg = t & 1;
        const uint32_t use = t >> 1;
        mbar_wait(&coef_empty[wg], (use & 1) ^ 1);
        for (int r = lane; r < WS_BM; r += 32) {
          const long long row = (long long)rt * WS_BM + r;
          float a = 1.f, b = 0.f;
          if (row < q.M) ln_row_coeffs(p, row, a, b);
          s_coef[wg * WS_BM + r] = make_float2(a, b);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&coef_full[wg]);
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  const bool issuer = (threadIdx.x & 127) == 0;
  uint8_t* stg = smem + OFF_STAGING + wg * STAGING;
  const uint32_t base = smem_u32(smem);
  const uint64_t descA0 = wgmma_desc(base + OFF_A, 16, 1024, kSw128);
  const uint64_t descW0 = wgmma_desc(base, 16, 1024, kSw128);
  const int quad = lane & 3;
  const int r0 = (warp & 3) * 16 + (lane >> 2);          // this thread's tile rows: r0 and r0 + 8
  const int n_base = col * WS_BN + 2 * quad;
  // Not zero-filled: each tile's first wgmma runs with scale-d = 0 (see gemm_tc_kernel).
  float acc[WS_BN / 2];
  mbar_wait(w_full, 0);

  for (int t = wg;; t += 2) {
    const int rt = grp + t * q.groups;
    if (rt >= q.row_tiles) break;
    const uint32_t use = t >> 1;
    {
      // The warpgroups take turns: tile t's MMAs start once tile t - 1's have retired. Both read one ring, and a parity
      // wait is only unambiguous on a barrier at most one phase ahead of the waiter: the turn guarantees that every
      // earlier use of this tile's stages has been waited for. (Tile 0's wait, parity 1 on a fresh barrier, passes.)
      mbar_wait(&mma_turn[wg], (use & 1) ^ (wg == 0 ? 1u : 0u));
      const int g = t * q.kc;                            // the ring's k-block count before this tile
      int stage = g % WS_STAGES, prev = 0;
      uint32_t phase = (g / WS_STAGES) & 1;
      for (int kb = 0; kb < q.kc; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < WS_BK / 16; ++k)
          wgmma_ss<WS_BN>(acc, descA0 + (A_BOX >> 4) * stage + 2 * k, descW0 + (W_BOX >> 4) * kb + 2 * k,
                          (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (kb > 0 && issuer) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == WS_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (issuer) {
        mbar_arrive(&empty[prev]);
        mbar_arrive(&mma_turn[wg ^ 1]);
      }
    }

    // ---------- epilogue: rows r0, r0 + 8 of the tile, columns 8j + 2 quad + {0, 1} ----------
    long long grow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long row = (long long)rt * WS_BM + r0 + 8 * h;
      grow[h] = row < q.M ? row : -1;
    }
    const float* rv_row[2];
    rowvec_rows(p, grow, n_base, rv_row);

    if (MODE == EPI_GEGLU) {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        if ((j & 3) >= 2) continue;
        const float2 bv = *reinterpret_cast<const float2*>(s_bias + 2 * quad + 8 * j);
        const float2 bg = *reinterpret_cast<const float2*>(s_bias + 2 * quad + 8 * j + 16);
#pragma unroll
        for (int h = 0; h < 2; ++h) geglu_add(acc, j, h, bv, bg);
      }
      if (p.rowvec != nullptr) {
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          if ((j & 3) >= 2) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
            if (grow[h] >= 0) {
              const float* rv = rv_row[h] + 8 * j;
              t = make_float4(rv[0], rv[1], rv[16], rv[17]);
            }
            geglu_add(acc, j, h, make_float2(t.x, t.y), make_float2(t.z, t.w));
          }
        }
      }
      if (issuer) bulk_wait_read_all();                 // the previous tile's store has left the staging buffer
      named_barrier_sync(1 + wg, 128);
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        if ((j & 3) >= 2) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<uint32_t*>(stg + stage_off<32>(r0 + 8 * h, 2 * geglu_out_col(j, quad))) = geglu_out(acc, j, h);
      }
      fence_proxy_async_smem();
      named_barrier_sync(1 + wg, 128);
      if (issuer) {
        for (int b = 0; b < WS_BN / 32; ++b) tma_store_2d(&q.mapOut, stg + b * (WS_BM * 32), col * (WS_BN / 2) + 16 * b, rt * WS_BM);
        bulk_commit();
      }
      continue;
    }

    float ln_a[2] = {1.f, 1.f}, ln_b[2] = {0.f, 0.f};
    if (ln) {
      mbar_wait(&coef_full[wg], use & 1);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float2 c = s_coef[wg * WS_BM + r0 + 8 * h];
        ln_a[h] = c.x;
        ln_b[h] = c.y;
      }
    }
    if (has_res) mbar_wait(&res_full[wg], use & 1);
    // each column block takes every term in turn: bias or the folded LayerNorm, row vector, residual (rows past the
    // matrix are TMA's zero fill), second residual
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const float2 b2 = *reinterpret_cast<const float2*>(s_bias + 2 * quad + 8 * j);
      const float2 s2 = *reinterpret_cast<const float2*>(s_colsum + 2 * quad + 8 * j);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float &v0 = acc[4 * j + 2 * h], &v1 = acc[4 * j + 2 * h + 1];
        epi_bias(v0, v1, b2, s2, ln, ln_a[h], ln_b[h]);
        if (p.rowvec != nullptr) {
          float2 t2 = make_float2(0.f, 0.f);
          if (grow[h] >= 0) t2 = *reinterpret_cast<const float2*>(rv_row[h] + 8 * j);
          epi_add(v0, v1, t2);
        }
        if (has_res) {
          const int r = r0 + 8 * h, c = 8 * j + 2 * quad;
          epi_add(v0, v1, res_bf16 ? __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(stg + stage_off<64>(r, 2 * c)))
                                   : *reinterpret_cast<const float2*>(stg + stage_off<128>(r, 4 * c)));
        }
        if (MODE == EPI_F32 && p.residual2 != nullptr) {
          float2 t2 = make_float2(0.f, 0.f);
          if (grow[h] >= 0) t2 = *reinterpret_cast<const float2*>(p.residual2 + grow[h] * p.ldr2 + n_base + 8 * j);
          epi_add(v0, v1, t2);
        }
      }
    }
    if (issuer) bulk_wait_read_all();
    named_barrier_sync(1 + wg, 128);                    // every thread has read its residual before any overwrites it
    if (ln && issuer) mbar_arrive(&coef_empty[wg]);

    float st_sum[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, st_sq[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // [row][column half]
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h, c = 8 * j + 2 * quad;
        const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (MODE == EPI_F32) {
          *reinterpret_cast<float2*>(stg + stage_off<128>(r, 4 * c)) = make_float2(v0, v1);
        } else {
          *reinterpret_cast<uint32_t*>(stg + stage_off<64>(r, 2 * c)) = pack_bf16x2(v0, v1);
          row_stats_add<NJ>(st_sum, st_sq, h, j, v0, v1);
        }
      }
    fence_proxy_async_smem();
    named_barrier_sync(1 + wg, 128);
    if (issuer) {
      const int box = MODE == EPI_F32 ? WS_BM * 128 : WS_BM * 64;
      for (int b = 0; b < WS_BN / 32; ++b) tma_store_2d(&q.mapOut, stg + b * box, col * WS_BN + 32 * b, rt * WS_BM);
      bulk_commit();
      if (has_res) {                                    // hand the staging buffer back for this warpgroup's next residual
        bulk_wait_read_all();
        mbar_arrive(&res_empty[wg]);
      }
    }
    if (MODE == EPI_BF16 && p.ln_stats_out != nullptr) row_stats_store(p, st_sum, st_sq, grow, col, quad);
  }
  if (issuer) bulk_wait_all();
}

int launch_gemm_ws(GemmParams& p, EpiMode mode, const void* A, long long rows, long long row_stride, int C, cudaStream_t stream) {
  GemmWsParams q;
  std::memset(&q, 0, sizeof(q));
  const uint64_t dimsA[2] = {(uint64_t)C, (uint64_t)rows};
  const uint64_t strA[1] = {(uint64_t)row_stride};
  const uint32_t boxA[2] = {(uint32_t)WS_BK, (uint32_t)WS_BM};
  int rc = cached_tmap_bf16(&p.mapA, A, 2, dimsA, strA, boxA, 128);
  if (rc != PN_OK) return rc;
  const uint64_t n_out = mode == EPI_GEGLU ? p.N / 2 : p.N;
  if (mode == EPI_F32) {
    rc = cached_tmap_f32_2d(&q.mapOut, p.out, n_out, rows, p.ldo, WS_BM);
  } else {
    const uint64_t dims[2] = {n_out, (uint64_t)rows};
    const uint64_t str[1] = {(uint64_t)p.ldo};
    const uint32_t box[2] = {mode == EPI_GEGLU ? 16u : 32u, (uint32_t)WS_BM};
    rc = cached_tmap_bf16(&q.mapOut, p.out, 2, dims, str, box, mode == EPI_GEGLU ? 32 : 64);
  }
  if (rc != PN_OK) return rc;
  if (p.residual != nullptr) {
    if (p.res_bf16) {
      const uint64_t dims[2] = {(uint64_t)p.N, (uint64_t)rows};
      const uint64_t str[1] = {(uint64_t)p.ldr};
      const uint32_t box[2] = {32u, (uint32_t)WS_BM};
      rc = cached_tmap_bf16(&q.mapRes, p.residual, 2, dims, str, box, 64);
    } else {
      rc = cached_tmap_f32_2d(&q.mapRes, p.residual, p.N, rows, p.ldr, WS_BM);
    }
    if (rc != PN_OK) return rc;
  }
  q.p = p;
  q.M = (int)rows;
  q.row_tiles = (int)((rows + WS_BM - 1) / WS_BM);
  q.groups = std::min(sm_count() / p.tiles_col, q.row_tiles);
  q.kc = C / WS_BK;
  void (*kern)(GemmWsParams) = mode == EPI_GEGLU ? gemm_ws_kernel<EPI_GEGLU>
                              : mode == EPI_BF16 ? gemm_ws_kernel<EPI_BF16> : gemm_ws_kernel<EPI_F32>;
  rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), WS_SMEM);
  if (rc != PN_OK) return rc;
  kern<<<(unsigned)(q.groups * p.tiles_col), WS_THREADS, WS_SMEM, stream>>>(q);
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}

}  // namespace pn
