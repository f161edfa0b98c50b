// wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
//   out[row, n] = epilogue( sum_{tap, c} A[pixel(row) + tap][c] * Wt[n][tap * C + c] )
//
// A is a channels-last bf16 activation tensor [NB, H, W, C] read through ONE rank-4 TMA tensor map; the
// "taps" (1x1 for nn.Linear, 3x3 for the panorama Conv2d, 3x1 over the frame axis for the temporal
// Conv1d) are coordinate offsets of the same map, so im2col never exists in memory and the conv zero
// padding is TMA's out-of-bounds zero fill (outer panorama border only, reference: openaimodel.py:413,
// 455-462 Conv2d(padding=1) on the width-concatenated 6-view image; :418,468-476 Conv1d(k=3,padding=1)).
// B is the packed weight matrix [N, taps*C] (K-major, bf16). Accumulation is fp32 in registers.
//
// Kernel structure (one CTA per 128 x BN output tile, 256 threads, TWO CTAs per SM):
//   warps 0-3, 4-7 : two consumer warpgroups, 64 tile rows each: wgmma m64nBNk16 from the shared-memory ring,
//                    then the epilogue straight from the accumulator registers (bias / row vector / LayerNorm fold /
//                    GEGLU / residuals -> global)
//   thread 0       : also issues the TMA loads (A box [tn,th,tw,64] + B box [BN,64] per k-block, 128B swizzle): the
//                    first STAGES - 1 k-blocks up front, then one per k-block from inside the consumer loop, into the
//                    stage both warpgroups have just released.
// Two co-resident CTAs per SM let one tile's barrier set-up, first load latency and epilogue run under the other
// tile's MMAs. That needs <= 4 warps per SM sub-partition (a 9-warp CTA with a dedicated producer warp puts 5 warps on
// one sub-partition for two CTAs, capping threads at 96 registers, below the 80-float m64n160 accumulator plus
// addressing) and <= 114 KB of shared memory per CTA (3 stages at BN = 160).
// Pipeline: STAGES-deep full/empty mbarrier ring; a stage is handed back once the wgmma group that read it retired.
#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle atom row
constexpr int SM_SMEM_BYTES = 233472;      // 228 KB of shared memory per H100 SM ...
constexpr int CTA_SMEM_RESERVED = 1024;    // ... of which the system reserves 1 KB per resident CTA
constexpr int GEMM_THREADS = 256;
constexpr int GEMM_CTAS_PER_SM = 2;
// Fewest rows for which pn_gemm runs an eligible 1x1 GEMM on gemm_ws.cu's persistent kernel. With an fp32 residual at
// K = 320 (H100 80GB HBM3, 700 W) it took 7.4 / 7.9 us at 512 rows and N = 320 / 1280, against gemm_tc_kernel's 8.5 / 8.7;
// the 16-row time-embedding linear stays on gemm_tc_kernel.
constexpr long long WS_MIN_ROWS = 512;

template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;   // a multiple of 1024: every tile starts on a swizzle atom
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 2 * STAGES * 8 + 1024;
};

template <int BN, int STAGES, int MODE>    // MODE: an EpiMode
__global__ void __launch_bounds__(GEMM_THREADS, GEMM_CTAS_PER_SM) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  using S = GemmSmem<BN, STAGES>;
  constexpr int NJ = BN / 8;                   // 8-column accumulator blocks per thread row
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * S::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // column tile fastest: the CTAs that run together share an A tile in L2
  const int tcol = blockIdx.x % p.tiles_col;
  int tm = blockIdx.x / p.tiles_col;
  const int twi = tm % p.tiles_w; tm /= p.tiles_w;
  const int thi = tm % p.tiles_h;
  const int tni = tm / p.tiles_h;
  const int num_k_blocks = p.taps_h * p.taps_w * p.kc_per_tap;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.mapA);
    tma_prefetch_desc(&p.mapB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);             // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  // The next k-block to load -> (tap row, tap column, 64-channel chunk), channel chunk fastest, advanced one k-block at
  // a time. Every thread keeps it, so thread 0's loads are issued by predicate, not by branch.
  int ld_kb = 0, ld_kc = 0, ld_dx = -p.pad_w, ld_dy = -p.pad_h;
  auto load_next = [&](int stage, bool issue) {
    uint8_t* sA = smem + stage * S::STAGE_BYTES;
    tma_load_stage_if(issue, &full_bar[stage], S::STAGE_BYTES, sA, &p.mapA, ld_kc * BK, twi * p.tw + ld_dx, thi * p.th + ld_dy,
                      tni * p.tn, sA + S::A_BYTES, &p.mapB, ld_kb * BK, tcol * BN);
    ++ld_kb;
    if (++ld_kc == p.kc_per_tap) {
      ld_kc = 0;
      if (++ld_dx > p.taps_w - 1 - p.pad_w) { ld_dx = -p.pad_w; ++ld_dy; }
    }
  };
  for (int s = 0; s < STAGES - 1 && s < num_k_blocks; ++s) load_next(s, threadIdx.x == 0);

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  // Not zero-filled: a tile's first wgmma runs with scale-d = 0 and overwrites it. A fill here would be a non-wgmma
  // definition of the accumulator registers, which makes ptxas serialise every wgmma of the loop (C7515).
  float acc[BN / 2];
  {
    const uint32_t base = smem_u32(smem);
    const uint64_t descA0 = wgmma_desc(base + wg * (64 * 128), 16, 1024, kSw128);
    const uint64_t descB0 = wgmma_desc(base + S::A_BYTES, 16, 1024, kSw128);
    constexpr uint64_t STAGE_STEP = S::STAGE_BYTES >> 4;      // start-address field is in 16-byte units
    // prev = the stage of k-block kb - 1 = the stage k-block kb + STAGES - 1 is loaded into. Before the first k-block
    // it is the last, still unused stage: its empty barrier's "previous" phase (parity 1) counts as complete.
    int stage = 0, prev = STAGES - 1;
    uint32_t phase = 0, prev_phase = 1;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        wgmma_ss<BN>(acc, descA0 + STAGE_STEP * stage + 2 * k, descB0 + STAGE_STEP * stage + 2 * k, (kb > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();                         // the group of the previous k-block has retired: refill its stage
      if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      // Once BOTH warpgroups have released the stage (the empty barrier's phase for that use completes), thread 0 loads
      // k-block kb + STAGES - 1 into it. Every consumer thread waits and the load is predicated: a branch that depends
      // on the thread (or a conditional wait) while this k-block's wgmma group is in flight makes ptxas serialise the
      // wgmma instructions (C7518 / C7515).
      mbar_wait(&empty_bar[prev], prev_phase);
      load_next(prev, threadIdx.x == 0 && kb + STAGES - 1 < num_k_blocks);
      prev = stage;
      prev_phase = phase;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
  }

  // ===================== epilogue: this thread owns tile rows r0 and r0 + 8, columns 8j + 2 (lane % 4) + {0, 1} =====
  const int quad = lane & 3;
  long long grow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;   // tile rows are ordered [tn][th][tw] = TMA box order
    const int x = twi * p.tw + r % p.tw, y = thi * p.th + (r / p.tw) % p.th, n = tni * p.tn + r / (p.tw * p.th);
    grow[h] = (x < p.W && y < p.H && n < p.NB) ? ((long long)n * p.H + y) * p.W + x : -1;
  }
  const int n_base = tcol * BN + 2 * quad;
  const int n_left = p.N - n_base;                         // column block j is inside the matrix iff 8 j < n_left
  // this thread's first element (row h, column n_base) of a row-major [rows, ld] matrix; a row outside the output
  // (grow < 0) points at row 0 and is never dereferenced
  auto row_at = [&](auto* base, long long ld, int h) { return base + (grow[h] < 0 ? 0 : grow[h]) * ld + n_base; };
  const float* rv_row[2];
  rowvec_rows(p, grow, n_base, rv_row);

  // The epilogue walks the tile in chunks of CJ column blocks. For each chunk, pass one folds every term the chunk
  // reads into acc[] in place, one term after the other, so each element still sees bias (or the LayerNorm fold), row
  // vector, residual, second residual in that order; pass two stores the chunk. `out` may be `residual` (in-place
  // residual add, same leading dimension), so the compiler cannot move a load above an earlier store: stores mixed
  // with the loads made one dependent memory round trip per 8-column block and row. Pass one has no store, and each
  // term is straight-line code whose loads are predicated and whose adds are not (an element outside the matrix adds 0
  // and is never stored), so a term's loads of a chunk are in flight together. The stores between chunks keep the
  // compiler from hoisting the next chunk's loads, which bounds the registers they hold: all 80 accumulators of
  // BN = 160 are live, and two CTAs per SM allow 128 registers per thread (CJ = 4: no spills).
  // Reading a chunk's residuals before its stores is exact: each thread reads exactly the elements it later writes, and
  // no other thread writes them.
  constexpr int CJ = 4;
  static_assert(NJ % CJ == 0, "the chunks must tile the accumulator blocks");
  // acc[j][h] += row_h[8 j], row_h[8 j + 1] over the chunk's blocks, row_h = this thread's first element of its row h
  // of a float or bf16 term
  auto fold = [&](int j0, const auto* row0, const auto* row1) {
#pragma unroll
    for (int j = j0; j < j0 + CJ; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const auto* row = h == 0 ? row0 : row1;
        float2 t = make_float2(0.f, 0.f);
        if (8 * j < n_left && grow[h] >= 0) {
          if constexpr (sizeof(*row) == 2) t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + 8 * j));
          else t = *reinterpret_cast<const float2*>(row + 8 * j);
        }
        epi_add(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], t);
      }
    }
  };

  if (MODE == EPI_GEGLU) {
    static_assert(CJ == 4, "a GEGLU chunk is one group of value and gate blocks");
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
#pragma unroll
    for (int j0 = 0; j0 < NJ; j0 += CJ) {
#pragma unroll
      for (int j = j0; j < j0 + 2; ++j) {
        float2 bv = make_float2(0.f, 0.f), bg = make_float2(0.f, 0.f);
        if (p.bias != nullptr && 8 * j < n_left) {
          bv = __ldg(reinterpret_cast<const float2*>(p.bias + n_base + 8 * j));
          bg = __ldg(reinterpret_cast<const float2*>(p.bias + n_base + 8 * j + 16));
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) geglu_add(acc, j, h, bv, bg);
      }
      if (p.rowvec != nullptr) {
#pragma unroll
        for (int j = j0; j < j0 + 2; ++j) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
            if (8 * j < n_left && grow[h] >= 0) {
              const float* rv = rv_row[h] + 8 * j;
              t = make_float4(rv[0], rv[1], rv[16], rv[17]);
            }
            geglu_add(acc, j, h, make_float2(t.x, t.y), make_float2(t.z, t.w));
          }
        }
      }
#pragma unroll
      for (int j = j0; j < j0 + 2; ++j) {
        if (8 * j >= n_left) continue;
        const int no = (tcol * BN) / 2 + geglu_out_col(j, quad);
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (grow[h] >= 0) *reinterpret_cast<uint32_t*>(out + grow[h] * p.ldo + no) = geglu_out(acc, j, h);
      }
    }
    return;
  }

  float ln_a[2] = {1.f, 1.f}, ln_b[2] = {0.f, 0.f};       // folded LayerNorm: out = a * acc + b * s_n + t_n
  if (MODE == EPI_BF16 && p.ln_stats_in != nullptr) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (grow[h] >= 0) ln_row_coeffs(p, grow[h], ln_a[h], ln_b[h]);
    }
  }
  float st_sum[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, st_sq[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // [row][column half]
#pragma unroll
  for (int j0 = 0; j0 < NJ; j0 += CJ) {
    // pass one
#pragma unroll
    for (int j = j0; j < j0 + CJ; ++j) {
      float2 b2 = make_float2(0.f, 0.f), s2 = make_float2(0.f, 0.f);
      if (p.bias != nullptr && 8 * j < n_left) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + n_base + 8 * j));
      if (MODE == EPI_BF16 && p.ln_stats_in != nullptr && 8 * j < n_left)
        s2 = __ldg(reinterpret_cast<const float2*>(p.ln_colsum + n_base + 8 * j));
#pragma unroll
      for (int h = 0; h < 2; ++h)
        epi_bias(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], b2, s2, MODE == EPI_BF16 && p.ln_stats_in != nullptr, ln_a[h], ln_b[h]);
    }
    if (p.rowvec != nullptr) fold(j0, rv_row[0], rv_row[1]);
    if (p.residual != nullptr) {
      if (MODE == EPI_BF16 && p.res_bf16) {
        const __nv_bfloat16* res = reinterpret_cast<const __nv_bfloat16*>(p.residual);
        fold(j0, row_at(res, p.ldr, 0), row_at(res, p.ldr, 1));
      } else {
        const float* res = reinterpret_cast<const float*>(p.residual);
        fold(j0, row_at(res, p.ldr, 0), row_at(res, p.ldr, 1));
      }
    }
    if (MODE == EPI_F32 && p.residual2 != nullptr) fold(j0, row_at(p.residual2, p.ldr2, 0), row_at(p.residual2, p.ldr2, 1));

    // pass two
#pragma unroll
    for (int j = j0; j < j0 + CJ; ++j) {
      if (8 * j >= n_left) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (grow[h] < 0) continue;
        const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (MODE == EPI_F32) {
          *reinterpret_cast<float2*>(row_at(reinterpret_cast<float*>(p.out), p.ldo, h) + 8 * j) = make_float2(v0, v1);
        } else {
          *reinterpret_cast<uint32_t*>(row_at(reinterpret_cast<__nv_bfloat16*>(p.out), p.ldo, h) + 8 * j) = pack_bf16x2(v0, v1);
          row_stats_add<NJ>(st_sum, st_sq, h, j, v0, v1);
        }
      }
    }
  }
  if (MODE == EPI_BF16 && p.ln_stats_out != nullptr) row_stats_store(p, st_sum, st_sq, grow, tcol, quad);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// Pick the [tn, th, tw] box (product 128, powers of two) that wastes the fewest MMA rows.
static void pick_tile(long long NB, long long H, long long W, int* tw, int* th, int* tn) {
  double best = 1e30;
  for (int a = 128; a >= 1; a >>= 1) {         // tw
    for (int b = 128 / a; b >= 1; b >>= 1) {   // th
      const int c = 128 / (a * b);             // tn
      const long long tiles = ((W + a - 1) / a) * ((H + b - 1) / b) * ((NB + c - 1) / c);
      const double waste = double(tiles) * 128.0 / double(NB * H * W);
      // prefer less waste; among equals prefer the widest inner run
      const double score = waste - 1e-6 * a - 1e-9 * b;
      if (score < best) { best = score; *tw = a; *th = b; *tn = c; }
    }
  }
}

template <int BN, int STAGES>
static int launch_gemm(const GemmParams& p, EpiMode mode, long long tiles, cudaStream_t stream) {
  using S = GemmSmem<BN, STAGES>;
  static_assert(GEMM_CTAS_PER_SM * (S::TOTAL + CTA_SMEM_RESERVED) <= SM_SMEM_BYTES,
                "shared memory budget exceeded: two CTAs must fit one SM");
  void (*kern)(GemmParams) = mode == EPI_GEGLU ? gemm_tc_kernel<BN, STAGES, EPI_GEGLU>
                             : mode == EPI_BF16 ? gemm_tc_kernel<BN, STAGES, EPI_BF16> : gemm_tc_kernel<BN, STAGES, EPI_F32>;
  const int rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), S::TOTAL, /*max_carveout=*/true);
  if (rc != PN_OK) return rc;
  kern<<<(unsigned)tiles, GEMM_THREADS, S::TOTAL, stream>>>(p);
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}

// Column-tile width of a GEMM with N output columns. Every channel count of the network is a multiple of 160
// (320/640/960/1280/1920/2560/5120/10240); a 128 x 160 fp32 accumulator is 80 registers per consumer thread.
static int gemm_bn(int N) { return N % 160 == 0 ? 160 : N >= 128 ? 128 : N > 32 ? 64 : 32; }

}  // namespace pn

using namespace pn;

extern "C" int pn_gemm(const pn_gemm_args* a, void* stream_v) {
  if (a == nullptr) return fail(PN_ERR_INVALID, "pn_gemm: null args");
  PN_REQUIRE(a->A && a->B && a->out, "pn_gemm: null tensor pointer");
  PN_REQUIRE(a->C > 0 && a->C % 64 == 0, "pn_gemm: C=%lld must be a positive multiple of 64", (long long)a->C);
  PN_REQUIRE(a->N > 0 && a->N % 8 == 0, "pn_gemm: N=%d must be a positive multiple of 8", a->N);
  PN_REQUIRE(a->taps_h >= 1 && a->taps_h <= 3 && a->taps_w >= 1 && a->taps_w <= 3, "pn_gemm: taps must be 1..3");
  PN_REQUIRE(a->NB > 0 && a->H > 0 && a->W > 0, "pn_gemm: empty A geometry");
  PN_REQUIRE((reinterpret_cast<uintptr_t>(a->A) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->B) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
             "pn_gemm: pointers must be 16-byte aligned");
  PN_REQUIRE(a->a_stride_w % 8 == 0 && a->a_stride_h % 8 == 0 && a->a_stride_n % 8 == 0,
             "pn_gemm: A strides must be multiples of 8 elements (16 bytes)");
  const int n_out = a->geglu ? a->N / 2 : a->N;
  PN_REQUIRE(a->ldo >= n_out && a->ldo % 8 == 0, "pn_gemm: ldo=%lld too small or misaligned", (long long)a->ldo);
  if (a->geglu) PN_REQUIRE(a->out_bf16 && a->residual == nullptr && a->N % 32 == 0, "pn_gemm: GEGLU needs bf16 out, no residual, N%%32==0");
  if (a->residual) PN_REQUIRE(a->ldr >= a->N && a->ldr % 4 == 0, "pn_gemm: bad ldr");
  if (a->residual_bf16) PN_REQUIRE(a->residual && a->out_bf16 && !a->geglu && a->residual2 == nullptr && a->ldr % 8 == 0,
                                   "pn_gemm: a bf16 residual needs bf16 output, no GEGLU, no second residual, ldr%%8==0");
  if (a->residual2) PN_REQUIRE(!a->out_bf16 && !a->geglu && a->ldr2 >= a->N && a->ldr2 % 4 == 0, "pn_gemm: residual2 needs fp32 out and a valid ldr2");
  if (a->rowvec) PN_REQUIRE(a->rows_per_group > 0 && a->n_groups > 0, "pn_gemm: rowvec needs rows_per_group/n_groups");
  if (a->ln_stats_in) PN_REQUIRE(a->bias != nullptr, "pn_gemm: a folded LayerNorm needs bias = W beta (+ bias)");
  if (a->ln_stats_in) PN_REQUIRE(a->ln_colsum && a->ln_parts_in > 0 && a->ln_parts_in <= 64 && a->out_bf16 && !a->geglu && a->taps_h == 1 && a->taps_w == 1,
                                 "pn_gemm: a folded LayerNorm needs ln_colsum, 1..64 partial sums per row, a 1x1 GEMM and bf16 output");


  GemmParams p;
  std::memset(&p, 0, sizeof(p));
  long long NB = a->NB, H = a->H, W = a->W;
  long long sw = a->a_stride_w, sh = a->a_stride_h, sn = a->a_stride_n;
  const bool pointwise = (a->taps_h == 1 && a->taps_w == 1);
  if (pointwise && sh == sw * W && sn == sh * H) {  // plain GEMM over a dense row set: flatten to [1,1,M]
    W = NB * H * W; H = 1; NB = 1; sh = sw * W; sn = sh;
  }
  int tw, th, tn;
  pick_tile(NB, H, W, &tw, &th, &tn);
  p.NB = (int)NB; p.H = (int)H; p.W = (int)W;
  p.tw = tw; p.th = th; p.tn = tn;
  p.tiles_w = (int)((W + tw - 1) / tw);
  p.tiles_h = (int)((H + th - 1) / th);
  p.tiles_n = (int)((NB + tn - 1) / tn);
  p.kc_per_tap = (int)(a->C / 64);
  p.taps_h = a->taps_h; p.taps_w = a->taps_w;
  p.pad_h = a->taps_h / 2; p.pad_w = a->taps_w / 2;
  p.N = a->N;
  p.out = a->out; p.bias = a->bias; p.rowvec = a->rowvec; p.residual = a->residual;
  p.residual2 = a->residual2;
  p.ldo = a->ldo; p.ldr = a->ldr; p.ldr2 = a->ldr2;
  p.ldv = a->rowvec_ld > 0 ? a->rowvec_ld : a->N;
  p.rows_per_group = a->rows_per_group > 0 ? a->rows_per_group : 1;
  p.n_groups = a->n_groups > 0 ? a->n_groups : 1;
  p.res_bf16 = a->residual_bf16;
  p.ln_stats_in = a->ln_stats_in; p.ln_colsum = a->ln_colsum; p.ln_stats_out = a->ln_stats_out;
  p.ln_parts_in = a->ln_parts_in; p.ln_eps = a->ln_eps; p.ln_inv_dim = 1.0f / (float)a->C;

  const int BN = gemm_bn(a->N);
  p.tiles_col = (a->N + BN - 1) / BN;
  if (a->ln_stats_out) {
    PN_REQUIRE(a->out_bf16 && !a->geglu && a->ln_stats_in == nullptr && pn_gemm_ln_parts(a->N) == 2 * p.tiles_col,
               "pn_gemm: ln_stats_out needs bf16 out, no GEGLU, no folded LayerNorm input and N %% 160 or 128 == 0");
    p.ln_parts_out = 2 * p.tiles_col;
  }
  const long long tiles = (long long)p.tiles_w * p.tiles_h * p.tiles_n * p.tiles_col;
  PN_REQUIRE(tiles > 0 && tiles < (1ll << 31), "pn_gemm: too many output tiles");

  const uint64_t K = (uint64_t)a->taps_h * a->taps_w * a->C;
  const uint64_t dimsB[2] = {K, (uint64_t)a->N};
  const uint64_t strB[1] = {K};
  const uint32_t boxB[2] = {64u, (uint32_t)BN};
  int rc = cached_tmap_bf16(&p.mapB, a->B, 2, dimsB, strB, boxB, 128);
  if (rc != PN_OK) return rc;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const EpiMode mode = a->geglu ? EPI_GEGLU : a->out_bf16 ? EPI_BF16 : EPI_F32;

  // 1x1 GEMMs over many dense rows whose 160 x K weight tile fits in shared memory (the level-0 linears, K = 320): the
  // persistent weight-stationary kernel of gemm_ws.cu. Its TMA maps over the residual need a 16-byte aligned base.
  if (pointwise && NB == 1 && H == 1 && a->C <= 320 && a->N % 160 == 0 && W >= WS_MIN_ROWS &&
      p.tiles_col <= sm_count() && (reinterpret_cast<uintptr_t>(a->residual) & 15) == 0)
    return launch_gemm_ws(p, mode, a->A, W, sw, (int)a->C, stream);

  const uint64_t dimsA[4] = {(uint64_t)a->C, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
  const uint64_t strA[3] = {(uint64_t)sw, (uint64_t)sh, (uint64_t)sn};
  const uint32_t boxA[4] = {64u, (uint32_t)tw, (uint32_t)th, (uint32_t)tn};
  rc = cached_tmap_bf16(&p.mapA, a->A, 4, dimsA, strA, boxA, 128);
  if (rc != PN_OK) return rc;
  switch (BN) {
    // the deepest rings that still fit two CTAs per SM (111,664 / 99,376 / 99,392 / 103,504 bytes per CTA)
    case 160: return launch_gemm<160, 3>(p, mode, tiles, stream);
    case 128: return launch_gemm<128, 3>(p, mode, tiles, stream);
    case 64: return launch_gemm<64, 4>(p, mode, tiles, stream);
    default: return launch_gemm<32, 5>(p, mode, tiles, stream);
  }
}

// number of partial (sum, sum of squares) pairs per row that a bf16 pn_gemm with N output columns writes to
// ln_stats_out (2 per 160- or 128-wide column tile)
extern "C" int pn_gemm_ln_parts(int N) {
  return N > 0 && (N % 160 == 0 || N % 128 == 0) ? 2 * (N / gemm_bn(N)) : 0;
}
