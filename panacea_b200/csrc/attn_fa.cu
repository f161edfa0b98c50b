// wgmma flash attention for the decomposed-4D attention of Panacea (head_dim 64 — the reference config — or 80,
// BASELINE.json configs[4]; bf16 operands, fp32 softmax).
//
// One kernel serves the three tensor-core attention variants; they differ only in which K/V tiles a query tile
// visits, and every tile is a TMA box of ONE rank-5 tensor map over the token buffer [F, H, V, w, C]
// (frames, latent rows, views, columns per view, channels) — the views are never sliced or copied:
//   * intra-view  (attention.py:407-489)  : K/V = the query's own view;
//   * cross-view  (attention.py:518-610)  : K/V = the neighbour views from a table
//                                            {5,1},{0,2},{1,3},{2,4},{3,5},{4} (the reference's asymmetric ring);
//   * text cross-attention (attention.py:229-291, 77 keys): V=1, one K/V block per batch element, tail masked.
// (Temporal self-attention over T<=16 frames is a CUDA-core kernel, attn_small.cu.)
//
// CTA = one query tile (<= 128 queries of one frame/view/head), 288 threads:
//   warps 0-3 / 4-7: two consumer warpgroups, query rows 0-63 / 64-127. Per key block of <= N keys:
//                    S = Q K^T   wgmma m64nNk16, Q and K K-major from shared memory (fp32 S in registers);
//                    online softmax in registers (a query row lives in the 4 lanes of a quad);
//                    O += P V    N / 16 wgmma m64n64k16 with P as the REGISTER A operand (the S accumulator fragment is
//                                the A fragment layout) and V the MN-major B operand from shared memory.
//                    S of block j + 1 and P V of block j issue as one run of wgmmas and retire together (one wait
//                    per block, not two); the softmax of block j + 1 runs while the other warpgroup's MMAs use the
//                    tensor cores. (A wait<1> between the two, meant to run the exponentials under P V of the same
//                    warpgroup, is moved by ptxas ahead of them, so the kernel does not pretend to have one.)
//   warp 8:          TMA producer (Q once, K and V boxes through a STAGES-deep mbarrier ring).
// N, the width of the S wgmma, is the key block's row count rounded up to 16 (every block of a call has the same count:
// kh divides Hk), so no MMA, exponential or mask runs on keys that do not exist beyond that rounding. Query tiles are a
// rectangle of the view (qw x qh tokens) or, where a rectangle of whole rows would leave MMA rows empty and the view width
// is a multiple of 8, 128 consecutive tokens of the view in row-major order, loaded as 8-token boxes (one 1024 B
// swizzle atom each, so the tile lands in shared memory exactly as one 128-row box would).
// head_dim 80 is a 64-channel part plus a 16-channel part (a TMA box with a 128 B swizzle cannot be wider than 64
// bf16): every Q/K/V tile has a second, 32 B-row tile; S gets a fifth K = 16 step on the 16-channel tiles and
// O = P V a second wgmma of N = 16 per key step into output channels 64..79.
#include "common.cuh"
#include "ptx.cuh"
#include "operand.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

constexpr int FA_THREADS = 288;
constexpr int FA_TILE_BYTES = 128 * 128;          // 128 rows x 64 bf16 (128 B rows, 128B swizzle)
constexpr int FA_XTILE_BYTES = 128 * 32;          // head_dim 80: the channels 64..79 of 128 rows (32 B rows, 32B swizzle)
constexpr int FA_MAX_KEYS = 128;                  // keys per block: the largest N of the S wgmma
constexpr int FA_QBOX = 8;                        // tokens per Q box of a row-major query tile

template <int D>
struct FaL {
  static constexpr int STAGES = 3;
  static constexpr int XB = D == 64 ? 0 : FA_XTILE_BYTES;
  static constexpr int Q = 0;
  static constexpr int QX = FA_TILE_BYTES;
  static constexpr int KV = FA_TILE_BYTES + XB;                 // stage s: [K | V | Kx | Vx]
  static constexpr int STAGE_BYTES = 2 * FA_TILE_BYTES + 2 * XB;
  static constexpr int BAR = KV + STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR + 128 + 1024;
};

struct FaParams {
  CUtensorMap mapQ;
  CUtensorMap mapK;
  CUtensorMap mapV;
  CUtensorMap mapQx, mapKx, mapVx;   // head_dim 80: 16-channel boxes (32B swizzle) of the same tensors
  int heads;
  int F, H, V, W;              // query token grid
  int q_rowmajor;              // 1: query tile ti = tokens [128 ti, 128 ti + 128) of the view, row-major; 0: a qw x qh rectangle
  int qw, qh, tiles_x, tiles_y;
  int tiles_per_group;         // query tiles of one (frame, view, head)
  int kw, kh, kv_rows, kv_yblocks;
  int kv_views[8][2];
  int kv_view_count[8];
  int kv_frame_div;            // kv frame = q frame / kv_frame_div
  float scale_log2;            // softmax scale * log2(e)
  __nv_bfloat16* out;
  long long out_ld;            // token stride of out (elements)
};

template <int D, int N>
__global__ void __launch_bounds__(FA_THREADS, 1) attn_fa_kernel(const __grid_constant__ FaParams p) {
  static_assert(N % 16 == 0 && N >= 16 && N <= FA_MAX_KEYS, "a key block is a whole number of K = 16 steps of P V");
  using L = FaL<D>;
  constexpr int STAGES = L::STAGES;
  constexpr int GROUPS = N / 8;                  // 8-key column groups of the S fragment
  constexpr int KSTEPS = N / 16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::BAR);
  uint64_t* q_full = bars;                     // [1]
  uint64_t* kv_full = bars + 1;                // [STAGES]
  uint64_t* kv_empty = bars + 1 + STAGES;      // [STAGES]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // zero Q/K/V staging once: rows a TMA box does not cover (keys kv_rows..N-1, queries beyond the tile) must read as 0,
  // never as stale NaNs
  {
    uint4* z = reinterpret_cast<uint4*>(smem);
    for (int i = threadIdx.x; i < L::BAR / 16; i += FA_THREADS) z[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();
  }
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  // query tile fastest, then head, view, frame: CTAs that run concurrently share K/V in L2
  int item = blockIdx.x;
  const int ti = item % p.tiles_per_group; item /= p.tiles_per_group;
  const int head = item % p.heads; item /= p.heads;
  const int view = item % p.V;
  const int frame = item / p.V;
  const int nblk = p.kv_view_count[view] * p.kv_yblocks;

  if (warp == 8) {
    // ===================== TMA producer (warp-wide loop, TMA issue under elect.sync) =====================
    const uint32_t row_bytes = D == 80 ? 160u : 128u;
    const uint32_t kv_bytes = (uint32_t)p.kv_rows * row_bytes;
    if (elect_one()) {
      tma_prefetch_desc(&p.mapQ);
      tma_prefetch_desc(&p.mapK);
      tma_prefetch_desc(&p.mapV);
      if (p.q_rowmajor) {
        // W % 8 == 0, so an 8-token box never crosses a view row and the tile's last box is either full or absent
        const int t0 = ti * 128;
        const int rows = min(128, p.H * p.W - t0);
        mbar_arrive_expect_tx(q_full, (uint32_t)rows * row_bytes);
        for (int r = 0; r < rows; r += FA_QBOX) {
          const int y = (t0 + r) / p.W, x = t0 + r - y * p.W;
          tma_load_5d(smem + L::Q + r * 128, &p.mapQ, q_full, head * D, x, view, y, frame);
          if (D == 80) tma_load_5d(smem + L::QX + r * 32, &p.mapQx, q_full, head * D + 64, x, view, y, frame);
        }
      } else {
        mbar_arrive_expect_tx(q_full, (uint32_t)(p.qw * p.qh) * row_bytes);
        const int x0 = (ti % p.tiles_x) * p.qw, y0 = (ti / p.tiles_x) * p.qh;
        tma_load_5d(smem + L::Q, &p.mapQ, q_full, head * D, x0, view, y0, frame);
        if (D == 80) tma_load_5d(smem + L::QX, &p.mapQx, q_full, head * D + 64, x0, view, y0, frame);
      }
    }
    const int kv_frame = frame / p.kv_frame_div;
    int vi = 0, yb = 0;
    for (int j = 0; j < nblk; ++j) {
      const int st = j % STAGES;
      const int kvv = p.kv_views[view][vi];
      mbar_wait(&kv_empty[st], (uint32_t)(((j / STAGES) & 1) ^ 1));
      if (elect_one()) {
        uint8_t* sK = smem + L::KV + st * L::STAGE_BYTES;
        mbar_arrive_expect_tx(&kv_full[st], 2 * kv_bytes);
        tma_load_5d(sK, &p.mapK, &kv_full[st], head * D, 0, kvv, yb * p.kh, kv_frame);
        tma_load_5d(sK + FA_TILE_BYTES, &p.mapV, &kv_full[st], head * D, 0, kvv, yb * p.kh, kv_frame);
        if (D == 80) {
          tma_load_5d(sK + 2 * FA_TILE_BYTES, &p.mapKx, &kv_full[st], head * D + 64, 0, kvv, yb * p.kh, kv_frame);
          tma_load_5d(sK + 2 * FA_TILE_BYTES + L::XB, &p.mapVx, &kv_full[st], head * D + 64, 0, kvv, yb * p.kh, kv_frame);
        }
      }
      if (++yb == p.kv_yblocks) { yb = 0; ++vi; }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  const int quad = lane & 3;
  const uint32_t base = smem_u32(smem);
  const uint64_t dQ = wgmma_desc(base + L::Q + wg * 64 * 128, 16, 1024, kSw128);
  const uint64_t dQx = wgmma_desc(base + L::QX + wg * 64 * 32, 16, 256, kSw32);
  const uint64_t dK0 = wgmma_desc(base + L::KV, 16, 1024, kSw128);
  const uint64_t dV0 = wgmma_desc(base + L::KV + FA_TILE_BYTES, 1024, 1024, kSw128);
  const uint64_t dKx0 = wgmma_desc(base + L::KV + 2 * FA_TILE_BYTES, 16, 256, kSw32);
  const uint64_t dVx0 = wgmma_desc(base + L::KV + 2 * FA_TILE_BYTES + L::XB, 256, 256, kSw32);
  constexpr uint64_t STAGE_STEP = L::STAGE_BYTES >> 4;          // start-address field is in 16-byte units
  const float c = p.scale_log2;
  // keys kv_rows..N-1 exist only when kv_rows % 16 != 0, and then only in the last two 8-key groups
  const bool mask = p.kv_rows < N;

  float o[32], ox[8];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ox[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // raw-logit maximum and row sum, rows r and r + 8
  float s[N / 2];                                                   // S, then P, of the current block
  uint32_t pa[KSTEPS][4];                                           // P as the A fragments of the K = 16 key steps
  float alpha[2];                                                   // rescale of O and l for the block in s

  auto issue_s = [&](int st) {
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss<N>(s, dQ + 2 * k, dK0 + STAGE_STEP * st + 2 * k, k > 0 ? 1u : 0u);
    if (D == 80) wgmma_ss<N>(s, dQx, dKx0 + STAGE_STEP * st, 1u);
    wgmma_commit();
  };
  auto issue_pv = [&](int st) {
#pragma unroll
    for (int kk = 0; kk < KSTEPS; ++kk) {      // 16 keys per step: 16 rows (128 B each) of V
      wgmma_rs_tb<64>(o, pa[kk], dV0 + STAGE_STEP * st + kk * (2048 >> 4), 1u);
      if (D == 80) wgmma_rs_tb<16>(ox, pa[kk], dVx0 + STAGE_STEP * st + kk * (512 >> 4), 1u);
    }
    wgmma_commit();
  };
  // online softmax of the raw logits in s: running maximum and sum, alpha, and s <- exp2(c * (s - m))
  auto softmax = [&]() {
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < GROUPS; ++jj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (jj >= GROUPS - 2 && mask && 8 * jj + 2 * quad + (e & 1) >= p.kv_rows) s[4 * jj + e] = -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * jj + e]);
      }
    }
    float mc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_run[h], mx[h]);
      alpha[h] = ex2_approx((m_run[h] - m_new) * c);              // first block: exp2(-inf) = 0
      m_run[h] = m_new;
      mc[h] = m_new * c;
    }
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int jj = 0; jj < GROUPS; ++jj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float x = fmaf(s[4 * jj + e], c, -mc[e >> 1]);      // scale and max-subtract in one FFMA
        const float v = ex2_approx(x);
        s[4 * jj + e] = v;
        rs[e >> 1] += v;
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + rs[h];
  };
  // O *= alpha, then P -> bf16 A fragments
  auto rescale_and_pack = [&]() {
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
    if (D == 80) {
#pragma unroll
      for (int i = 0; i < 8; ++i) ox[i] *= alpha[(i >> 1) & 1];
    }
#pragma unroll
    for (int jj = 0; jj < GROUPS; ++jj) {
#pragma unroll
      for (int h = 0; h < 2; ++h) pa[jj >> 1][(jj & 1) * 2 + h] = pack_bf16x2(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]);
    }
  };
  auto pv_retired = [&](int st) {
    wgmma_fence_regs(o);
    if (D == 80) wgmma_fence_regs(ox);
#pragma unroll
    for (int kk = 0; kk < KSTEPS; ++kk) wgmma_fence_regs(pa[kk]);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[st]);   // this warpgroup's reads of the stage have retired
  };

  mbar_wait(q_full, 0);
  mbar_wait(&kv_full[0], 0);
  wgmma_fence();
  issue_s(0);
  wgmma_wait<0>();
  wgmma_fence_regs(s);
  softmax();
  rescale_and_pack();
  for (int j = 1; j < nblk; ++j) {
    const int st = j % STAGES, prev = (j - 1) % STAGES;
    mbar_wait(&kv_full[st], (uint32_t)((j / STAGES) & 1));
    wgmma_fence();
    issue_s(st);
    issue_pv(prev);
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    pv_retired(prev);
    softmax();
    rescale_and_pack();
  }
  wgmma_fence();
  issue_pv((nblk - 1) % STAGES);
  wgmma_wait<0>();
  pv_retired((nblk - 1) % STAGES);

  // normalise by the row sums and store this thread's two query rows (bf16)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    int x, y;
    if (p.q_rowmajor) {
      const int t = ti * 128 + row;
      y = t / p.W;
      x = t - y * p.W;
    } else {
      if (row >= p.qw * p.qh) continue;
      const int yy = row / p.qw, xx = row - yy * p.qw;
      x = (ti % p.tiles_x) * p.qw + xx;
      y = (ti / p.tiles_x) * p.qh + yy;
    }
    if (x >= p.W || y >= p.H) continue;
    const long long token = (((long long)frame * p.H + y) * p.V + view) * p.W + x;
    __nv_bfloat16* dst = p.out + token * p.out_ld + head * D + 2 * quad;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
      *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    if (D == 80) {
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 64 + 8 * jj) = pack_bf16x2(ox[4 * jj + 2 * h] * inv, ox[4 * jj + 2 * h + 1] * inv);
    }
  }
}

// indexed by N / 16 - 1
template <int D>
void (*const fa_kernels[FA_MAX_KEYS / 16])(FaParams) = {attn_fa_kernel<D, 16>, attn_fa_kernel<D, 32>, attn_fa_kernel<D, 48>,
                                                        attn_fa_kernel<D, 64>, attn_fa_kernel<D, 80>, attn_fa_kernel<D, 96>,
                                                        attn_fa_kernel<D, 112>, attn_fa_kernel<D, 128>};

}  // namespace pn

using namespace pn;

extern "C" int pn_attention(const pn_attn_args* a, int operand_mode, void* stream_v) {
  PN_OPERAND_MODES(Modes, operand_mode, "pn_attention", PN_OPERAND_BF16, PN_OPERAND_SPLIT3, PN_OPERAND_F32);
  if (operand_mode != PN_OPERAND_BF16) return attention_f32(a, operand_mode, stream_v);
  if (a == nullptr) return fail(PN_ERR_INVALID, "pn_attention: null args");
  PN_REQUIRE(a->q && a->k && a->v && a->out, "pn_attention: null tensor pointer");
  PN_REQUIRE(a->head_dim == 64 || a->head_dim == 80, "pn_attention: head_dim %d unsupported (64 or 80)", a->head_dim);
  const int FA_D = a->head_dim;
  PN_REQUIRE(a->heads > 0 && a->F > 0 && a->H > 0 && a->V > 0 && a->V <= 8 && a->W > 0, "pn_attention: bad query geometry");
  PN_REQUIRE(a->Hk > 0 && a->Vk > 0 && a->Vk <= 8 && a->Wk > 0 && a->kv_frame_div > 0, "pn_attention: bad key geometry");
  PN_REQUIRE(a->q_ld % 8 == 0 && a->kv_ld % 8 == 0 && a->out_ld % 8 == 0, "pn_attention: token strides must be multiples of 8");
  PN_REQUIRE(a->q_ld >= a->heads * FA_D && a->kv_ld >= a->heads * FA_D && a->out_ld >= a->heads * FA_D,
             "pn_attention: token stride smaller than heads*64");

  FaParams p;
  std::memset(&p, 0, sizeof(p));
  p.heads = a->heads;
  p.F = (int)a->F; p.H = (int)a->H; p.V = (int)a->V; p.W = (int)a->W;
  // query tile: full view width when it fits, as many rows as keep <= 128 queries; 128 row-major tokens instead where
  // such a rectangle would leave rows of the 128-row MMA tile empty and 8-token boxes tile the view rows
  p.qw = (int)(a->W <= 128 ? a->W : 128);
  p.qh = 128 / p.qw;
  if (p.qh > a->H) p.qh = (int)a->H;
  if (p.qh < 1) p.qh = 1;
  p.tiles_x = (int)((a->W + p.qw - 1) / p.qw);
  p.tiles_y = (int)((a->H + p.qh - 1) / p.qh);
  p.q_rowmajor = a->W % FA_QBOX == 0 && a->W < 128 && p.qw * p.qh < 128 && a->H > p.qh;
  // key block: full key-view width (must fit one block row-wise), rows = largest divisor of Hk with <= 128 keys
  PN_REQUIRE(a->Wk <= FA_MAX_KEYS, "pn_attention: key view width %lld > %d unsupported", (long long)a->Wk, FA_MAX_KEYS);
  p.kw = (int)a->Wk;
  int kh = FA_MAX_KEYS / p.kw;
  if (kh > a->Hk) kh = (int)a->Hk;
  while (kh > 1 && (a->Hk % kh) != 0) --kh;
  p.kh = kh;
  p.kv_rows = p.kw * p.kh;
  p.kv_yblocks = (int)(a->Hk / p.kh);
  for (int v = 0; v < a->V; ++v) {
    const int cnt = a->kv_view_count[v];
    PN_REQUIRE(cnt >= 1 && cnt <= 2, "pn_attention: kv_view_count[%d]=%d must be 1 or 2", v, cnt);
    p.kv_view_count[v] = cnt;
    for (int i = 0; i < cnt; ++i) {
      PN_REQUIRE(a->kv_views[v][i] >= 0 && a->kv_views[v][i] < a->Vk, "pn_attention: kv view out of range");
      p.kv_views[v][i] = a->kv_views[v][i];
    }
  }
  p.kv_frame_div = a->kv_frame_div;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.out = reinterpret_cast<__nv_bfloat16*>(a->out);
  p.out_ld = a->out_ld;

  const uint64_t chq = (uint64_t)a->heads * FA_D;
  {
    const uint64_t dims[5] = {chq, (uint64_t)a->W, (uint64_t)a->V, (uint64_t)a->H, (uint64_t)a->F};
    const uint64_t ld = (uint64_t)a->q_ld;
    const uint64_t str[4] = {ld, ld * a->W, ld * a->W * a->V, ld * a->W * a->V * a->H};
    const uint32_t bw = p.q_rowmajor ? FA_QBOX : p.qw, bh = p.q_rowmajor ? 1 : p.qh;
    const uint32_t box[5] = {64u, bw, 1u, bh, 1u};
    int rc = cached_tmap_bf16(&p.mapQ, a->q, 5, dims, str, box, 128);
    if (rc != PN_OK) return rc;
    if (FA_D == 80) {
      const uint32_t boxx[5] = {16u, bw, 1u, bh, 1u};
      rc = cached_tmap_bf16(&p.mapQx, a->q, 5, dims, str, boxx, 32);
      if (rc != PN_OK) return rc;
    }
  }
  {
    const uint64_t Fk = (uint64_t)((a->F + a->kv_frame_div - 1) / a->kv_frame_div);
    const uint64_t dims[5] = {chq, (uint64_t)a->Wk, (uint64_t)a->Vk, (uint64_t)a->Hk, Fk};
    const uint64_t ld = (uint64_t)a->kv_ld;
    const uint64_t str[4] = {ld, ld * a->Wk, ld * a->Wk * a->Vk, ld * a->Wk * a->Vk * a->Hk};
    const uint32_t box[5] = {64u, (uint32_t)p.kw, 1u, (uint32_t)p.kh, 1u};
    int rc = cached_tmap_bf16(&p.mapK, a->k, 5, dims, str, box, 128);
    if (rc != PN_OK) return rc;
    rc = cached_tmap_bf16(&p.mapV, a->v, 5, dims, str, box, 128);
    if (rc != PN_OK) return rc;
    if (FA_D == 80) {
      const uint32_t boxx[5] = {16u, (uint32_t)p.kw, 1u, (uint32_t)p.kh, 1u};
      rc = cached_tmap_bf16(&p.mapKx, a->k, 5, dims, str, boxx, 32);
      if (rc != PN_OK) return rc;
      rc = cached_tmap_bf16(&p.mapVx, a->v, 5, dims, str, boxx, 32);
      if (rc != PN_OK) return rc;
    }
  }
  p.tiles_per_group = p.q_rowmajor ? (int)((a->H * a->W + 127) / 128) : p.tiles_x * p.tiles_y;
  const long long items = (long long)p.tiles_per_group * a->heads * a->V * a->F;
  PN_REQUIRE(items > 0 && items < (1ll << 31), "pn_attention: too many query tiles");
  const int n_idx = (p.kv_rows + 15) / 16 - 1;
  void (*kern)(FaParams) = FA_D == 80 ? fa_kernels<80>[n_idx] : fa_kernels<64>[n_idx];
  const size_t smem_total = FA_D == 80 ? FaL<80>::TOTAL : FaL<64>::TOTAL;
  {
    const int rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), smem_total);
    if (rc != PN_OK) return rc;
  }
  kern<<<(unsigned)items, FA_THREADS, smem_total, reinterpret_cast<cudaStream_t>(stream_v)>>>(p);
  PN_CHECK_CUDA(cudaGetLastError());
  return PN_OK;
}
