// Paste the recorded pixels back outside an edit (DESIGN.md section 13). For each pixel of each panel, d2 is the squared
// integer distance between its centre and the nearest pixel of a regenerated cell of the same panel; alpha is 1 inside
// a regenerated cell, falls linearly to 0 over `feather` pixels outside it, and the output blends the decode over the
// byte centre of the recorded pixel with it.
//
// A CTA owns a 64 x 16 pixel tile of one panel. Only cells within `feather` pixels of the tile can give alpha > 0, so it
// stages that window of cells in shared memory (cells up to feather pixels away on each side, clipped to the panel)
// and computes the distance separably:
//   G(y, cx) = min over regenerated cells (cy, cx) of the window of dy^2           (one entry per tile row, cell column)
//   d2(x, y) = min over cx of dx^2 + G(y, cx)
// Every step is integer or correctly rounded fp32, so the output is bitwise the same from call to call.
#include "common.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

constexpr int COMP_TILE_W = 64, COMP_TILE_H = 16, COMP_THREADS = 256, COMP_VIEWS = 6, COMP_MAX_FEATHER = 64;
constexpr int COMP_PIX = COMP_TILE_W * COMP_TILE_H / COMP_THREADS;              // pixels per thread
// cells of the window along each side at cell = 1 (the most): the tile plus feather pixels on both sides
constexpr int COMP_WIN_W = COMP_TILE_W + 2 * COMP_MAX_FEATHER, COMP_WIN_H = COMP_TILE_H + 2 * COMP_MAX_FEATHER;
constexpr int COMP_FAR = 0x3fffffff;

// 1D distance from pixel p to the pixel range [c * cell, c * cell + cell - 1]
__device__ __forceinline__ int cell_gap(int p, int c, int cell) { return max(max(c * cell - p, p - (c * cell + cell - 1)), 0); }

__global__ void __launch_bounds__(COMP_THREADS) composite_frames_kernel(
    const float* __restrict__ decoded, const float* __restrict__ recorded, const float* __restrict__ cells,
    float* __restrict__ out, float* __restrict__ alpha_out, int H, int w, int cell, int feather) {
  __shared__ unsigned char s_cell[COMP_WIN_H * COMP_WIN_W];
  __shared__ int s_g[COMP_TILE_H * COMP_WIN_W];
  const int frame = blockIdx.z / COMP_VIEWS, view = blockIdx.z % COMP_VIEWS;
  const int x0 = blockIdx.x * COMP_TILE_W, y0 = blockIdx.y * COMP_TILE_H;
  const int Wt = COMP_VIEWS * w, hc = H / cell, Wc = Wt / cell;
  const int cx_lo = max(x0 - feather, 0) / cell, cx_hi = min(x0 + COMP_TILE_W - 1 + feather, w - 1) / cell;
  const int cy_lo = max(y0 - feather, 0) / cell, cy_hi = min(y0 + COMP_TILE_H - 1 + feather, H - 1) / cell;
  const int ncx = cx_hi - cx_lo + 1, ncy = cy_hi - cy_lo + 1;

  const float* c = cells + (size_t)frame * hc * Wc + (size_t)view * (w / cell);
  bool any = false;
  for (int i = threadIdx.x; i < ncx * ncy; i += COMP_THREADS) {
    const bool on = c[(size_t)(cy_lo + i / ncx) * Wc + cx_lo + i % ncx] > 0.f;
    s_cell[i] = on;
    any |= on;
  }
  any = __syncthreads_or(any);
  if (any) {
    for (int i = threadIdx.x; i < COMP_TILE_H * ncx; i += COMP_THREADS) {
      const int r = i / ncx, cxi = i % ncx, y = y0 + r;
      int g = COMP_FAR;
      for (int cyi = 0; cyi < ncy; ++cyi)
        if (s_cell[cyi * ncx + cxi]) {
          const int dy = cell_gap(y, cy_lo + cyi, cell);
          g = min(g, dy * dy);
        }
      s_g[r * ncx + cxi] = g;
    }
    __syncthreads();
  }

  const size_t plane = (size_t)H * Wt;
  const float reach = (float)(feather + 1);
  float alpha[COMP_PIX];
#pragma unroll
  for (int k = 0; k < COMP_PIX; ++k) {
    const int j = threadIdx.x + k * COMP_THREADS, r = j / COMP_TILE_W, x = x0 + j % COMP_TILE_W;
    int d2 = COMP_FAR;
    if (any)
      for (int cxi = 0; cxi < ncx; ++cxi) {
        const int g = s_g[r * ncx + cxi];
        if (g != COMP_FAR) {
          const int dx = cell_gap(x, cx_lo + cxi, cell);
          d2 = min(d2, dx * dx + g);
        }
      }
    alpha[k] = d2 == 0 ? 1.f
             : d2 == COMP_FAR ? 0.f
             : fmaxf(0.f, __fsub_rn(1.f, __fdiv_rn(__fsqrt_rn((float)d2), reach)));
  }
#pragma unroll
  for (int k = 0; k < COMP_PIX; ++k) {
    const int j = threadIdx.x + k * COMP_THREADS, y = y0 + j / COMP_TILE_W, x = x0 + j % COMP_TILE_W;
    if (x >= w || y >= H) continue;
    const size_t p = (size_t)frame * 3 * plane + (size_t)y * Wt + (size_t)view * w + x;
    const float a = alpha[k];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float d = decoded[p + ch * plane];
      const float b = fminf(fmaxf(rintf(__fmul_rn(__fadd_rn(recorded[p + ch * plane], 1.f), 127.5f)), 0.f), 255.f);
      const float kc = __fsub_rn(__fdiv_rn(__fadd_rn(b, 0.5f), 127.5f), 1.f);     // centre of the recorded byte
      out[p + ch * plane] = a == 1.f ? d : a == 0.f ? kc : __fadd_rn(kc, __fmul_rn(a, __fsub_rn(d, kc)));
    }
    if (alpha_out) alpha_out[(size_t)frame * plane + (size_t)y * Wt + (size_t)view * w + x] = a;
  }
}

}  // namespace pn

static bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
  return a && b && pa < pb + nb && pb < pa + na;
}

extern "C" int pn_composite_frames(const float* decoded, const float* recorded, const float* cells, float* out, float* alpha,
                                   int64_t frames, int64_t height, int64_t view_width, int64_t cell, int64_t feather,
                                   void* stream_v) {
  PN_REQUIRE(decoded && recorded && cells && out, "pn_composite_frames: null pointer");
  PN_REQUIRE(cell >= 1 && cell <= 32 && (cell & (cell - 1)) == 0, "pn_composite_frames: cell %lld is not a power of two <= 32",
             (long long)cell);
  PN_REQUIRE(frames > 0 && frames <= 65535 / pn::COMP_VIEWS && height > 0 && view_width > 0 &&
             height * view_width * pn::COMP_VIEWS <= (int64_t)1 << 31 && height <= 65535 * (int64_t)pn::COMP_TILE_H,
             "pn_composite_frames: bad clip size %lld x %lld x %lld", (long long)frames, (long long)height,
             (long long)view_width);
  PN_REQUIRE(height % cell == 0 && view_width % cell == 0, "pn_composite_frames: %lld x %lld is not a multiple of cell %lld",
             (long long)height, (long long)view_width, (long long)cell);
  PN_REQUIRE(feather >= 0 && feather <= pn::COMP_MAX_FEATHER, "pn_composite_frames: feather %lld outside 0 .. %d",
             (long long)feather, pn::COMP_MAX_FEATHER);
  const size_t px = (size_t)frames * height * view_width * pn::COMP_VIEWS * sizeof(float);
  const size_t nc = (size_t)frames * (height / cell) * (view_width / cell) * pn::COMP_VIEWS * sizeof(float);
  PN_REQUIRE(!overlaps(out, 3 * px, decoded, 3 * px) && !overlaps(out, 3 * px, recorded, 3 * px) &&
             !overlaps(out, 3 * px, cells, nc) && !overlaps(alpha, px, decoded, 3 * px) &&
             !overlaps(alpha, px, recorded, 3 * px) && !overlaps(alpha, px, cells, nc) && !overlaps(alpha, px, out, 3 * px),
             "pn_composite_frames: out and alpha must not alias an input or each other");
  const dim3 grid((unsigned)((view_width + pn::COMP_TILE_W - 1) / pn::COMP_TILE_W),
                  (unsigned)((height + pn::COMP_TILE_H - 1) / pn::COMP_TILE_H), (unsigned)(frames * pn::COMP_VIEWS));
  pn::composite_frames_kernel<<<grid, pn::COMP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_v)>>>(
      decoded, recorded, cells, out, alpha, (int)height, (int)view_width, (int)cell, (int)feather);
  PN_CHECK_CUDA(cudaGetLastError());
  return pn::PN_OK;
}
