// The ControlNet's 19-channel layout maps (DESIGN.md section 12), rendered from per-panel primitive lists that
// panacea_b200/layout.py builds on the host. One launch renders a whole clip: T frames x 6 panels x 19 channels,
// straight into the fp32 [T, 19, H, 6w] hint that Engine.prepare_hint reads.
//
// A CTA owns a 32 x 8 pixel tile of one panel. It walks the panel's primitives in chunks of 256: each thread tests one
// primitive against the tile and the ones that overlap it are compacted into shared memory; then every thread
// composites its pixel against the compacted chunk. The compositing is order-free, so the atomic compaction leaves
// the output deterministic:
//  - depth rectangles (channels 3..12) keep the minimum byte per class channel;
//  - box fills, box edges (channels 0..2) and map segments (13..15) are painted over each other in the order of their
//    keys, so a pixel takes the colour of the highest key that covers it. The host gives the fill of the j-th box in
//    paint order key 2j and its edges key 2j+1, and the map segments their drawing order.
// Channels 16..18 are the camera-ray directions, an affine function of the pixel position evaluated in fp64.
#include "common.cuh"
#include "../../include/panacea_b200.h"

namespace pn {

constexpr int LAYOUT_TILE_W = 32, LAYOUT_TILE_H = 8, LAYOUT_THREADS = LAYOUT_TILE_W * LAYOUT_TILE_H;
constexpr int LAYOUT_CHANNELS = 19, LAYOUT_CLASSES = 10, LAYOUT_VIEWS = 6;

struct __align__(16) LayoutPrim {
  float4 head;   // kind, key (class of a rect), colour 0, colour 1
  float4 misc;   // colour 2 (byte value of a rect), radius, -, -
  float4 p01;    // rect: x0, y0, x1, y1 (half-open); quad: x0, y0, x1, y1; segment: ax, ay, bx, by
  float4 p23;    // quad: x2, y2, x3, y3
};
static_assert(sizeof(LayoutPrim) == PN_LAYOUT_PRIM_FLOATS * sizeof(float), "pn_render_layout record size");

__device__ __forceinline__ bool prim_overlaps(const LayoutPrim& p, float tx0, float ty0, float tx1, float ty1) {
  const int kind = (int)p.head.x;
  float x0, y0, x1, y1;
  if (kind == PN_LAYOUT_RECT) {                                   // half-open: pixels x0 .. x1-1
    x0 = p.p01.x; y0 = p.p01.y; x1 = p.p01.z - 1.f; y1 = p.p01.w - 1.f;
  } else if (kind == PN_LAYOUT_QUAD) {
    x0 = fminf(fminf(p.p01.x, p.p01.z), fminf(p.p23.x, p.p23.z));
    x1 = fmaxf(fmaxf(p.p01.x, p.p01.z), fmaxf(p.p23.x, p.p23.z));
    y0 = fminf(fminf(p.p01.y, p.p01.w), fminf(p.p23.y, p.p23.w));
    y1 = fmaxf(fmaxf(p.p01.y, p.p01.w), fmaxf(p.p23.y, p.p23.w));
  } else {
    const float r = p.misc.y;
    x0 = fminf(p.p01.x, p.p01.z) - r; x1 = fmaxf(p.p01.x, p.p01.z) + r;
    y0 = fminf(p.p01.y, p.p01.w) - r; y1 = fmaxf(p.p01.y, p.p01.w) + r;
  }
  return x0 <= tx1 && x1 >= tx0 && y0 <= ty1 && y1 >= ty0;
}

// even-odd rule at the pixel centre (cv2.fillPoly fills a self-intersecting quad the same way)
__device__ __forceinline__ bool quad_covers(const LayoutPrim& p, float px, float py) {
  const float xs[4] = {p.p01.x, p.p01.z, p.p23.x, p.p23.z}, ys[4] = {p.p01.y, p.p01.w, p.p23.y, p.p23.w};
  bool inside = false;
#pragma unroll
  for (int i = 0, j = 3; i < 4; j = i++) {
    if ((ys[i] > py) != (ys[j] > py) && px < (xs[j] - xs[i]) * (py - ys[i]) / (ys[j] - ys[i]) + xs[i]) inside = !inside;
  }
  return inside;
}

// a thick line is the set of pixel centres within `radius` of the segment (round caps)
__device__ __forceinline__ bool segment_covers(const LayoutPrim& p, float px, float py) {
  const float ax = p.p01.x, ay = p.p01.y, dx = p.p01.z - ax, dy = p.p01.w - ay, r = p.misc.y;
  const float qx = px - ax, qy = py - ay, len2 = dx * dx + dy * dy;
  const float t = len2 > 0.f ? fminf(fmaxf((qx * dx + qy * dy) / len2, 0.f), 1.f) : 0.f;
  const float ex = qx - t * dx, ey = qy - t * dy;
  return ex * ex + ey * ey <= r * r;
}

// One ray component of channels 16..18 as the reference's dataset computes it: the difference of img2lidar applied to
// (2u, 2v, 2, 1) and to (u, v, 1, 1), each a sequential fp64 dot product (no FMA contraction).
__device__ __forceinline__ double ray_component(const double* m, double u, double v) {
  const double far = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], 2.0 * u), __dmul_rn(m[1], 2.0 * v)), __dmul_rn(m[2], 2.0)), m[3]);
  const double near = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], u), __dmul_rn(m[1], v)), m[2]), m[3]);
  return __dsub_rn(far, near);
}

__global__ void __launch_bounds__(LAYOUT_THREADS) render_layout_kernel(
    const LayoutPrim* __restrict__ prims, const int32_t* __restrict__ panel_offsets, const double* __restrict__ rays,
    float* __restrict__ out, int H, int w) {
  __shared__ LayoutPrim s_prim[LAYOUT_THREADS];
  __shared__ int s_count;
  const int panel = blockIdx.z, frame = panel / LAYOUT_VIEWS, view = panel % LAYOUT_VIEWS;
  const int tx0 = blockIdx.x * LAYOUT_TILE_W, ty0 = blockIdx.y * LAYOUT_TILE_H;
  const int x = tx0 + threadIdx.x % LAYOUT_TILE_W, y = ty0 + threadIdx.x / LAYOUT_TILE_W;
  const float px = (float)x, py = (float)y;

  int depth[LAYOUT_CLASSES];
#pragma unroll
  for (int c = 0; c < LAYOUT_CLASSES; ++c) depth[c] = 255;
  float box_key = -1.f, map_key = -1.f;
  float box_rgb[3] = {255.f, 255.f, 255.f}, map_rgb[3] = {255.f, 255.f, 255.f};

  const int beg = panel_offsets[panel], end = panel_offsets[panel + 1];
  for (int base = beg; base < end; base += LAYOUT_THREADS) {
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    const int i = base + threadIdx.x;
    if (i < end) {
      const LayoutPrim p = prims[i];
      if (prim_overlaps(p, (float)tx0, (float)ty0, (float)(tx0 + LAYOUT_TILE_W - 1), (float)(ty0 + LAYOUT_TILE_H - 1)))
        s_prim[atomicAdd(&s_count, 1)] = p;
    }
    __syncthreads();
    const int n = s_count;
    for (int j = 0; j < n; ++j) {
      const LayoutPrim& p = s_prim[j];
      const int kind = (int)p.head.x;
      const float key = p.head.y;
      if (kind == PN_LAYOUT_RECT) {
        if (px >= p.p01.x && px < p.p01.z && py >= p.p01.y && py < p.p01.w) {
          const int cls = (int)key, val = (int)p.head.z;
#pragma unroll
          for (int c = 0; c < LAYOUT_CLASSES; ++c)
            if (c == cls) depth[c] = min(depth[c], val);
        }
      } else if (kind == PN_LAYOUT_MAP_SEGMENT) {
        if (key > map_key && segment_covers(p, px, py)) {
          map_key = key; map_rgb[0] = p.head.z; map_rgb[1] = p.head.w; map_rgb[2] = p.misc.x;
        }
      } else if (key > box_key && (kind == PN_LAYOUT_QUAD ? quad_covers(p, px, py) : segment_covers(p, px, py))) {
        box_key = key; box_rgb[0] = p.head.z; box_rgb[1] = p.head.w; box_rgb[2] = p.misc.x;
      }
    }
    __syncthreads();
  }
  if (x >= w || y >= H) return;

  // The reference flattens its (H, W) pixel grid and reads it back as (W, H) before transposing: output pixel (x, y)
  // carries the ray of pixel (r mod w, r div w) with r = x H + y (nuscenes_datasets_video.py:393-404).
  const long long r = (long long)x * H + y;
  const double u = (double)(r % w), v = (double)(r / w);
  const double* m = rays + view * 12;
  const double lo = rays[LAYOUT_VIEWS * 12], span = __dsub_rn(rays[LAYOUT_VIEWS * 12 + 1], lo);
  const size_t plane = (size_t)H * LAYOUT_VIEWS * w;
  float* o = out + (size_t)frame * LAYOUT_CHANNELS * plane + (size_t)y * LAYOUT_VIEWS * w + (size_t)view * w + x;
  const float full = 255.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * plane] = __fdiv_rn(box_rgb[c], full);
#pragma unroll
  for (int c = 0; c < LAYOUT_CLASSES; ++c) o[(3 + c) * plane] = __fdiv_rn((float)depth[c], full);
#pragma unroll
  for (int c = 0; c < 3; ++c) o[(13 + c) * plane] = __fdiv_rn(map_rgb[c], full);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double d = ray_component(m + 4 * c, u, v);
    const int q = min(max((int)__dmul_rn(__ddiv_rn(__dsub_rn(d, lo), span), 255.0), 0), 255);
    o[(16 + c) * plane] = __fdiv_rn((float)q, full);
  }
}

// ---------------------------------------------------------------- change mask (DESIGN.md section 13)
constexpr int MASK_THREADS = 256, MASK_MAX_CELLS = 49152;

// The per-pixel sources of pass 1. Each tells whether any of the `cell` pixels of column x, rows cy*cell .. cy*cell +
// cell - 1 of a frame is set. They load through __ldg: a struct member cannot carry the __restrict__ that would let the
// compiler use the read-only path on its own.
struct ChangedLayout {          // two 19-channel fp32 renders [T, 19, H, Wt]: set where any channel differs
  const float* a;
  const float* b;
  bool given() const { return a && b; }
  __device__ __forceinline__ bool operator()(int frame, int cy, int x, int H, int Wt, int cell) const {
    const size_t plane = (size_t)H * Wt;
    const size_t base = (size_t)frame * LAYOUT_CHANNELS * plane + (size_t)cy * cell * Wt + x;
    bool differs = false;
    for (int c = 0; c < LAYOUT_CHANNELS; ++c)
      for (int r = 0; r < cell; ++r) {
        const size_t i = base + c * plane + (size_t)r * Wt;
        differs |= __ldg(a + i) != __ldg(b + i);
      }
    return differs;
  }
};

struct DrawnPixels {            // a user-drawn uint8 mask [T, H, Wt]: set where nonzero
  const uint8_t* pixels;
  bool given() const { return pixels; }
  __device__ __forceinline__ bool operator()(int frame, int cy, int x, int H, int Wt, int cell) const {
    const uint8_t* p = pixels + ((size_t)frame * H + (size_t)cy * cell) * Wt + x;
    bool set = false;
    for (int r = 0; r < cell; ++r) set |= __ldg(p + (size_t)r * Wt) != 0;
    return set;
  }
};

// Pass 1: one thread per pixel column of a cell row asks the source about its `cell` pixels; the `cell` lanes of a cell
// (cell divides 32, so a cell never straddles two warps) combine their verdicts with one ballot.
template <class Source>
__global__ void __launch_bounds__(MASK_THREADS) pool_cells_kernel(const Source src, float* __restrict__ out, int H, int Wt,
                                                                  int cell) {
  const int x = blockIdx.x * MASK_THREADS + threadIdx.x, cy = blockIdx.y, frame = blockIdx.z;
  const bool set = x < Wt && src(frame, cy, x, H, Wt, cell);
  const unsigned votes = __ballot_sync(0xffffffffu, set);
  const int lane = threadIdx.x & 31;
  if (x < Wt && lane % cell == 0) {
    const unsigned group = cell == 32 ? 0xffffffffu : ((1u << cell) - 1u) << lane;
    out[((size_t)frame * (H / cell) + cy) * (Wt / cell) + x / cell] = (votes & group) ? 1.f : 0.f;
  }
}

// Pass 2: one CTA per panel dilates its cells in place: the panel is read whole into shared memory before any write.
__global__ void __launch_bounds__(MASK_THREADS) dilate_cells_kernel(float* __restrict__ out, int ch, int cw, int dilate) {
  __shared__ unsigned char s[MASK_MAX_CELLS];
  const int frame = blockIdx.x / LAYOUT_VIEWS, view = blockIdx.x % LAYOUT_VIEWS, Wc = LAYOUT_VIEWS * cw;
  float* o = out + (size_t)frame * ch * Wc + (size_t)view * cw;
  for (int i = threadIdx.x; i < ch * cw; i += MASK_THREADS) s[i] = o[(size_t)(i / cw) * Wc + i % cw] != 0.f;
  __syncthreads();
  for (int i = threadIdx.x; i < ch * cw; i += MASK_THREADS) {
    const int y = i / cw, x = i % cw;
    unsigned char v = 0;
    for (int yy = max(y - dilate, 0); yy <= min(y + dilate, ch - 1) && !v; ++yy)
      for (int xx = max(x - dilate, 0); xx <= min(x + dilate, cw - 1); ++xx) v |= s[yy * cw + xx];
    o[(size_t)y * Wc + x] = v ? 1.f : 0.f;
  }
}

// The checks, pass 1 over `src` and pass 2 of both cell-mask entry points; `fn` names the entry point in every message.
template <class Source>
static int cell_mask(const char* fn, const Source src, float* out, int64_t frames, int64_t height, int64_t view_width,
                     int64_t cell, int64_t dilate, void* stream_v) {
  PN_REQUIRE(src.given() && out, "%s: null pointer", fn);
  PN_REQUIRE(cell >= 1 && cell <= 32 && (cell & (cell - 1)) == 0, "%s: cell %lld is not a power of two <= 32", fn,
             (long long)cell);
  PN_REQUIRE(frames > 0 && frames <= 65535 / LAYOUT_VIEWS && height > 0 && view_width > 0 &&
             height * view_width * LAYOUT_VIEWS <= (int64_t)1 << 31,
             "%s: bad clip size %lld x %lld x %lld", fn, (long long)frames, (long long)height, (long long)view_width);
  PN_REQUIRE(height % cell == 0 && view_width % cell == 0, "%s: %lld x %lld is not a multiple of cell %lld", fn,
             (long long)height, (long long)view_width, (long long)cell);
  PN_REQUIRE((height / cell) * (view_width / cell) <= MASK_MAX_CELLS, "%s: more than %d cells per panel", fn, MASK_MAX_CELLS);
  PN_REQUIRE(dilate >= 0, "%s: dilate %lld < 0", fn, (long long)dilate);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
  const int64_t Wt = view_width * LAYOUT_VIEWS;
  const dim3 grid((unsigned)((Wt + MASK_THREADS - 1) / MASK_THREADS), (unsigned)(height / cell), (unsigned)frames);
  pool_cells_kernel<<<grid, MASK_THREADS, 0, st>>>(src, out, (int)height, (int)Wt, (int)cell);
  PN_CHECK_CUDA(cudaGetLastError());
  if (dilate > 0) {
    const int d = (int)(dilate < 65536 ? dilate : 65536);     // a panel has fewer cells per side
    dilate_cells_kernel<<<(unsigned)(frames * LAYOUT_VIEWS), MASK_THREADS, 0, st>>>(out, (int)(height / cell),
                                                                                     (int)(view_width / cell), d);
    PN_CHECK_CUDA(cudaGetLastError());
  }
  return PN_OK;
}

}  // namespace pn

extern "C" int pn_layout_change_mask(const float* a, const float* b, float* out, int64_t frames, int64_t height,
                                     int64_t view_width, int64_t cell, int64_t dilate, void* stream_v) {
  return pn::cell_mask("pn_layout_change_mask", pn::ChangedLayout{a, b}, out, frames, height, view_width, cell, dilate,
                       stream_v);
}

extern "C" int pn_mask_cells(const uint8_t* pixels, float* out, int64_t frames, int64_t height, int64_t view_width,
                             int64_t cell, int64_t dilate, void* stream_v) {
  return pn::cell_mask("pn_mask_cells", pn::DrawnPixels{pixels}, out, frames, height, view_width, cell, dilate, stream_v);
}

extern "C" int pn_render_layout(const float* prims, const int32_t* panel_offsets, const double* rays, float* out,
                                int64_t frames, int64_t height, int64_t view_width, void* stream_v) {
  PN_REQUIRE(prims && panel_offsets && rays && out, "pn_render_layout: null pointer");
  PN_REQUIRE(frames > 0 && frames <= 65535 / pn::LAYOUT_VIEWS && height > 0 && view_width > 0 &&
             height * view_width * pn::LAYOUT_VIEWS <= (int64_t)1 << 31,
             "pn_render_layout: bad clip size %lld x %lld x %lld", (long long)frames, (long long)height,
             (long long)view_width);
  PN_REQUIRE(((uintptr_t)prims & 15) == 0, "pn_render_layout: primitives must be 16-byte aligned");
  const dim3 grid((unsigned)((view_width + pn::LAYOUT_TILE_W - 1) / pn::LAYOUT_TILE_W),
                  (unsigned)((height + pn::LAYOUT_TILE_H - 1) / pn::LAYOUT_TILE_H), (unsigned)(frames * pn::LAYOUT_VIEWS));
  pn::render_layout_kernel<<<grid, pn::LAYOUT_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_v)>>>(
      reinterpret_cast<const pn::LayoutPrim*>(prims), panel_offsets, rays, out, (int)height, (int)view_width);
  PN_CHECK_CUDA(cudaGetLastError());
  return pn::PN_OK;
}
