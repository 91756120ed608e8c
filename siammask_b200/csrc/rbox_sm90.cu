// SiamMask's rotated box (tools/test.py:284-303) for N masks of different sizes: the largest outer contour's
// minimum-area rectangle, or the fallback rectangle of the state.  C ABI sm_rotated_box_ragged
// (include/siammask_b200.h); the numpy restatement is tests/rbox_reference.py.
//
// Six fixed-shape launches, grid (blocks, N) or N blocks, with no host round trip:
//   1. rb_init     labels: a foreground pixel's own raster index, -1 for background; per-stream state reset;
//   2. rb_merge    8-connected union-find over the W, NW, N and NE neighbours: atomicMin links a root to the smaller
//                  one, so every component ends up rooted at its raster-first pixel whatever the order of the unions;
//   3. rb_flatten  every pixel points at its root;
//   4. rb_trace    each root follows its component's outer border (Suzuki & Abe's border following) and keeps the
//                  doubled shoelace area; atomicMax of (area2 << 32 | root) selects the largest area and, among equal
//                  areas, the raster-last root, as cv2's contour order and np.argmax do;
//   5. rb_rows     the selected component's leftmost and rightmost pixel of every row (integer atomics);
//   6. rb_rect     one block per stream: Andrew's monotone chain over those row extremes, every hull edge's rectangle
//                  in integers, the least area compared exactly (first edge on ties), the vertices in float64 rounded
//                  to float32 in boxPoints' order; or the fallback rectangle when the area is not over 100.
// Every reduction is an integer atomic or a fixed-order loop, so equal inputs give equal bits.
#include <algorithm>

#include "common.cuh"
#include "../../include/siammask_b200.h"

namespace smk {
namespace {

constexpr int RB_THREADS = 256;
constexpr int RB_RECT_THREADS = 128;

__device__ __forceinline__ bool rb_fg(const uint8_t* m, int h, int w, int x, int y) {
  return x >= 0 && x < w && y >= 0 && y < h && m[(size_t)y * w + x] != 0;
}

__device__ __forceinline__ int rb_find(const int32_t* lab, int x) {
  int y;
  while ((y = lab[x]) != x) x = y;
  return x;
}

__device__ void rb_union(int32_t* lab, int a, int b) {
  while (true) {
    a = rb_find(lab, a);
    b = rb_find(lab, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&lab[b], a);          // link root b below root a; a concurrent link moved b: retry
    if (old == b) return;
    b = old;
  }
}

__global__ void __launch_bounds__(RB_THREADS) rb_init(const uint8_t* __restrict__ masks,
                                                      const sm_image_desc* __restrict__ desc, int32_t* __restrict__ lab,
                                                      unsigned long long* __restrict__ best, int32_t* __restrict__ rows,
                                                      int max_h) {
  const int b = blockIdx.y;
  const sm_image_desc d = desc[b];
  const int64_t n = (int64_t)d.h * d.w;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
    lab[d.offset + p] = masks[d.offset + p] ? (int32_t)p : -1;
  int32_t* r = rows + (size_t)b * 2 * max_h;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max_h; i += gridDim.x * blockDim.x) {
    r[2 * i] = INT32_MAX;                             // leftmost x of row i
    r[2 * i + 1] = -1;                                // rightmost x
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) best[b] = 0ull;
}

__global__ void __launch_bounds__(RB_THREADS) rb_merge(const uint8_t* __restrict__ masks,
                                                       const sm_image_desc* __restrict__ desc, int32_t* lab) {
  const int b = blockIdx.y;
  const sm_image_desc d = desc[b];
  const int64_t n = (int64_t)d.h * d.w;
  const uint8_t* m = masks + d.offset;
  int32_t* L = lab + d.offset;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    if (!m[p]) continue;
    const int y = (int)(p / d.w), x = (int)(p % d.w);
    if (rb_fg(m, d.h, d.w, x - 1, y)) rb_union(L, (int)p, (int)p - 1);
    if (rb_fg(m, d.h, d.w, x - 1, y - 1)) rb_union(L, (int)p, (int)p - d.w - 1);
    if (rb_fg(m, d.h, d.w, x, y - 1)) rb_union(L, (int)p, (int)p - d.w);
    if (rb_fg(m, d.h, d.w, x + 1, y - 1)) rb_union(L, (int)p, (int)p - d.w + 1);
  }
}

__global__ void __launch_bounds__(RB_THREADS) rb_flatten(const sm_image_desc* __restrict__ desc, int32_t* lab) {
  const int b = blockIdx.y;
  const sm_image_desc d = desc[b];
  const int64_t n = (int64_t)d.h * d.w;
  int32_t* L = lab + d.offset;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
    if (L[p] >= 0) L[p] = rb_find(L, (int)p);
}

// OpenCV's chain-code directions: 0 = east, counterclockwise on screen (y down)
__constant__ int8_t RB_DX[8] = {1, 1, 0, -1, -1, -1, 0, 1};
__constant__ int8_t RB_DY[8] = {0, -1, -1, -1, 0, 1, 1, 1};

__device__ __forceinline__ int rb_dir(int dx, int dy) {     // inverse of RB_DX / RB_DY
  constexpr int8_t T[9] = {3, 2, 1, 4, -1, 0, 5, 6, 7};      // index (dy + 1) * 3 + (dx + 1)
  return T[(dy + 1) * 3 + (dx + 1)];
}

// Doubled area of the outer border through (x0, y0), the raster-first pixel of its component: Suzuki & Abe (1985),
// algorithm 1, steps 3.1-3.5 (tests/rbox_reference.py: trace_outer).
__device__ int64_t rb_trace_area2(const uint8_t* m, int h, int w, int x0, int y0) {
  int first = -1;
  constexpr int8_t CW[8] = {4, 3, 2, 1, 0, 7, 6, 5};          // clockwise from the west neighbour
  for (int k = 0; k < 8 && first < 0; ++k)
    if (rb_fg(m, h, w, x0 + RB_DX[CW[k]], y0 + RB_DY[CW[k]])) first = CW[k];
  if (first < 0) return 0;                                     // an isolated pixel
  const int x1 = x0 + RB_DX[first], y1 = y0 + RB_DY[first];
  int px = x1, py = y1, cx = x0, cy = y0;
  int64_t s = 0;
  while (true) {
    const int d0 = rb_dir(px - cx, py - cy);
    int d = d0;
    for (int k = 1; k <= 8; ++k) {                             // counterclockwise from the neighbour after prev
      d = (d0 + k) & 7;
      if (rb_fg(m, h, w, cx + RB_DX[d], cy + RB_DY[d])) break;
    }
    const int nx = cx + RB_DX[d], ny = cy + RB_DY[d];
    s += (int64_t)cx * ny - (int64_t)nx * cy;
    if (nx == x0 && ny == y0 && cx == x1 && cy == y1) break;
    px = cx; py = cy; cx = nx; cy = ny;
  }
  return s < 0 ? -s : s;
}

__global__ void __launch_bounds__(RB_THREADS) rb_trace(const uint8_t* __restrict__ masks,
                                                       const sm_image_desc* __restrict__ desc,
                                                       const int32_t* __restrict__ lab,
                                                       unsigned long long* __restrict__ best) {
  const int b = blockIdx.y;
  const sm_image_desc d = desc[b];
  const int64_t n = (int64_t)d.h * d.w;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    if (lab[d.offset + p] != (int32_t)p) continue;             // roots only
    const int64_t a2 = rb_trace_area2(masks + d.offset, d.h, d.w, (int)(p % d.w), (int)(p / d.w));
    atomicMax(&best[b], ((unsigned long long)a2 << 32) | (unsigned long long)p);
  }
}

__device__ __forceinline__ bool rb_selected(unsigned long long key) { return (key >> 32) > 200ull; }   // area > 100

__global__ void __launch_bounds__(RB_THREADS) rb_rows(const sm_image_desc* __restrict__ desc,
                                                      const int32_t* __restrict__ lab,
                                                      const unsigned long long* __restrict__ best,
                                                      int32_t* __restrict__ rows, int max_h) {
  const int b = blockIdx.y;
  const unsigned long long key = best[b];
  if (!rb_selected(key)) return;
  const int32_t root = (int32_t)(key & 0xffffffffull);
  const sm_image_desc d = desc[b];
  const int64_t n = (int64_t)d.h * d.w;
  int32_t* r = rows + (size_t)b * 2 * max_h;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    if (lab[d.offset + p] != root) continue;
    const int y = (int)(p / d.w), x = (int)(p % d.w);
    atomicMin(&r[2 * y], x);
    atomicMax(&r[2 * y + 1], x);
  }
}

__device__ __forceinline__ int64_t rb_cross(int2 o, int2 a, int2 c) {
  return (int64_t)(a.x - o.x) * (c.y - o.y) - (int64_t)(a.y - o.y) * (c.x - o.x);
}

struct RbExtent {
  int64_t amin, amax, bmin, bmax;
};

// Projections of the hull onto edge i (from hull[i] to hull[i+1]) and its normal n = (-e_y, e_x), relative to hull[i].
__device__ RbExtent rb_extent(const int2* hull, int M, int i) {
  const int2 p = hull[i], q = hull[i + 1 == M ? 0 : i + 1];
  const int64_t ex = q.x - p.x, ey = q.y - p.y;
  RbExtent r{INT64_MAX, INT64_MIN, INT64_MAX, INT64_MIN};
  for (int j = 0; j < M; ++j) {
    const int64_t dx = hull[j].x - p.x, dy = hull[j].y - p.y;
    const int64_t a = ex * dx + ey * dy, bb = -ey * dx + ex * dy;
    r.amin = min(r.amin, a); r.amax = max(r.amax, a);
    r.bmin = min(r.bmin, bb); r.bmax = max(r.bmax, bb);
  }
  return r;
}

__global__ void __launch_bounds__(RB_RECT_THREADS) rb_rect(const sm_image_desc* __restrict__ desc,
                                                           const int32_t* __restrict__ rows,
                                                           const unsigned long long* __restrict__ best,
                                                           const double* __restrict__ fallback, int max_h,
                                                           int2* __restrict__ pts_ws, int2* __restrict__ hull_ws,
                                                           unsigned long long* __restrict__ q_ws,
                                                           double* __restrict__ poly, int32_t* __restrict__ flag,
                                                           int64_t* __restrict__ area2) {
  const int b = blockIdx.x;
  const unsigned long long key = best[b];
  double* out = poly + 8 * (size_t)b;
  if (!rb_selected(key)) {                                     // cxy_wh_2_rect of the pre-clamp state
    if (threadIdx.x == 0) {
      const double* f = fallback + 4 * (size_t)b;
      const double x0 = __dadd_rn(f[0], -(f[2] / 2)), y0 = __dadd_rn(f[1], -(f[3] / 2));
      const double x1 = __dadd_rn(x0, f[2]), y1 = __dadd_rn(y0, f[3]);
      out[0] = x0; out[1] = y0; out[2] = x1; out[3] = y0; out[4] = x1; out[5] = y1; out[6] = x0; out[7] = y1;
      flag[b] = 0;
      area2[b] = (int64_t)(key >> 32);
    }
    return;
  }
  const int h = desc[b].h;
  const int32_t* r = rows + (size_t)b * 2 * max_h;
  int2* pts = pts_ws + (size_t)b * 2 * max_h;
  int2* hull = hull_ws + (size_t)b * (2 * max_h + 1);
  unsigned long long* qa = q_ws + (size_t)b * 2 * (2 * max_h + 1);
  __shared__ int s_M;
  if (threadIdx.x == 0) {
    // the row extremes sorted by (y, x), then Andrew's monotone chain: first chain, second chain, collinear dropped
    int n = 0;
    for (int y = 0; y < h; ++y) {
      if (r[2 * y] > r[2 * y + 1]) continue;
      pts[n++] = make_int2(r[2 * y], y);
      if (r[2 * y + 1] != r[2 * y]) pts[n++] = make_int2(r[2 * y + 1], y);
    }
    int k = 0;
    for (int i = 0; i < n; ++i) {
      while (k >= 2 && rb_cross(hull[k - 2], hull[k - 1], pts[i]) <= 0) --k;
      hull[k++] = pts[i];
    }
    for (int i = n - 2, t = k + 1; i >= 0; --i) {
      while (k >= t && rb_cross(hull[k - 2], hull[k - 1], pts[i]) <= 0) --k;
      hull[k++] = pts[i];
    }
    s_M = k - 1;                                               // the last point repeats the first
  }
  __syncthreads();
  const int M = s_M;
  for (int i = threadIdx.x; i < M; i += blockDim.x) {         // edge i: area * |e|^2 and |e|^2
    const RbExtent e = rb_extent(hull, M, i);
    const int2 p = hull[i], q = hull[i + 1 == M ? 0 : i + 1];
    qa[2 * i] = (unsigned long long)((e.amax - e.amin) * (e.bmax - e.bmin));
    qa[2 * i + 1] = (unsigned long long)((int64_t)(q.x - p.x) * (q.x - p.x) + (int64_t)(q.y - p.y) * (q.y - p.y));
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  int bi = 0;
  for (int i = 1; i < M; ++i)                                  // exact: Q_i / L_i < Q_b / L_b; the first of equals stays
    if ((unsigned __int128)qa[2 * i] * qa[2 * bi + 1] < (unsigned __int128)qa[2 * bi] * qa[2 * i + 1]) bi = i;
  const RbExtent e = rb_extent(hull, M, bi);
  const int2 p = hull[bi], q = hull[bi + 1 == M ? 0 : bi + 1];
  const int64_t ex = q.x - p.x, ey = q.y - p.y;
  // boxPoints' width direction (cv2 4.x angle in [-90, 0)): the rotation k of e with x >= 0 and y < 0
  const int64_t rx[4] = {ex, -ey, -ex, ey}, ry[4] = {ey, ex, -ey, -ex};
  int k = 0;
  while (!(rx[k] >= 0 && ry[k] < 0)) ++k;
  const int64_t ca[4] = {e.amin, e.amin, e.amax, e.amax}, cb[4] = {e.bmax, e.bmin, e.bmin, e.bmax};
  const double L = (double)(ex * ex + ey * ey);
  for (int j = 0; j < 4; ++j) {
    const int64_t a = ca[(k + j) & 3], bb = cb[(k + j) & 3];
    const double nx = (double)(a * ex - bb * ey), ny = (double)(a * ey + bb * ex);
    out[2 * j] = (double)__double2float_rn(__dadd_rn((double)p.x, __ddiv_rn(nx, L)));
    out[2 * j + 1] = (double)__double2float_rn(__dadd_rn((double)p.y, __ddiv_rn(ny, L)));
  }
  flag[b] = 1;
  area2[b] = (int64_t)(key >> 32);
}

}  // namespace

size_t rotated_box_workspace_size(int64_t total, int N, int max_h) {
  const size_t a = (size_t)total * sizeof(int32_t);
  const size_t per = (size_t)N * (sizeof(unsigned long long)                       // best
                                  + 2 * (size_t)max_h * sizeof(int32_t)            // row extremes
                                  + 2 * (size_t)max_h * sizeof(int2)               // sorted points
                                  + (2 * (size_t)max_h + 1) * sizeof(int2)         // hull
                                  + 2 * (2 * (size_t)max_h + 1) * sizeof(unsigned long long));
  return ((a + 15) / 16) * 16 + per + 64;
}

void launch_rotated_box(const uint8_t* masks, const sm_image_desc* desc, int N, int max_h, int max_w,
                        const double* fallback, void* workspace, double* poly, int32_t* flag, int64_t* area2,
                        int64_t total, cudaStream_t st) {
  char* w = static_cast<char*>(workspace);
  int32_t* lab = reinterpret_cast<int32_t*>(w);
  w += (((size_t)total * sizeof(int32_t) + 15) / 16) * 16;
  auto* best = reinterpret_cast<unsigned long long*>(w);
  w += (size_t)N * sizeof(unsigned long long);
  auto* qa = reinterpret_cast<unsigned long long*>(w);
  w += (size_t)N * 2 * (2 * (size_t)max_h + 1) * sizeof(unsigned long long);
  auto* pts = reinterpret_cast<int2*>(w);
  w += (size_t)N * 2 * max_h * sizeof(int2);
  auto* hull = reinterpret_cast<int2*>(w);
  w += (size_t)N * (2 * (size_t)max_h + 1) * sizeof(int2);
  auto* rows = reinterpret_cast<int32_t*>(w);
  const int64_t px = (int64_t)max_h * max_w;
  const dim3 grid((unsigned)std::min<int64_t>((px + RB_THREADS - 1) / RB_THREADS, 1024), (unsigned)N);
  rb_init<<<grid, RB_THREADS, 0, st>>>(masks, desc, lab, best, rows, max_h);
  SMK_CUDA(cudaGetLastError());
  rb_merge<<<grid, RB_THREADS, 0, st>>>(masks, desc, lab);
  SMK_CUDA(cudaGetLastError());
  rb_flatten<<<grid, RB_THREADS, 0, st>>>(desc, lab);
  SMK_CUDA(cudaGetLastError());
  rb_trace<<<grid, RB_THREADS, 0, st>>>(masks, desc, lab, best);
  SMK_CUDA(cudaGetLastError());
  rb_rows<<<grid, RB_THREADS, 0, st>>>(desc, lab, best, rows, max_h);
  SMK_CUDA(cudaGetLastError());
  rb_rect<<<N, RB_RECT_THREADS, 0, st>>>(desc, rows, best, fallback, max_h, pts, hull, qa, poly, flag, area2);
  SMK_CUDA(cudaGetLastError());
}

}  // namespace smk
