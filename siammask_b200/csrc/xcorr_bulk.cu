// Standalone depthwise cross-correlation `conv2d_dw_group` (models/rpn.py:32-38), fp32 NCHW, for sm_90a:
//   out[p][i][j] = sum_{u,v<5} x[p][i+u][j+v] * k[p][u][v]      p = (b, c) plane, valid, no flip.
// HBM-bound (5.2 FLOP/B).  The operand planes of one (b,c) are contiguous in memory and so are consecutive planes,
// therefore a tile of G planes is ONE contiguous byte range on each side:
//   * a copy warp stages x (G*H*W*4 B) and k (G*100 B) of a tile into shared memory with `cp.async.bulk`
//     (1-D TMA, SASS UBLKCP) signalling an mbarrier, two stages deep, and drains the results with a bulk store
//     (smem -> global) — no LSU instruction touches HBM, every request is a multi-KB burst;
//   * compute warps map LANE = PLANE (32 consecutive planes; the plane pitch H*W is odd, so every shared-memory access of
//     a warp is bank-conflict free) and WARP = a (row block x 5-column strip) task: a thread slides a 5-row window down
//     its strip, 9 loads feed 125 FMAs per output row (the previous one-warp-per-plane kernel spent an instruction
//     slot per 0.75 FMA on loads, shuffles and idle lanes and stalled at 0.36 of the HBM roofline);
//   * results stay in registers until every warp has finished reading the stage, are then written over the stage's
//     own (dead) input bytes and leave through the bulk store, so two stages of 32 planes fit the 227 KB.
// Generic geometry (other H/W, e.g. 45x45 @ search 383) runs the same pipeline with G planes x 32/G tasks per warp.
#include "common.cuh"
#include "ptx.cuh"

namespace smk {

namespace {

__device__ __forceinline__ void bulk_load(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_store(void* dst, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src_smem)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void named_barrier(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

constexpr int KH = 5, KW = 5;

// One task: output rows [r0, r0+NR) x columns [c0, c0+SW) of one plane.  NR/SW are compile-time so the window indices
// are.  STATIC = the task is exactly NR x SW (no clipping: straight-line code without predicates); otherwise `nr`/`nc`
// (<= NR/SW) clip the last row block / strip.
template <int W, int Wo, int NR, int SW, bool STATIC>
__device__ __forceinline__ void xcorr_task(const float* __restrict__ xp, const float (&kk)[KH][KW], int r0, int c0,
                                           int nr, int nc, float (&acc)[NR][SW]) {
#pragma unroll
  for (int i = 0; i < NR; ++i)
#pragma unroll
    for (int c = 0; c < SW; ++c) acc[i][c] = 0.f;
  const float* row = xp + r0 * W + c0;
  const int ncol_in = nc + KW - 1;
#pragma unroll
  for (int r = 0; r < NR + KH - 1; ++r) {      // input row r0 + r feeds output rows r0 + r - u
    if (STATIC || r < nr + KH - 1) {
      float xr[SW + KW - 1];
#pragma unroll
      for (int c = 0; c < SW + KW - 1; ++c) xr[c] = (STATIC || c < ncol_in) ? row[r * W + c] : 0.f;
#pragma unroll
      for (int u = 0; u < KH; ++u) {
        const int i = r - u;
        if (i >= 0 && i < NR && (STATIC || i < nr)) {
#pragma unroll
          for (int c = 0; c < SW; ++c)
#pragma unroll
            for (int v = 0; v < KW; ++v) acc[i][c] = fmaf(xr[c + v], kk[u][v], acc[i][c]);
        }
      }
    }
  }
}

template <int Wo, int NR, int SW>
__device__ __forceinline__ void xcorr_store(float* __restrict__ op, const float (&acc)[NR][SW], int nr, int nc) {
#pragma unroll
  for (int i = 0; i < NR; ++i)
    if (i < nr) {
#pragma unroll
      for (int c = 0; c < SW; ++c)
        if (c < nc) op[i * Wo + c] = acc[i][c];
    }
}

// G planes per stage; tasks = NRB row blocks x NST strips per plane; a warp carries 32/G tasks of G planes.
template <int H, int W, int G, int NR, int SW, int NWARPS>
__global__ void __launch_bounds__(NWARPS * 32 + 32, 1)
xcorr_bulk_kernel(const float* __restrict__ x, const float* __restrict__ k, float* __restrict__ out, int tiles) {
  constexpr int Ho = H - KH + 1, Wo = W - KW + 1;
  constexpr int NRB = (Ho + NR - 1) / NR, NST = (Wo + SW - 1) / SW;
  constexpr int TPW = 32 / G;                              // tasks per warp
  constexpr int IN_BYTES = G * H * W * 4, K_BYTES = G * KH * KW * 4, OUT_BYTES = G * Ho * Wo * 4;
  constexpr int STAGE_BYTES = (IN_BYTES + K_BYTES + 127) / 128 * 128;
  static_assert(IN_BYTES % 16 == 0 && K_BYTES % 16 == 0 && OUT_BYTES % 16 == 0, "bulk copies move 16-byte units");
  static_assert(NRB * NST <= NWARPS * TPW, "not enough warps for the tasks of a stage");
  extern __shared__ __align__(128) uint8_t smem_x[];
  __shared__ uint64_t full_bar[2], ready_bar[2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&ready_bar[s], NWARPS);                    // one arrival per compute warp
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  const int my_tiles = (tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (warp == NWARPS) {
    // ===================== copy warp =====================
    if (lane == 0) {
      auto load = [&](int it) {
        const size_t tile = (size_t)blockIdx.x + (size_t)it * gridDim.x;
        const int s = it & 1;
        uint8_t* st = smem_x + s * STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[s], IN_BYTES + K_BYTES);
        bulk_load(st, reinterpret_cast<const uint8_t*>(x) + tile * IN_BYTES, IN_BYTES, &full_bar[s]);
        bulk_load(st + IN_BYTES, reinterpret_cast<const uint8_t*>(k) + tile * K_BYTES, K_BYTES, &full_bar[s]);
      };
      for (int it = 0; it < 2 && it < my_tiles; ++it) load(it);
      for (int it = 0; it < my_tiles; ++it) {
        const int s = it & 1;
        const uint32_t ph = (it >> 1) & 1;
        mbar_wait(&ready_bar[s], ph);                      // results of tile `it` sit at the start of stage s
        const size_t tile = (size_t)blockIdx.x + (size_t)it * gridDim.x;
        bulk_store(reinterpret_cast<uint8_t*>(out) + tile * OUT_BYTES, smem_x + s * STAGE_BYTES, OUT_BYTES);
        tma_store_commit();
        if (it + 2 < my_tiles) {
          tma_store_wait_read<0>();                        // the store has read the stage: refill it
          load(it + 2);
        }
      }
      tma_store_wait_all();
    }
    return;
  }

  // ===================== compute warps =====================
  const int plane = lane % G;
  const int task = warp * TPW + lane / G;                  // warp-uniform when G == 32
  const bool has_task = task < NRB * NST;
  const int rb = has_task ? task / NST : 0, stp = has_task ? task % NST : 0;
  // balanced split: the first (Ho - NRB*(NR-1)) row blocks have NR rows, the rest NR-1 (25 rows -> 7,6,6,6); same for
  // the strips (41 columns -> 6,6,6,6,6,6,5)
  constexpr int R_EXTRA = Ho - NRB * (NR - 1), C_EXTRA = Wo - NST * (SW - 1);
  static_assert(R_EXTRA >= 1 && R_EXTRA <= NRB && C_EXTRA >= 1 && C_EXTRA <= NST, "balanced task split");
  const int r0 = rb * (NR - 1) + min(rb, R_EXTRA), c0 = stp * (SW - 1) + min(stp, C_EXTRA);
  const int nr = NR - 1 + (rb < R_EXTRA ? 1 : 0), nc = SW - 1 + (stp < C_EXTRA ? 1 : 0);
  for (int it = 0; it < my_tiles; ++it) {
    const int s = it & 1;
    const uint32_t ph = (it >> 1) & 1;
    uint8_t* st = smem_x + s * STAGE_BYTES;
    mbar_wait(&full_bar[s], ph);
    const float* ks = reinterpret_cast<const float*>(st + IN_BYTES) + plane * (KH * KW);
    const float* xp = reinterpret_cast<const float*>(st) + plane * (H * W);
    float* op = reinterpret_cast<float*>(st) + plane * (Ho * Wo) + r0 * Wo + c0;
    float kk[KH][KW];
    if (has_task) {
#pragma unroll
      for (int u = 0; u < KH; ++u)
#pragma unroll
        for (int v = 0; v < KW; ++v) kk[u][v] = ks[u * KW + v];
    }
    if constexpr (G == 32 && C_EXTRA == NST && NRB * NST == NWARPS) {
      // the task is warp-uniform and every strip is SW wide: full-size and one-row-short blocks get their own
      // straight-line code (no predicates)
      if (nr == NR) {
        float acc[NR][SW];
        xcorr_task<W, Wo, NR, SW, true>(xp, kk, r0, c0, NR, SW, acc);
        named_barrier(1, NWARPS * 32);                     // every warp has consumed the stage's inputs
        xcorr_store<Wo, NR, SW>(op, acc, NR, SW);
      } else {
        float acc[NR - 1][SW];
        xcorr_task<W, Wo, NR - 1, SW, true>(xp, kk, r0, c0, NR - 1, SW, acc);
        named_barrier(1, NWARPS * 32);
        xcorr_store<Wo, NR - 1, SW>(op, acc, NR - 1, SW);
      }
    } else {
      float acc[NR][SW];
      if (has_task) xcorr_task<W, Wo, NR, SW, false>(xp, kk, r0, c0, nr, nc, acc);
      named_barrier(1, NWARPS * 32);
      if (has_task) xcorr_store<Wo, NR, SW>(op, acc, nr, nc);
    }
    fence_proxy_async();                                   // generic-proxy writes -> visible to the bulk store
    __syncwarp();
    if (lane == 0) mbar_arrive(&ready_bar[s]);
  }
}

template <int H, int W, int G, int NR, int SW, int NWARPS>
void launch_bulk(const float* x, const float* k, float* out, int tiles, cudaStream_t st) {
  constexpr int IN_BYTES = G * H * W * 4, K_BYTES = G * 100;
  constexpr int STAGE_BYTES = (IN_BYTES + K_BYTES + 127) / 128 * 128;
  constexpr int SMEM = 2 * STAGE_BYTES;
  static_assert(SMEM <= 226 * 1024, "two stages must fit shared memory");
  auto kern = xcorr_bulk_kernel<H, W, G, NR, SW, NWARPS>;
  static unsigned long long attr = 0;
  ensure_dynamic_smem(kern, SMEM, attr);
  int dev = 0, sms = 132;
  SMK_CUDA(cudaGetDevice(&dev));
  SMK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = tiles < sms ? tiles : sms;
  kern<<<grid, NWARPS * 32 + 32, SMEM, st>>>(x, k, out, tiles);
  SMK_CUDA(cudaGetLastError());
}

}  // namespace

// Returns the number of leading planes handled (a multiple of the tile size); the caller runs the remainder (and
// unsupported geometries: returns 0) through the one-warp-per-plane kernel.
int launch_xcorr_bulk_f32(const float* x, const float* k, float* out, int planes, int H, int W, int kh, int kw,
                          cudaStream_t st) {
  if (kh != 5 || kw != 5) return 0;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(out)) & 15) return 0;
  if (H == 29 && W == 29) {           // search 255: 25x25 response; 32 planes per stage, 4 row blocks (7,6,6,6) x 5 strips
    const int tiles = planes / 32;
    if (tiles > 0) launch_bulk<29, 29, 32, 7, 5, 20>(x, k, out, tiles, st);
    return tiles * 32;
  }
  if (H == 45 && W == 45) {           // search 383: 41x41 response; 8 planes per stage, 6 row blocks x 7 strips of 6
    const int tiles = planes / 8;
    if (tiles > 0) launch_bulk<45, 45, 8, 7, 6, 11>(x, k, out, tiles, st);
    return tiles * 8;
  }
  return 0;
}

}  // namespace smk
