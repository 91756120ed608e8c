// Implicit-GEMM convolution on the Hopper tensor cores (wgmma) for sm_90a.
//
//   out[m][n] = epilogue( sum_k A[m][k] * W[n][k] ),  m = (b, ho, wo) flattened, k = (r, s, c) with c fastest.
//
// * A (NHWC fp16 activation planes) is staged by TMA: plain 2-D tiles for 1x1/stride-1 convs, im2col-mode
//   tiles (cp.async.bulk.tensor.4d...im2col) for everything else — padding, stride and dilation are resolved
//   by the TMA unit, out-of-image taps arrive as zeros, and the 128-pixel M tile runs across row and image
//   boundaries so batch absorbs the odd spatial sizes (31x31, 29x29, 25x25 ...).
// * W (K-major fp16, [Cout_pad][KH*KW*Cin]) is staged by 2-D TMA tiles.  Both land in swizzled smem (128 B rows for
//   64-wide k-blocks, 64 B rows for 32-wide ones, see Cfg), in a ring of k-block stages guarded by full / empty
//   mbarriers, and are consumed by wgmma.mma_async (M=64 per warpgroup, N=BLOCK_N, K=16) accumulating in fp32
//   registers.
// * Precision: NSPLIT=1 multiplies the fp16 hi planes only.  NSPLIT=2 ("exact") keeps activations and
//   weights as hi+lo fp16 pairs (22 significant bits) and issues three MMAs per k-step
//   (hi*hi into one accumulator, hi*lo + lo*hi into a second one, summed in the epilogue: the tensor pipe truncates
//   on every accumulate, so the small cross terms must not be fed into the large running sum) — fp32-class results
//   from the fp16 tensor pipe.
// * K may consist of up to two segments that accumulate into the same tile: (conv over input 0) + (conv over
//   input 1) fuses a bottleneck's downsample branch with its conv3.
// * Epilogue: acc*alpha[c]+beta[c] (+ residual*res_scale) (ReLU).  NHWC outputs (split fp16 planes or fp32) are
//   written into a per-warpgroup staging buffer in the swizzled layout of 64-row TMA boxes and leave by TMA stores
//   that overlap the warpgroup's next tile; a residual tile arrives in the same buffer by TMA, loaded by the producer
//   while the tile's k-blocks run.  NCHW fp32 outputs (the reference's boundary layout, tools/test.py:205-206) are
//   written straight from the accumulator registers: a 64-row box cannot follow an M tile across the image boundary.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one elected lane of warp 0; the warpgroup hands most of its
// registers to the consumers), warpgroups 1 and 2 = consumers, each computing 64 of the tile's 128 rows and writing
// them out.  Persistent: grid = min(tiles, SMs), static round-robin over (m_tile, n_tile).
#include "common.cuh"
#include "ptx.cuh"

#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>

namespace smk {

namespace {

constexpr int BLOCK_M = 128;
constexpr int WG_ROWS = 64;     // tile rows per consumer warpgroup (one staging buffer, one store box row range)
constexpr int CIN_GRAIN = 64;   // convs need Cin % 64 == 0
constexpr int MMA_K = 16;
constexpr int SMEM_LIMIT = 227 * 1024;
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int NUM_THREADS = 128 + 32 * NUM_CONSUMER_WARPS;
// register split between the producer warpgroup and the two consumer warpgroups (128*40 + 256*232 <= 64 K)
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;

template <int BLOCK_N, int NSPLIT>
struct Cfg {
  // epilogue staging per consumer warpgroup: 64 rows x BLOCK_N at 4 bytes (fp32, or hi + lo fp16 planes; a residual's
  // planes arrive in the same bytes)
  static constexpr int STAGING_BYTES = WG_ROWS * BLOCK_N * 4;
  static constexpr int RING_BYTES = SMEM_LIMIT - 2048 - 2 * STAGING_BYTES;
  static constexpr int stage_bytes(int bk) { return NSPLIT * (BLOCK_M + BLOCK_N) * bk * 2; }
  // 64-wide k-blocks (128 B swizzle) unless fewer than three of them fit beside the staging buffers, which happens in
  // exact mode at N = 128: there 32-wide k-blocks (64 B swizzle) keep five stages in flight
  static constexpr int BLOCK_K = RING_BYTES / stage_bytes(64) >= 3 ? 64 : 32;
  static constexpr int SW = BLOCK_K * 2;                 // operand swizzle span = k-block row in bytes
  static constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_TILE_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = NSPLIT * (A_TILE_BYTES + B_TILE_BYTES);
  static constexpr int RAW_STAGES = RING_BYTES / STAGE_BYTES;
  static constexpr int STAGES = RAW_STAGES > 6 ? 6 : RAW_STAGES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * STAGING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int ACC = BLOCK_N / 2;               // fp32 accumulator registers per thread and accumulator
  // store / residual boxes: 64 rows of at most 128 bytes; the swizzle span equals the box row
  static constexpr int H_BOX = BLOCK_N < 64 ? BLOCK_N : 64;   // fp16 columns per box
  static constexpr int F_BOX = BLOCK_N < 32 ? BLOCK_N : 32;   // fp32 columns per box
  static constexpr int H_PLANE = WG_ROWS * BLOCK_N * 2;       // one fp16 plane of a warpgroup's rows
  static_assert(STAGES >= 3, "pipeline needs at least three stages");
  static_assert(BLOCK_N % 16 == 0 && BLOCK_N >= 16 && BLOCK_N <= 128, "N tile (register accumulators)");
  static_assert(STAGE_BYTES % 1024 == 0 && B_TILE_BYTES % 1024 == 0, "stage parts stay 1024-aligned (swizzle atoms)");
  static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory budget");
};

// tile -> M block.  With reverse_m the persistent CTAs walk the M tiles from the end: a layer then starts on the rows
// its producer wrote last, which are the ones still resident in L2.
__device__ __forceinline__ int m_block(const GemmParams& p, int tile) {
  const int mb = tile / p.n_tiles;
  return p.reverse_m ? p.m_tiles - 1 - mb : mb;
}

// byte offset inside a TMA box of SPAN-byte rows -> its swizzled smem offset (the box starts 1024-aligned): the 16-byte
// chunk index is XORed with the row's position in the 1024-byte swizzle atom
template <int SPAN>
__device__ __forceinline__ uint32_t swizzle(uint32_t o) {
  return o ^ (((o >> 7) & (SPAN / 16 - 1)) << 4);
}

__device__ __forceinline__ void named_barrier_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

template <int BLOCK_N, int NSPLIT>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_gemm_kernel(const __grid_constant__ GemmParams p) {
  using C = Cfg<BLOCK_N, NSPLIT>;
  constexpr int STAGES = C::STAGES;
  constexpr int BLOCK_K = C::BLOCK_K;
  constexpr int A_TILE_BYTES = C::A_TILE_BYTES;

  extern __shared__ uint8_t smem_raw[];
  // 1024-aligned by pointer arithmetic on smem_raw, so the epilogue's staging accesses stay st/ld.shared
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* staging = smem + STAGES * C::STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + 2 * C::STAGING_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* free_bar = empty_bar + STAGES;   // [wg]: the warpgroup's previous TMA store has read its staging buffer
  uint64_t* res_bar = free_bar + 2;          // [wg]: the residual tile has landed in the staging buffer

  // warp index through a shuffle: provably warp-uniform for the compiler, so the role branches below are convergent
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    for (int i = 0; i < NSPLIT; ++i) {
      for (int sgi = 0; sgi < p.nseg; ++sgi) tma_prefetch_desc(&p.seg[sgi].tmA[i]);
      tma_prefetch_desc(&p.tmB[i]);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], NUM_CONSUMER_WARPS);   // one arrival per consumer warp
    }
    for (int w = 0; w < 2; ++w) {
      mbar_init(&free_bar[w], 1);
      mbar_init(&res_bar[w], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp != 0) return;
    const bool leader = elect_one();
    int stage = 0;
    uint32_t phase = 0;
    uint32_t iter = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++iter) {
      const int m0 = m_block(p, tile) * BLOCK_M;
      const int n0 = (tile % p.n_tiles) * BLOCK_N;
      const int q = m0 % p.Wo;
      const int t = m0 / p.Wo;
      const int pq = t % p.Ho;
      const int nb = t / p.Ho;
      for (int sgi = 0; sgi < p.nseg; ++sgi) {
        const GemmSegment& sg = p.seg[sgi];
        const int wb = q * sg.stride - sg.pad;
        const int hb = pq * sg.stride - sg.pad;
#pragma unroll 1
        for (int kb = 0; kb < sg.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          if (leader) mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          uint8_t* st = smem + stage * C::STAGE_BYTES;
          const int tap = kb / sg.cblks;
          const int c0 = (kb - tap * sg.cblks) * BLOCK_K;
#pragma unroll
          for (int s = 0; s < NSPLIT; ++s) {
            uint8_t* a_dst = st + s * A_TILE_BYTES;
            if (leader) {
              if (sg.mode == 0) {
                tma_load_2d(a_dst, &sg.tmA[s], &full_bar[stage], c0, m0);
              } else {
                const int r = tap / sg.KW;
                const int sx = tap - r * sg.KW;
                tma_load_im2col_4d(a_dst, &sg.tmA[s], &full_bar[stage], c0, wb, hb, nb,
                                   static_cast<uint16_t>(sx * sg.dil), static_cast<uint16_t>(r * sg.dil));
              }
              tma_load_2d(st + NSPLIT * A_TILE_BYTES + s * C::B_TILE_BYTES, &p.tmB[s], &full_bar[stage],
                          sg.b_col0 + kb * BLOCK_K, n0);
            }
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      if (p.has_res) {
        // the residual tile of each warpgroup, into its staging buffer once the previous tile's store has read it
        // (the consumers signal that after their first k-block of this tile, which is already in the ring)
#pragma unroll 1
        for (int w = 0; w < 2; ++w) {
          mbar_wait(&free_bar[w], iter & 1);
          const int r0 = m0 + w * WG_ROWS;
          if (leader) {
            mbar_arrive_expect_tx(&res_bar[w], r0 < p.M ? NSPLIT * C::H_PLANE : 0);
            if (r0 < p.M) {
              uint8_t* dst = staging + w * C::STAGING_BYTES;
#pragma unroll
              for (int s = 0; s < NSPLIT; ++s)
#pragma unroll
                for (int b = 0; b < BLOCK_N / C::H_BOX; ++b)
                  tma_load_2d(dst + s * C::H_PLANE + b * (WG_ROWS * C::H_BOX * 2), &p.tmR[s], &res_bar[w],
                              n0 + b * C::H_BOX, r0);
            }
          }
          __syncwarp();
        }
      }
    }
    return;
  }

  // ===================== consumers: MMA + epilogue, 64 tile rows per warpgroup =====================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = (warp >> 2) - 1;
  const int wl = warp & 3;
  const bool store_thread = wl == 0 && lane == 0;     // issues (and later waits for) the warpgroup's TMA stores
  const Epilogue& ep = p.ep;
  const int HoWo = p.Ho * p.Wo;
  uint8_t* my_staging = staging + wg * C::STAGING_BYTES;
  float acc[C::ACC];
  float acc2[C::ACC];     // exact mode: the hi*lo + lo*hi cross terms
  int stage = 0;
  uint32_t phase = 0;
  uint32_t iter = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++iter) {
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) { acc[i] = 0.f; acc2[i] = 0.f; }
    int prev = -1;
    for (int sgi = 0; sgi < p.nseg; ++sgi) {
      const int nkb = p.seg[sgi].num_kb;
#pragma unroll 1
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_hi = smem_u32(smem + stage * C::STAGE_BYTES) + wg * (WG_ROWS * BLOCK_K * 2);
        const uint32_t b_hi = smem_u32(smem + stage * C::STAGE_BYTES) + NSPLIT * A_TILE_BYTES;
        const uint64_t da_hi0 = wgmma_desc_kmajor<C::SW>(a_hi);
        const uint64_t db_hi0 = wgmma_desc_kmajor<C::SW>(b_hi);
        const uint64_t da_lo0 = wgmma_desc_kmajor<C::SW>(a_hi + A_TILE_BYTES);
        const uint64_t db_lo0 = wgmma_desc_kmajor<C::SW>(b_hi + C::B_TILE_BYTES);
        // one MMA sequence for every k-block: a data-dependent branch between in-flight wgmma groups makes ptxas
        // insert warpgroup.arrive serialisation around the accumulators
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
          const uint64_t kadd = static_cast<uint64_t>(k * MMA_K * 2 / 16);
          wgmma_f16<BLOCK_N>(acc, da_hi0 + kadd, db_hi0 + kadd);
          if constexpr (NSPLIT == 2) {
            wgmma_f16<BLOCK_N>(acc2, da_hi0 + kadd, db_lo0 + kadd);
            wgmma_f16<BLOCK_N>(acc2, da_lo0 + kadd, db_hi0 + kadd);
          }
        }
        wgmma_commit();
        // keep this k-block's MMAs in flight; the previous k-block's have finished reading their stage
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        } else if (store_thread) {
          // first k-block of the tile is in flight: by now the previous tile's store has long read the staging buffer
          tma_store_wait_read<0>();
          mbar_arrive(&free_bar[wg]);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if constexpr (NSPLIT == 2) fence_regs(acc2);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);

    // ---- epilogue: thread holds tile rows rl, rl + 8 (of its warpgroup's 64) and column pairs 2 * (lane & 3) + 8j
    // (see wgmma_f16)
    const int m0 = m_block(p, tile) * BLOCK_M + wg * WG_ROWS;
    const int n0 = (tile % p.n_tiles) * BLOCK_N;
    const int rl = wl * 16 + (lane >> 2);
    const int cl = 2 * (lane & 3);
    if (ep.out_mode == OUT_NCHW_F32) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + rl + 8 * h;
        if (m >= p.M) continue;
        const int b = m / HoWo;
        const int hw = m - b * HoWo;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int n = n0 + cl + 8 * j;
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if constexpr (NSPLIT == 2) {
            v0 += acc2[4 * j + 2 * h];
            v1 += acc2[4 * j + 2 * h + 1];
          }
          const float2 al = __ldg(reinterpret_cast<const float2*>(ep.alpha + n));
          const float2 be = __ldg(reinterpret_cast<const float2*>(ep.beta + n));
          v0 = fmaf(v0, al.x, be.x);
          v1 = fmaf(v1, al.y, be.y);
          if (ep.relu) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
          if (n < p.Cout) {  // write-once output: stream past L2; the last N tile may be ragged
            float* dst = ep.out_f32 + (static_cast<size_t>(b) * p.Cout + n) * HoWo + hw;
            __stcs(dst, v0);
            if (n + 1 < p.Cout) __stcs(dst + HoWo, v1);
          }
        }
      }
      continue;
    }

    // staged NHWC epilogue.  The residual's arrival implies the previous store has read the buffer (the producer
    // waited for that before loading it); without a residual, wait for that directly.
    mbar_wait(p.has_res ? &res_bar[wg] : &free_bar[wg], iter & 1);
    const bool split = ep.out_mode == OUT_NHWC_SPLIT;
    const bool two_planes = ep.out_lo != nullptr;
    float amax = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rl + 8 * h;
      const bool row_in = m0 + r < p.M;    // rows past M are clipped by the store; they carry beta, keep them out of amax
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int c = cl + 8 * j;
        const int n = n0 + c;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if constexpr (NSPLIT == 2) {
          v0 += acc2[4 * j + 2 * h];
          v1 += acc2[4 * j + 2 * h + 1];
        }
        const float2 al = __ldg(reinterpret_cast<const float2*>(ep.alpha + n));
        const float2 be = __ldg(reinterpret_cast<const float2*>(ep.beta + n));
        v0 = fmaf(v0, al.x, be.x);
        v1 = fmaf(v1, al.y, be.y);
        // fp16 planes: box c / H_BOX, 2-byte columns
        const uint32_t oh = (c / C::H_BOX) * (WG_ROWS * C::H_BOX * 2) +
                            swizzle<C::H_BOX * 2>(r * (C::H_BOX * 2) + (c % C::H_BOX) * 2);
        if (p.has_res) {
          float2 f = __half22float2(*reinterpret_cast<const __half2*>(my_staging + oh));
          if constexpr (NSPLIT == 2) {
            const float2 l = __half22float2(*reinterpret_cast<const __half2*>(my_staging + C::H_PLANE + oh));
            f.x += l.x;
            f.y += l.y;
          }
          v0 += f.x * ep.res_scale;
          v1 += f.y * ep.res_scale;
        }
        if (ep.relu) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        if (split) {
          if (row_in) amax = fmaxf(amax, fmaxf(fabsf(v0), fabsf(v1)));
          const __half2 hv = __floats2half2_rn(v0, v1);
          const float2 hf = __half22float2(hv);
          *reinterpret_cast<__half2*>(my_staging + oh) = hv;
          if (two_planes)
            *reinterpret_cast<__half2*>(my_staging + C::H_PLANE + oh) = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
        } else {
          const uint32_t of = (c / C::F_BOX) * (WG_ROWS * C::F_BOX * 4) +
                              swizzle<C::F_BOX * 4>(r * (C::F_BOX * 4) + (c % C::F_BOX) * 4);
          *reinterpret_cast<float2*>(my_staging + of) = make_float2(v0, v1);
        }
      }
    }
    // generic-proxy writes -> visible to the TMA unit, then one thread stores the warpgroup's boxes
    fence_proxy_async();
    named_barrier_sync(1 + wg, 128);
    if (store_thread && m0 < p.M) {
      if (split) {
        for (int s = 0; s < (two_planes ? 2 : 1); ++s)
#pragma unroll
          for (int b = 0; b < BLOCK_N / C::H_BOX; ++b)
            tma_store_2d(&p.tmO[s], my_staging + s * C::H_PLANE + b * (WG_ROWS * C::H_BOX * 2), n0 + b * C::H_BOX, m0);
      } else {
#pragma unroll
        for (int b = 0; b < BLOCK_N / C::F_BOX; ++b)
          tma_store_2d(&p.tmO[0], my_staging + b * (WG_ROWS * C::F_BOX * 4), n0 + b * C::F_BOX, m0);
      }
      tma_store_commit();
    }
    if (split) flag_if_out_of_range(amax, ep.ovf);
  }
  if (store_thread) tma_store_wait_all();
}

// ------------------------------------------------------------------ host side: tensor maps
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
using EncodeIm2colFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct DriverApi {
  EncodeTiledFn tiled = nullptr;
  EncodeIm2colFn im2col = nullptr;
  int driver_version = 0;
};

// The driver entry points are resolved at run time so the library has no link-time libcuda
// dependency (it must load on a box without a GPU driver for the symbol-export test).
const DriverApi& driver_api() {
  static DriverApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    SMK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    SMK_CHECK(fn != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
    api.tiled = reinterpret_cast<EncodeTiledFn>(fn);
    fn = nullptr;
    SMK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q));
    SMK_CHECK(fn != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeIm2col not available");
    api.im2col = reinterpret_cast<EncodeIm2colFn>(fn);
    SMK_CUDA(cudaDriverGetVersion(&api.driver_version));
  });
  return api;
}

// Tensor-map cache.  cuTensorMapEncode* costs a few microseconds on the host and a launch needs up to eight maps; the
// engine's bump arenas hand out the same addresses every step, so the (pointer, geometry) key of every map repeats from
// the second step on.  Keyed by the encode arguments themselves, so a hit is exactly what the driver would build.
struct MapKey {
  uint64_t v[16];
  bool operator==(const MapKey& o) const { return std::memcmp(v, o.v, sizeof v) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = 0x9E3779B97F4A7C15ull;
    for (uint64_t x : k.v) { h ^= x + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); }
    return (size_t)h;
  }
};
template <typename F>
CUtensorMap cached_map(const MapKey& key, F&& encode) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  int dev = 0;
  cudaGetDevice(&dev);
  MapKey k = key;
  k.v[15] = (uint64_t)dev;
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(k);
  if (it != cache.end()) return it->second;
  if (cache.size() > 65536) cache.clear();             // unbounded callers (standalone ops on fresh buffers)
  CUtensorMap m = encode();
  cache.emplace(k, m);
  return m;
}

CUtensorMap make_map_2d_raw(const __half* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer) {
  CUtensorMap m;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {inner * sizeof(__half)};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  // operand tiles: the swizzle span equals the k-block row (64 fp16 -> 128 B, 32 fp16 -> 64 B)
  const CUtensorMapSwizzle sw = box_inner == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = driver_api().tiled(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides,
                                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SMK_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed, code " + std::to_string((int)r));
  return m;
}

CUtensorMap make_map_2d(const __half* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer) {
  MapKey k{};
  k.v[0] = 1; k.v[1] = (uint64_t)base; k.v[2] = inner; k.v[3] = outer; k.v[4] = box_inner; k.v[5] = box_outer;
  return cached_map(k, [&] { return make_map_2d_raw(base, inner, outer, box_inner, box_outer); });
}

CUtensorMap make_map_im2col_raw(const __half* base, const Act& in, const ConvGeom& g, int bk) {
  CUtensorMap m;
  cuuint64_t dims[4] = {(cuuint64_t)in.C, (cuuint64_t)in.W, (cuuint64_t)in.H, (cuuint64_t)in.B};
  cuuint64_t strides[3] = {(cuuint64_t)in.C * 2, (cuuint64_t)in.W * in.C * 2, (cuuint64_t)in.H * in.W * in.C * 2};
  // fprop corners (cutlass/conv/collective/detail.hpp compute_{lower,upper}_corner_whd):
  //   lower = -pad, upper = pad - (k-1)*dilation; base pixel = lower + q*stride, tap offset = s*dilation.
  int lower[2] = {-g.pad, -g.pad};
  int upper[2] = {g.pad - (g.KW - 1) * g.dil, g.pad - (g.KH - 1) * g.dil};
  cuuint32_t estr[4] = {1, (cuuint32_t)g.stride, (cuuint32_t)g.stride, 1};
  const DriverApi& api = driver_api();
  CUresult r = api.im2col(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(base), dims, strides, lower,
                          upper, bk, BLOCK_M, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SMK_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeIm2col failed, code " + std::to_string((int)r));
  // Same small-tensor descriptor fix-up CuTe applies for drivers <= 13.1
  // (cute/atom/copy_traits_sm90_im2col.hpp, make_im2col_tma_copy_desc).
  if (api.driver_version <= 13010 && in.numel() * sizeof(__half) < 131072)
    reinterpret_cast<uint64_t*>(&m)[1] &= ~(1ull << 21);
  return m;
}

CUtensorMap make_map_im2col(const __half* base, const Act& in, const ConvGeom& g, int bk) {
  MapKey k{};
  k.v[0] = 3; k.v[1] = (uint64_t)base;
  k.v[2] = ((uint64_t)in.B << 32) | (uint32_t)in.H; k.v[3] = ((uint64_t)in.W << 32) | (uint32_t)in.C;
  k.v[4] = ((uint64_t)g.KH << 32) | (uint32_t)g.KW; k.v[5] = ((uint64_t)g.stride << 32) | (uint32_t)g.pad;
  k.v[6] = ((uint64_t)g.dil << 32) | (uint32_t)bk;
  return cached_map(k, [&] { return make_map_im2col_raw(base, in, g, bk); });
}

}  // namespace

// 2-D fp16 tensor map with a chosen swizzle span (32 / 64 / 128 bytes); shared with stem_sm90.cu
static CUtensorMap make_map_2d_any_raw(const __half* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer,
                            int swizzle_bytes) {
  CUtensorMap m;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {inner * sizeof(__half)};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = driver_api().tiled(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides,
                                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SMK_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed, code " + std::to_string((int)r));
  return m;
}

CUtensorMap make_map_2d_any(const __half* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer,
                            int swizzle_bytes) {
  MapKey k{};
  k.v[0] = 5; k.v[1] = (uint64_t)base; k.v[2] = inner; k.v[3] = outer; k.v[4] = box_inner; k.v[5] = box_outer;
  k.v[6] = (uint64_t)swizzle_bytes;
  return cached_map(k, [&] { return make_map_2d_any_raw(base, inner, outer, box_inner, box_outer, swizzle_bytes); });
}

// N-dimensional tiled-mode fp16 tensor map (rank 2..5), operand-load flavour (L2 promotion 256 B); shared with
// conv3x3_patch_sm90.cu
static CUtensorMap make_map_tiled_nd_raw(const __half* base, int rank, const uint64_t* dims,
                                         const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  SMK_CHECK(rank >= 2 && rank <= 5, "tensor map rank");
  CUtensorMap m;
  cuuint64_t d[5], sb[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) sb[i] = strides_bytes[i];
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = driver_api().tiled(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<__half*>(base), d, sb,
                                  bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SMK_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (nd) failed, code " + std::to_string((int)r));
  return m;
}

CUtensorMap make_map_tiled_nd(const __half* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                              const uint32_t* box, int swizzle_bytes) {
  SMK_CHECK(rank >= 2 && rank <= 5, "tensor map rank");
  MapKey k{};
  k.v[0] = 4 | ((uint64_t)rank << 8) | ((uint64_t)swizzle_bytes << 16);
  k.v[1] = (uint64_t)base;
  for (int i = 0; i < rank; ++i) k.v[2 + i] = dims[i] | ((uint64_t)box[i] << 40);
  for (int i = 0; i + 1 < rank; ++i) k.v[7 + i] = strides_bytes[i];
  return cached_map(k, [&] { return make_map_tiled_nd_raw(base, rank, dims, strides_bytes, box, swizzle_bytes); });
}

bool gemm_conv_supported(const ConvGeom& g) { return g.Cin % CIN_GRAIN == 0 && g.Cout >= 1; }

int gemm_cout_pad(int cout) {
  if (cout <= 16) return 16;
  if (cout <= 32) return 32;
  if (cout <= 64) return 64;
  if (cout <= 128) return 128;
  return (cout + 255) / 256 * 256;
}

// 2-D fp32 tensor map for the epilogue's TMA stores of NHWC fp32 outputs
static CUtensorMap make_map_2d_f32(const float* base, uint64_t inner, uint64_t outer, uint32_t box_inner,
                                   uint32_t box_outer, int swizzle_bytes) {
  MapKey k{};
  k.v[0] = 6; k.v[1] = (uint64_t)base; k.v[2] = inner; k.v[3] = outer; k.v[4] = box_inner; k.v[5] = box_outer;
  k.v[6] = (uint64_t)swizzle_bytes;
  return cached_map(k, [&] {
    CUtensorMap m;
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {inner * sizeof(float)};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
    CUresult r = driver_api().tiled(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides,
                                    box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SMK_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (f32) failed, code " + std::to_string((int)r));
    return m;
  });
}

// The k-block width depends on the tile configuration (Cfg::BLOCK_K), so the operand maps and k-block counts are
// built here, per instantiation.
template <int BLOCK_N, int NSPLIT>
static void launch_cfg(GemmParams& p, const GemmInput* convs, const __half* w_hi, const __half* w_lo, int cout_pad,
                       int w_ld, int num_sms, cudaStream_t st) {
  using C = Cfg<BLOCK_N, NSPLIT>;
  constexpr int bk = C::BLOCK_K;
  for (int i = 0; i < p.nseg; ++i) {
    const ConvGeom& g = convs[i].g;
    const Act& in = convs[i].in;
    GemmSegment& sg = p.seg[i];
    sg.cblks = g.Cin / bk;
    sg.num_kb = g.KH * g.KW * sg.cblks;
    for (int s = 0; s < NSPLIT; ++s) {
      const __half* a = s == 0 ? in.hi : in.lo;
      sg.tmA[s] = sg.mode == 0 ? make_map_2d(a, g.Cin, (uint64_t)in.M(), bk, BLOCK_M) : make_map_im2col(a, in, g, bk);
    }
    if (NSPLIT == 1) sg.tmA[1] = sg.tmA[0];
  }
  if (p.nseg == 1) p.seg[1] = p.seg[0];
  for (int s = 0; s < NSPLIT; ++s) p.tmB[s] = make_map_2d(s == 0 ? w_hi : w_lo, (uint64_t)w_ld, cout_pad, bk, BLOCK_N);
  if (NSPLIT == 1) p.tmB[1] = p.tmB[0];

  auto kern = conv_gemm_kernel<BLOCK_N, NSPLIT>;
  static unsigned long long attr_done = 0;
  ensure_dynamic_smem(kern, C::SMEM_BYTES, attr_done);
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = tiles < num_sms ? tiles : num_sms;     // one CTA per SM
  kern<<<grid, NUM_THREADS, C::SMEM_BYTES, st>>>(p);
  SMK_CUDA(cudaGetLastError());
}

void launch_gemm_conv(const Act& in, const ConvGeom& g, const __half* w_hi, const __half* w_lo, int cout_pad,
                      const Epilogue& ep, int nsplit, int num_sms, cudaStream_t st) {
  GemmInput gi{in, g, 0};
  launch_gemm_multi(&gi, 1, nullptr, w_hi, w_lo, cout_pad, g.KH * g.KW * g.Cin, ep, nsplit, num_sms, st);
}

void launch_gemm_multi(const GemmInput* convs, int nconv, const Act* residual, const __half* w_hi,
                       const __half* w_lo, int cout_pad, int w_ld, const Epilogue& ep, int nsplit, int num_sms,
                       cudaStream_t st, bool reverse_m) {
  SMK_CHECK(nconv >= 1 && nconv <= 2, "1 or 2 convolution segments");
  const ConvGeom& g0 = convs[0].g;
  const Act& in0 = convs[0].in;
  const int Ho = g0.out_h(in0.H), Wo = g0.out_w(in0.W);
  GemmParams p;
  std::memset(&p, 0, sizeof p);
  p.M = in0.B * Ho * Wo;
  p.Cout = g0.Cout;
  p.Ho = Ho;
  p.Wo = Wo;
  // Tile: 128 x min(Cout_pad, 128).  The accumulators live in registers (exact mode: two of them, 2 x 64 fp32 per
  // consumer thread at N = 128), which caps the N tile at 128 columns.
  const int block_n = cout_pad < 128 ? cout_pad : 128;
  SMK_CHECK(cout_pad % block_n == 0, "cout_pad must be a multiple of the N tile");
  if (ep.out_mode != OUT_NCHW_F32) SMK_CHECK(g0.Cout == cout_pad, "NHWC outputs need Cout to match the padded tile width");
  p.n_tiles = cout_pad / block_n;
  p.m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  p.reverse_m = reverse_m ? 1 : 0;
  p.nseg = nconv;
  for (int i = 0; i < nconv; ++i) {
    const ConvGeom& g = convs[i].g;
    const Act& in = convs[i].in;
    SMK_CHECK(gemm_conv_supported(g), "Cin must be a multiple of 64 for the tensor-core conv");
    SMK_CHECK(in.C == g.Cin && g.Cout == g0.Cout && in.B == in0.B, "segment channels/batch mismatch");
    SMK_CHECK(g.out_h(in.H) == Ho && g.out_w(in.W) == Wo, "segments must produce the same output size");
    SMK_CHECK(nsplit == 1 || (in.lo != nullptr && w_lo != nullptr), "exact mode needs lo planes");
    GemmSegment& sg = p.seg[i];
    sg.KW = g.KW;
    sg.stride = g.stride;
    sg.pad = g.pad;
    sg.dil = g.dil;
    sg.mode = (g.KH == 1 && g.KW == 1 && g.stride == 1 && g.pad == 0) ? 0 : 1;
    sg.b_col0 = convs[i].w_col0;
    SMK_CHECK(sg.b_col0 % 64 == 0 && sg.b_col0 + g.KH * g.KW * g.Cin <= w_ld, "weight column range");
  }
  // epilogue TMA boxes: 64 rows of min(block_n, 64) fp16 / min(block_n, 32) fp32 columns, swizzle span = box row
  const uint32_t hbox = block_n < 64 ? block_n : 64, fbox = block_n < 32 ? block_n : 32;
  auto aligned = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (ep.out_mode == OUT_NHWC_SPLIT) {
    SMK_CHECK(aligned(ep.out_hi) && (ep.out_lo == nullptr || aligned(ep.out_lo)), "NHWC output planes 16-byte aligned");
    for (int s = 0; s < (ep.out_lo != nullptr ? 2 : 1); ++s)
      p.tmO[s] = make_map_2d_any(s == 0 ? ep.out_hi : ep.out_lo, (uint64_t)p.Cout, (uint64_t)p.M, hbox, 64, hbox * 2);
  } else if (ep.out_mode == OUT_NHWC_F32) {
    SMK_CHECK(aligned(ep.out_f32), "NHWC fp32 output 16-byte aligned");
    p.tmO[0] = make_map_2d_f32(ep.out_f32, (uint64_t)p.Cout, (uint64_t)p.M, fbox, 64, fbox * 4);
  }
  if (residual != nullptr) {
    SMK_CHECK(ep.out_mode == OUT_NHWC_SPLIT, "a residual needs an NHWC split-plane output");
    SMK_CHECK(residual->C == g0.Cout && residual->M() == p.M, "residual shape");
    SMK_CHECK(nsplit == 1 || residual->lo != nullptr, "exact mode residual needs both planes");
    SMK_CHECK(aligned(residual->hi) && (nsplit == 1 || aligned(residual->lo)), "residual planes 16-byte aligned");
    p.has_res = 1;
    for (int s = 0; s < nsplit; ++s)
      p.tmR[s] = make_map_2d_any(s == 0 ? residual->hi : residual->lo, (uint64_t)p.Cout, (uint64_t)p.M, hbox, 64,
                                 hbox * 2);
  }
  p.ep = ep;

#define SMK_DISPATCH(BN)                                                                         \
  case BN:                                                                                       \
    if (nsplit == 2) launch_cfg<BN, 2>(p, convs, w_hi, w_lo, cout_pad, w_ld, num_sms, st);       \
    else launch_cfg<BN, 1>(p, convs, w_hi, w_lo, cout_pad, w_ld, num_sms, st);                   \
    break;
  switch (block_n) {
    SMK_DISPATCH(16)
    SMK_DISPATCH(32)
    SMK_DISPATCH(64)
    SMK_DISPATCH(128)
    default: SMK_CHECK(false, "unsupported N tile");
  }
#undef SMK_DISPATCH
}

}  // namespace smk
