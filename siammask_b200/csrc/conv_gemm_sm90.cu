// Implicit-GEMM convolution on the Hopper tensor cores (wgmma) for sm_90a.
//
//   out[m][n] = epilogue( sum_k A[m][k] * W[n][k] ),  m = (b, ho, wo) flattened, k = (r, s, c) with c fastest.
//
// * A (NHWC fp16 activation planes) is staged by TMA: plain 2-D tiles for 1x1/stride-1 convs, im2col-mode
//   tiles (cp.async.bulk.tensor.4d...im2col) for everything else — padding, stride and dilation are resolved
//   by the TMA unit, out-of-image taps arrive as zeros, and the 128-pixel M tile runs across row and image
//   boundaries so batch absorbs the odd spatial sizes (31x31, 29x29, 25x25 ...).
// * W (K-major fp16, [Cout_pad][KH*KW*Cin]) is staged by 2-D TMA tiles.  Both land in 128B-swizzled smem, in a ring
//   of k-block stages guarded by full / empty mbarriers, and are consumed by wgmma.mma_async (M=64 per warpgroup,
//   N=BLOCK_N, K=16) accumulating in fp32 registers.
// * Precision: NSPLIT=1 multiplies the fp16 hi planes only.  NSPLIT=2 ("exact") keeps activations and
//   weights as hi+lo fp16 pairs (22 significant bits) and issues three MMAs per k-step
//   (hi*hi into one accumulator, hi*lo + lo*hi into a second one, summed in the epilogue: the tensor pipe truncates
//   on every accumulate, so the small cross terms must not be fed into the large running sum) — fp32-class results
//   from the fp16 tensor pipe.
// * Epilogue straight from the accumulator registers: acc*alpha[c]+beta[c] (+ residual) (ReLU) -> NHWC split-fp16
//   planes, NHWC fp32, or NCHW fp32 (the boundary layout of the reference's outputs, tools/test.py:205-206).
//
// * K may consist of up to two SEGMENTS that accumulate into the same tile: (conv over input 0) + (conv over
//   input 1) fuses a bottleneck's downsample branch with its conv3, and an IDENTITY segment
//   acc += residual * diag(2^e) streams the residual tensor through the same TMA/MMA pipeline (one extra
//   k-block per 64 output columns) instead of stalling the epilogue on it.
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
constexpr int BLOCK_K = 64;     // k-block width in fp16 elements: 128-byte swizzled rows
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
  static constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_TILE_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = NSPLIT * (A_TILE_BYTES + B_TILE_BYTES);
  static constexpr int RAW_STAGES = (SMEM_LIMIT - 2048) / STAGE_BYTES;
  static constexpr int STAGES = RAW_STAGES > 6 ? 6 : RAW_STAGES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int ACC = BLOCK_N / 2;               // fp32 accumulator registers per thread and accumulator
  static_assert(STAGES >= 2, "pipeline needs at least two stages");
  static_assert(BLOCK_N % 16 == 0 && BLOCK_N >= 16 && BLOCK_N <= 128, "N tile (register accumulators)");
  static_assert(B_TILE_BYTES % 1024 == 0, "stage parts stay 1024-aligned (swizzle atoms)");
  static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory budget");
};

// tile -> M block.  With reverse_m the persistent CTAs walk the M tiles from the end: a layer then starts on the rows
// its producer wrote last, which are the ones still resident in L2.
__device__ __forceinline__ int m_block(const GemmParams& p, int tile) {
  const int mb = tile / p.n_tiles;
  return p.reverse_m ? p.m_tiles - 1 - mb : mb;
}

template <int BLOCK_N, int NSPLIT>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_gemm_kernel(const __grid_constant__ GemmParams p) {
  using C = Cfg<BLOCK_N, NSPLIT>;
  constexpr int STAGES = C::STAGES;
  constexpr int A_TILE_BYTES = C::A_TILE_BYTES;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

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
    auto acquire = [&](uint32_t bytes) {
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (leader) mbar_arrive_expect_tx(&full_bar[stage], bytes);
    };
    auto load_2d = [&](void* dst, const CUtensorMap* map, int c0, int c1) {
      if (leader) tma_load_2d(dst, map, &full_bar[stage], c0, c1);
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = m_block(p, tile) * BLOCK_M;
      const int n0 = (tile % p.n_tiles) * BLOCK_N;
      const int q = m0 % p.Wo;
      const int t = m0 / p.Wo;
      const int pq = t % p.Ho;
      const int nb = t / p.Ho;
      for (int sgi = 0; sgi < p.nseg; ++sgi) {
        const GemmSegment& sg = p.seg[sgi];
        if (sg.kind == 1) {
          // identity segment: A = residual tile [128 rows x 64 cols] (K-major), B = diag(2^e) block (its lo plane is
          // zero; it is loaded anyway so that every k-block runs the same MMA sequence)
#pragma unroll 1
          for (int kb = 0; kb < BLOCK_N / BLOCK_K; ++kb) {
            acquire(C::STAGE_BYTES);
            uint8_t* st = smem + stage * C::STAGE_BYTES;
#pragma unroll
            for (int s = 0; s < NSPLIT; ++s) {
              load_2d(st + s * A_TILE_BYTES, &sg.tmA[s], n0 + kb * BLOCK_K, m0);
              load_2d(st + NSPLIT * A_TILE_BYTES + s * C::B_TILE_BYTES, &p.tmB[s], sg.b_col0 + n0 + kb * BLOCK_K, n0);
            }
            __syncwarp();
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
          continue;
        }
        const int wb = q * sg.stride - sg.pad;
        const int hb = pq * sg.stride - sg.pad;
#pragma unroll 1
        for (int kb = 0; kb < sg.num_kb; ++kb) {
          acquire(C::STAGE_BYTES);
          uint8_t* st = smem + stage * C::STAGE_BYTES;
          const int tap = kb / sg.cblks;
          const int c0 = (kb - tap * sg.cblks) * BLOCK_K;
#pragma unroll
          for (int s = 0; s < NSPLIT; ++s) {
            uint8_t* a_dst = st + s * A_TILE_BYTES;
            if (sg.mode == 0) {
              load_2d(a_dst, &sg.tmA[s], c0, m0);
            } else if (leader) {
              const int r = tap / sg.KW;
              const int sx = tap - r * sg.KW;
              tma_load_im2col_4d(a_dst, &sg.tmA[s], &full_bar[stage], c0, wb, hb, nb,
                                 static_cast<uint16_t>(sx * sg.dil), static_cast<uint16_t>(r * sg.dil));
            }
            load_2d(st + NSPLIT * A_TILE_BYTES + s * C::B_TILE_BYTES, &p.tmB[s], sg.b_col0 + kb * BLOCK_K, n0);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: MMA + epilogue, 64 tile rows per warpgroup =====================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = (warp >> 2) - 1;
  const int wl = warp & 3;
  const Epilogue& ep = p.ep;
  const int HoWo = p.Ho * p.Wo;
  float acc[C::ACC];
  float acc2[C::ACC];     // exact mode: the hi*lo + lo*hi cross terms
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) { acc[i] = 0.f; acc2[i] = 0.f; }
    int prev = -1;
    for (int sgi = 0; sgi < p.nseg; ++sgi) {
      const GemmSegment& sg = p.seg[sgi];
      const bool ident = sg.kind == 1;
      const int nkb = ident ? BLOCK_N / BLOCK_K : sg.num_kb;
#pragma unroll 1
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_hi = smem_u32(smem + stage * C::STAGE_BYTES) + wg * (64 * BLOCK_K * 2);
        const uint32_t b_hi = smem_u32(smem + stage * C::STAGE_BYTES) + NSPLIT * A_TILE_BYTES;
        const uint64_t da_hi0 = wgmma_desc_kmajor<128>(a_hi);
        const uint64_t db_hi0 = wgmma_desc_kmajor<128>(b_hi);
        const uint64_t da_lo0 = wgmma_desc_kmajor<128>(a_hi + A_TILE_BYTES);
        const uint64_t db_lo0 = wgmma_desc_kmajor<128>(b_hi + C::B_TILE_BYTES);
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

    // ---- epilogue: thread holds rows row0, row0 + 8 and column pairs col0 + 8j (see wgmma_f16)
    const int row0 = m_block(p, tile) * BLOCK_M + wg * 64 + wl * 16 + (lane >> 2);
    const int col0 = (tile % p.n_tiles) * BLOCK_N + 2 * (lane & 3);
    float amax = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = row0 + 8 * h;
      if (m >= p.M) continue;
      const int b = m / HoWo;
      const int hw = m - b * HoWo;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int n = col0 + 8 * j;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if constexpr (NSPLIT == 2) {
          v0 += acc2[4 * j + 2 * h];
          v1 += acc2[4 * j + 2 * h + 1];
        }
        const float2 al = __ldg(reinterpret_cast<const float2*>(ep.alpha + n));
        const float2 be = __ldg(reinterpret_cast<const float2*>(ep.beta + n));
        v0 = fmaf(v0, al.x, be.x);
        v1 = fmaf(v1, al.y, be.y);
        const size_t off = static_cast<size_t>(m) * p.Cout + n;
        if (ep.res_hi != nullptr) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(ep.res_hi + off));
          v0 += f.x;
          v1 += f.y;
          if (ep.res_lo != nullptr) {
            const float2 l = __half22float2(*reinterpret_cast<const __half2*>(ep.res_lo + off));
            v0 += l.x;
            v1 += l.y;
          }
        }
        if (ep.relu) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        if (ep.out_mode == OUT_NHWC_SPLIT) {
          amax = fmaxf(amax, fmaxf(fabsf(v0), fabsf(v1)));
          const __half2 hv = __floats2half2_rn(v0, v1);
          const float2 hf = __half22float2(hv);
          *reinterpret_cast<__half2*>(ep.out_hi + off) = hv;
          if (ep.out_lo != nullptr)
            *reinterpret_cast<__half2*>(ep.out_lo + off) = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
        } else if (ep.out_mode == OUT_NHWC_F32) {
          *reinterpret_cast<float2*>(ep.out_f32 + off) = make_float2(v0, v1);
        } else if (n < p.Cout) {  // OUT_NCHW_F32 (write-once output: stream past L2); the last N tile may be ragged
          float* dst = ep.out_f32 + (static_cast<size_t>(b) * p.Cout + n) * HoWo + hw;
          __stcs(dst, v0);
          if (n + 1 < p.Cout) __stcs(dst + HoWo, v1);
        }
      }
    }
    if (ep.out_mode == OUT_NHWC_SPLIT) flag_if_out_of_range(amax, ep.ovf);
  }
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

template <int BLOCK_N, int NSPLIT>
void launch_cfg(const GemmParams& p, int num_sms, cudaStream_t st) {
  using C = Cfg<BLOCK_N, NSPLIT>;
  auto kern = conv_gemm_kernel<BLOCK_N, NSPLIT>;
  static unsigned long long attr_done = 0;
  ensure_dynamic_smem(kern, C::SMEM_BYTES, attr_done);
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = tiles < num_sms ? tiles : num_sms;     // one CTA per SM
  kern<<<grid, NUM_THREADS, C::SMEM_BYTES, st>>>(p);
  SMK_CUDA(cudaGetLastError());
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

void launch_gemm_conv(const Act& in, const ConvGeom& g, const __half* w_hi, const __half* w_lo, int cout_pad,
                      const Epilogue& ep, int nsplit, int num_sms, cudaStream_t st) {
  GemmInput gi{in, g, 0};
  launch_gemm_multi(&gi, 1, nullptr, -1, w_hi, w_lo, cout_pad, g.KH * g.KW * g.Cin, ep, nsplit, num_sms, st);
}

void launch_gemm_multi(const GemmInput* convs, int nconv, const Act* residual, int res_col0, const __half* w_hi,
                       const __half* w_lo, int cout_pad, int w_ld, const Epilogue& ep_in, int nsplit, int num_sms,
                       cudaStream_t st, bool reverse_m) {
  SMK_CHECK(nconv >= 1 && nconv <= 2, "1 or 2 convolution segments");
  SMK_CHECK(nconv + (residual != nullptr ? 1 : 0) <= 2, "at most two K segments");
  Epilogue ep = ep_in;
  const ConvGeom& g0 = convs[0].g;
  const Act& in0 = convs[0].in;
  const int Ho = g0.out_size(in0.H), Wo = g0.out_size(in0.W);
  GemmParams p;
  p.M = in0.B * Ho * Wo;
  p.Cout = g0.Cout;
  p.Ho = Ho;
  p.Wo = Wo;
  // Tile: 128 x min(Cout_pad, 128).  The accumulators live in registers (exact mode: two of them, 2 x 64 fp32 per
  // consumer thread at N = 128), which caps the N tile at 128 columns.
  const int block_n = cout_pad < 128 ? cout_pad : 128;
  const int bk = BLOCK_K;
  SMK_CHECK(cout_pad % block_n == 0, "cout_pad must be a multiple of the N tile");
  if (ep.out_mode != OUT_NCHW_F32) SMK_CHECK(g0.Cout == cout_pad, "NHWC outputs need Cout to match the padded tile width");
  p.n_tiles = cout_pad / block_n;
  p.m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  p.reverse_m = reverse_m ? 1 : 0;
  p.nseg = 0;
  for (int i = 0; i < nconv; ++i) {
    const ConvGeom& g = convs[i].g;
    const Act& in = convs[i].in;
    SMK_CHECK(gemm_conv_supported(g), "Cin must be a multiple of 64 for the tensor-core conv");
    SMK_CHECK(in.C == g.Cin && g.Cout == g0.Cout && in.B == in0.B, "segment channels/batch mismatch");
    SMK_CHECK(g.out_size(in.H) == Ho && g.out_size(in.W) == Wo, "segments must produce the same output size");
    SMK_CHECK(nsplit == 1 || (in.lo != nullptr && w_lo != nullptr), "exact mode needs lo planes");
    GemmSegment& sg = p.seg[p.nseg++];
    sg.kind = 0;
    sg.cblks = g.Cin / bk;
    sg.num_kb = g.KH * g.KW * sg.cblks;
    sg.KW = g.KW;
    sg.stride = g.stride;
    sg.pad = g.pad;
    sg.dil = g.dil;
    sg.mode = (g.KH == 1 && g.KW == 1 && g.stride == 1 && g.pad == 0) ? 0 : 1;
    sg.b_col0 = convs[i].w_col0;
    SMK_CHECK(sg.b_col0 % 64 == 0 && sg.b_col0 + g.KH * g.KW * g.Cin <= w_ld, "weight column range");
    for (int s = 0; s < nsplit; ++s) {
      const __half* a = s == 0 ? in.hi : in.lo;
      sg.tmA[s] = sg.mode == 0 ? make_map_2d(a, g.Cin, (uint64_t)in.M(), bk, BLOCK_M) : make_map_im2col(a, in, g, bk);
    }
    if (nsplit == 1) sg.tmA[1] = sg.tmA[0];
  }
  if (residual != nullptr) {
    // the residual rides the tensor pipe: needs the diag(2^e) block in the weights and 64-wide column blocks
    SMK_CHECK(res_col0 >= 0 && res_col0 % 64 == 0 && res_col0 + g0.Cout <= w_ld && block_n % 64 == 0,
              "identity segment needs a diagonal block in the packed weights");
    SMK_CHECK(residual->C == g0.Cout && residual->M() == p.M, "residual shape");
    SMK_CHECK(nsplit == 1 || residual->lo != nullptr, "exact mode residual needs both planes");
    GemmSegment& sg = p.seg[p.nseg++];
    sg.kind = 1;
    sg.mode = 0;
    sg.num_kb = block_n / bk;
    sg.cblks = sg.KW = sg.stride = sg.dil = 1;
    sg.pad = 0;
    sg.b_col0 = res_col0;
    for (int s = 0; s < nsplit; ++s)
      sg.tmA[s] = make_map_2d(s == 0 ? residual->hi : residual->lo, g0.Cout, (uint64_t)p.M, bk, BLOCK_M);
    if (nsplit == 1) sg.tmA[1] = sg.tmA[0];
    ep.res_hi = ep.res_lo = nullptr;       // accumulated by the MMA, not by the epilogue
  }
  if (p.nseg == 1) p.seg[1] = p.seg[0];
  for (int s = 0; s < nsplit; ++s)
    p.tmB[s] = make_map_2d(s == 0 ? w_hi : w_lo, (uint64_t)w_ld, cout_pad, bk, block_n);
  if (nsplit == 1) p.tmB[1] = p.tmB[0];
  p.ep = ep;

#define SMK_DISPATCH(BN)                                             \
  case BN:                                                           \
    if (nsplit == 2) launch_cfg<BN, 2>(p, num_sms, st);              \
    else launch_cfg<BN, 1>(p, num_sms, st);                          \
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
