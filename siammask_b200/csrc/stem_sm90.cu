// Stem of the backbone on the tensor cores: conv 7x7 stride 2 pad 0, 3 -> 64 channels, + BN + ReLU
// (experiments/siammask_sharp/resnet.py:154,218-220), reading the raw NCHW fp32 pixels the tracker loop hands
// over (tools/test.py:61-64) and writing p0 as NHWC split-fp16 planes.
//
// Cin = 3 is useless to TMA (6-byte pixels), so the A operand is BUILT: eight producer warps gather each output
// pixel's 7x7x3 window straight from global memory (L1/L2 resident: neighbouring windows overlap 5/7), split it
// into fp16 hi/lo and write it into the 128B-swizzled K-major tile layout wgmma expects
// (K = 147 padded to 192 = three 64-wide k-blocks, a 4-deep ring).  The 64 x 192 weight matrix stays resident in
// shared memory for the whole persistent CTA.  Two consumer warpgroups (64 tile rows each) run the wgmma k-loop of
// conv_gemm_sm90.cu with N = 64 and write BN + ReLU results from their accumulator registers.
//
// Warps (512 threads): 0..7 = A producers (two threads per tile row; lane 0 of warp 0 also loads the weights),
// 8..15 = consumers.
#include "common.cuh"
#include "ptx.cuh"

namespace smk {

namespace {

constexpr int BM = 128, BN = 64, BK = 64, UK = 16;
constexpr int KBLOCKS = 3;                 // K = 7*7*3 = 147 -> 192
constexpr int KREAL = 147;
constexpr int STAGES = 4;
constexpr int A_TILE = BM * BK * 2;        // 16 KB
constexpr int B_TILE = BN * BK * 2;        // 8 KB
constexpr int NPROD = 256;                 // two producer threads per tile row (each builds half of every k-block:
                                           // the gather is a per-thread latency chain of 147 loads + conversions)
constexpr int NCONS_WARPS = 8;
constexpr int NTHREADS = NPROD + 32 * NCONS_WARPS;

struct StemParams {
  CUtensorMap tmB[2];     // weights [64][192] fp16 K-major, box 64 x 64, hi / lo
  __half* out_hi;         // p0 planes [M][64]
  __half* out_lo;
  const float* x;         // [B][3][S][S]
  const float* alpha;     // [64] 2^-e
  const float* beta;      // [64]
  int* ovf;               // overflow flag (values outside fp16's range), may be null
  int B, S, So, M, m_tiles;
};

template <int NSPLIT>
struct SCfg {
  static constexpr int STAGE_BYTES = NSPLIT * A_TILE;
  static constexpr int B_BYTES = KBLOCKS * NSPLIT * B_TILE;
  static constexpr int SMEM = B_BYTES + STAGES * STAGE_BYTES + 1024 + 256;
  static_assert(SMEM <= 227 * 1024, "smem budget");
};

// one 64-wide k-block of this thread's row: k = (r*7 + s)*3 + c
// JH = which half of the k-block (4 of its 8 16-byte chunks) this thread builds; compile-time so that k -> (r, s, c)
// folds into constant offsets
template <int KB, int NSPLIT, int JH>
__device__ __forceinline__ void build_kblock(const float* __restrict__ base, bool valid, int S, uint8_t* stage,
                                             int row) {
  uint8_t* rowp = stage + (row >> 3) * 1024 + (row & 7) * 128;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    constexpr int J0 = JH * 4;
    const int j = J0 + jj;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = KB * 64 + j * 8 + e;
      if (k < KREAL) {
        const int c = k % 3, rs = k / 3, r = rs / 7, s = rs % 7;
        v[e] = valid ? __ldg(base + ((size_t)c * S + r) * S + s) : 0.f;
      } else {
        v[e] = 0.f;
      }
    }
    uint4 h, l;
    __half2* hh = reinterpret_cast<__half2*>(&h);
    __half2* ll = reinterpret_cast<__half2*>(&l);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const __half2 hv = __floats2half2_rn(v[2 * t], v[2 * t + 1]);
      hh[t] = hv;
      const float2 hf = __half22float2(hv);
      ll[t] = __floats2half2_rn(v[2 * t] - hf.x, v[2 * t + 1] - hf.y);
    }
    const int off = (j ^ (row & 7)) << 4;       // SWIZZLE_128B: 16B chunk index ^= row & 7
    *reinterpret_cast<uint4*>(rowp + off) = h;
    if constexpr (NSPLIT == 2) *reinterpret_cast<uint4*>(rowp + A_TILE + off) = l;
  }
}

template <int NSPLIT>
__global__ void __launch_bounds__(NTHREADS, 1) stem_tc_kernel(const __grid_constant__ StemParams p) {
  using C = SCfg<NSPLIT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* b_smem = smem;                                  // [kb][plane][64 x 128B]
  uint8_t* a_smem = b_smem + C::B_BYTES;                   // ring of [plane][128 x 128B]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(a_smem + STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* b_bar = empty_bar + STAGES;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < NSPLIT; ++i) tma_prefetch_desc(&p.tmB[i]);
    // one arrival per WARP (after its lanes' fences): single-thread arrivals would serialise on the barrier word
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], NPROD / 32); mbar_init(&empty_bar[s], NCONS_WARPS); }
    mbar_init(b_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < NPROD / 32) {
    if (warp == 0) {
      // resident weights: 3 k-blocks x NSPLIT planes
      if (elect_one()) {
        mbar_arrive_expect_tx(b_bar, C::B_BYTES);
        for (int kb = 0; kb < KBLOCKS; ++kb)
          for (int s = 0; s < NSPLIT; ++s)
            tma_load_2d(b_smem + (kb * NSPLIT + s) * B_TILE, &p.tmB[s], b_bar, kb * BK, 0);
      }
      __syncwarp();
    }
    // ===================== A producers: one output pixel (tile row) per thread =====================
    const int row = threadIdx.x & (BM - 1);
    const bool upper = threadIdx.x >= BM;               // warp-uniform: warps 0-3 build chunks 0-3, warps 4-7 chunks 4-7
    int stage = 0;
    uint32_t phase = 0;
    const int So2 = p.So * p.So;
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x) {
      const int m = tile * BM + row;
      const bool valid = m < p.M;
      const int b = m / So2;
      const int rem = m - b * So2;
      const int y = rem / p.So;
      const int xo = rem - y * p.So;
      const float* base = p.x + ((size_t)b * 3 * p.S + 2 * y) * p.S + 2 * xo;
#define SMK_STEM_KB(KB)                                                          \
  mbar_wait(&empty_bar[stage], phase ^ 1);                                       \
  if (upper) build_kblock<KB, NSPLIT, 1>(base, valid, p.S, a_smem + stage * C::STAGE_BYTES, row); \
  else build_kblock<KB, NSPLIT, 0>(base, valid, p.S, a_smem + stage * C::STAGE_BYTES, row); \
  fence_proxy_async();                                                           \
  __syncwarp();                                                                  \
  if (lane == 0) mbar_arrive(&full_bar[stage]);                                  \
  if (++stage == STAGES) { stage = 0; phase ^= 1; }
      SMK_STEM_KB(0)
      SMK_STEM_KB(1)
      SMK_STEM_KB(2)
#undef SMK_STEM_KB
    }
    return;
  }

  // ===================== consumers: wgmma over the three k-blocks, then +beta, ReLU, split, store =====================
  const int wg = (warp - NPROD / 32) >> 2;
  const int wl = warp & 3;
  float acc[BN / 2], acc2[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  mbar_wait(b_bar, 0);
  for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[i] = 0.f; acc2[i] = 0.f; }
#pragma unroll 1
    for (int kb = 0; kb < KBLOCKS; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_hi = smem_u32(a_smem + stage * C::STAGE_BYTES) + wg * (64 * BK * 2);
      const uint32_t b_hi = smem_u32(b_smem + kb * NSPLIT * B_TILE);
      const uint64_t da_hi0 = wgmma_desc_kmajor<128>(a_hi), db_hi0 = wgmma_desc_kmajor<128>(b_hi);
      const uint64_t da_lo0 = wgmma_desc_kmajor<128>(a_hi + A_TILE), db_lo0 = wgmma_desc_kmajor<128>(b_hi + B_TILE);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / UK; ++k) {
        const uint64_t kadd = static_cast<uint64_t>(k * UK * 2 / 16);     // 32 B per K step in the address field
        wgmma_f16<BN>(acc, da_hi0 + kadd, db_hi0 + kadd);
        if constexpr (NSPLIT == 2) {
          wgmma_f16<BN>(acc2, da_lo0 + kadd, db_hi0 + kadd);
          wgmma_f16<BN>(acc2, da_hi0 + kadd, db_lo0 + kadd);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    fence_regs(acc);
    if constexpr (NSPLIT == 2) fence_regs(acc2);
    // thread holds rows row0, row0 + 8 and column pairs 8j + 2(lane % 4) (see wgmma_f16)
    const int row0 = tile * BM + wg * 64 + wl * 16 + (lane >> 2);
    float amax = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = row0 + 8 * h;
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = 8 * j + 2 * (lane & 3);
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if constexpr (NSPLIT == 2) {
          v0 += acc2[4 * j + 2 * h];
          v1 += acc2[4 * j + 2 * h + 1];
        }
        const float2 al = __ldg(reinterpret_cast<const float2*>(p.alpha + n));
        const float2 be = __ldg(reinterpret_cast<const float2*>(p.beta + n));
        v0 = fmaxf(fmaf(v0, al.x, be.x), 0.f);
        v1 = fmaxf(fmaf(v1, al.y, be.y), 0.f);
        amax = fmaxf(amax, fmaxf(v0, v1));
        const __half2 hv = __floats2half2_rn(v0, v1);
        const float2 hf = __half22float2(hv);
        const size_t off = static_cast<size_t>(m) * BN + n;
        *reinterpret_cast<__half2*>(p.out_hi + off) = hv;
        if constexpr (NSPLIT == 2) *reinterpret_cast<__half2*>(p.out_lo + off) = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
      }
    }
    flag_if_out_of_range(amax, p.ovf);
  }
}

}  // namespace

CUtensorMap make_map_2d_any(const __half* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer,
                            int swizzle_bytes);

void launch_stem_tc(const float* x, int B, int S, const __half* w_hi, const __half* w_lo, const float* alpha,
                    const float* beta, Act out, int num_sms, cudaStream_t st, int* ovf) {
  const int So = (S - 7) / 2 + 1;
  SMK_CHECK(out.H == So && out.W == So && out.C == 64 && out.B == B, "stem output shape");
  StemParams p;
  p.ovf = ovf;
  p.x = x;
  p.alpha = alpha;
  p.beta = beta;
  p.B = B;
  p.S = S;
  p.So = So;
  p.M = B * So * So;
  p.m_tiles = (p.M + BM - 1) / BM;
  const int nsplit = out.lo != nullptr ? 2 : 1;
  for (int s = 0; s < nsplit; ++s) {
    p.tmB[s] = make_map_2d_any(s == 0 ? w_hi : w_lo, KBLOCKS * BK, BN, BK, BN, 128);
  }
  if (nsplit == 1) p.tmB[1] = p.tmB[0];
  p.out_hi = out.hi;
  p.out_lo = out.lo;
  const int grid = p.m_tiles < num_sms ? p.m_tiles : num_sms;
  if (nsplit == 2) {
    static unsigned long long attr = 0;
    ensure_dynamic_smem(stem_tc_kernel<2>, SCfg<2>::SMEM, attr);
    stem_tc_kernel<2><<<grid, NTHREADS, SCfg<2>::SMEM, st>>>(p);
  } else {
    static unsigned long long attr = 0;
    ensure_dynamic_smem(stem_tc_kernel<1>, SCfg<1>::SMEM, attr);
    stem_tc_kernel<1><<<grid, NTHREADS, SCfg<1>::SMEM, st>>>(p);
  }
  SMK_CUDA(cudaGetLastError());
}

}  // namespace smk
