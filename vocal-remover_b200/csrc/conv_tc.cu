// wgmma / TMA implicit-GEMM convolution for sm_90a with fused folded-BN bias + activation.
//
// Replaces the reference's Conv2DBNActiv (lib/layers.py:8-26) for the dense 3x3 / 1x1 / strided / dilated
// layers that carry 99.8 % of the FLOPs (SURVEY App. B).  GEMM view per CTA tile:
//     D[128 pixels][BN couts] += A[128 pixels][K] * B[BN][K]^T ,   K = taps * CinPad
//   * A is never materialised: for every (tap, 64/32/16-channel chunk) ONE TMA tiled load fetches the
//     shifted (dilated / strided, zero-filled out of bounds = conv padding) pixel box of the NHWC
//     split-bf16 activation, both planes (hi, lo) in one instruction, straight into the 128B/64B/32B
//     swizzled K-major layout wgmma consumes.
//   * B (BN-folded weights, split into bf16 hi/lo once at load time) arrives by TMA the same way.
//   * Two consumer warpgroups (pixels [0,64) and [64,128) of the tile) issue wgmma.mma_async m64nBNk16
//     (bf16 x bf16 -> fp32 in registers).  Three passes per k-step, hi*hi + lo*hi + hi*lo, give a ~2^-16
//     relative product error - the precision the 1e-3 mask gate needs (single-pass bf16/fp16 measurably
//     fails it, DESIGN.md).
//   * The paired variants (PAIR_M / PAIR_N, DESIGN 5.3) run four consumer warpgroups that share one operand box
//     per stage: two m-tiles share the weights, or both N tiles of a layer share the activations.
//   * Warp-specialised persistent kernel: the warp after the consumers is the TMA producer; the consumer
//     warpgroups release a stage as soon as the wgmma group that read it has completed, then run the epilogue
//     (bias -> ReLU/LeakyReLU -> split to bf16 hi/lo -> 16-byte stores of 8 channels where the layout allows -> slice of the destination NHWC buffer, which is how concats are written in
//     place) from registers while the producer already fills the ring for the next tile.
#include <cuda.h>
#include <stdio.h>

#include <map>
#include <tuple>

#include "engine.h"
#include "tc_common.cuh"
#include "tc_plan.h"

namespace vr {

static constexpr int kMaxStages = 8;
// two consumer warpgroups, or four in the paired variants (PAIR_M / PAIR_N), + the TMA producer warp
__host__ __device__ constexpr int consumer_warps(int mode) { return mode == PAIR_NONE ? 8 : 16; }
__host__ __device__ constexpr int tc_threads(int mode) { return 32 * consumer_warps(mode) + 32; }
// channels of K per pipeline stage: 32 in the paired variants, so that at BN = 128 a stage is 48 KB and four fit
__host__ __device__ constexpr int stage_k(int mode) { return mode == PAIR_NONE ? 64 : 32; }
// 16-byte stores where a warpgroup has registers to spare for the transpose (without them, the BN >= 80 paired
// variants spill)
__host__ __device__ constexpr bool generic_vec16(int mode, int bn) { return mode == PAIR_NONE || bn <= 64; }
static constexpr int kStaticSmem = 2048;   // shared memory not given to the dynamic part: barriers and staged bias

struct TcParams {
  int N, Ho, Wo, Wt, Ht, Nt, tiles_w, tiles_h, m_tiles, n_tiles;
  int stride, pad_h, pad_w, dil_h, dil_w, KW;
  int cchunks, total_sub, CinPadTC, Cout, act, stages;
  bf16* out_hi;
  bf16* out_lo;
  int64_t osn, osh;
  int osw;
  const float* bias;
  int vec16;   // 16-byte stores of 8 channels (tc_vec16)
};

// ------------------------------------------------------------------------------------------------
// KB: channels per operand sub-tile (64 / 32 / 16 = SWIZZLE_128B / 64B / 32B); a pipeline stage holds stage_k / KB
// sub-tiles.  BN: output channels per tile (the wgmma N), a multiple of 16 up to 128.
// MODE (TcPair): PAIR_NONE, a CTA unit is one 128-pixel x BN tile for two consumer warpgroups.  PAIR_M, a unit is the
// m-tiles 2q and 2q + 1 of one N tile for four warpgroups (0-1 and 2-3), which share each B box.  PAIR_N, a unit is one
// m-tile with both N tiles of a two-tile layer (warpgroups 0-1 and 2-3), which share each A box.  Every warpgroup
// owns one 64-pixel x BN accumulator block and receives its products in the same order in all three.
template <int KB, int BN, int MODE>
__global__ void __launch_bounds__(tc_threads(MODE), 1)
    conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcParams p) {
  constexpr int kConsumerWarps = consumer_warps(MODE);
  constexpr int SUBS = stage_k(MODE) / KB;
  constexpr int NA = MODE == PAIR_M ? 2 : 1;     // A boxes per sub-tile (m-tiles of a unit)
  constexpr int NB = MODE == PAIR_N ? 2 : 1;     // B boxes per sub-tile (N tiles of a unit)
  constexpr int kSteps = KB / 16;
  constexpr uint32_t kAPlane = 128 * KB * 2;     // one plane of an A sub-tile (128 pixels x KB channels)
  constexpr uint32_t kASub = 2 * kAPlane;        // hi + lo
  constexpr uint32_t kBPlane = BN * KB * 2;
  constexpr uint32_t kBSub = 2 * kBPlane;
  constexpr uint32_t kStageBytes = SUBS * (NA * kASub + NB * kBSub);
  constexpr uint32_t kBRegion = SUBS * NA * kASub;   // B sub-tiles follow the A sub-tiles inside a stage
  constexpr uint32_t kLayout = KB == 64 ? 1u : KB == 32 ? 2u : 3u;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[kMaxStages];
  __shared__ __align__(8) uint64_t bar_empty[kMaxStages];
  __shared__ float bias_s[256];   // folded-BN bias of every N tile, staged once (a global load per use stalled the epilogue)

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);   // provably warp-uniform: keeps wgmma unserialised
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  // units: m groups of NA m-tiles (the last one short when m_tiles is odd) x N groups of NB N tiles
  const int n_units = p.n_tiles / NB;
  const int total_units = (p.m_tiles + NA - 1) / NA * n_units;
  const int num_iters = (p.total_sub + SUBS - 1) / SUBS;

  if (warp == kConsumerWarps && lane == 0) {
    tma_prefetch(&tmA);
    tma_prefetch(&tmB);
    MbarRing(smem_u32(&bar_full[0]), smem_u32(&bar_empty[0]), 0, p.stages).init(1, kConsumerWarps);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < p.n_tiles * BN; i += blockDim.x) bias_s[i] = __ldg(p.bias + i);
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===================== TMA producer (one elected lane runs the whole loop nest) =====================
    if (elect_one_sync()) {
      MbarRing ring(smem_u32(&bar_full[0]), smem_u32(&bar_empty[0]), 0, p.stages);
      for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
        const int nt0 = unit % n_units * NB;
        const int mt0 = unit / n_units * NA;
        // the m-tiles of the unit that exist: a PAIR_M unit past the last m-tile loads (and its warpgroups store) nothing
        const int na = min(NA, p.m_tiles - mt0);
        int wbase[NA], hbase[NA], n0[NA];
#pragma unroll
        for (int a = 0; a < NA; ++a) {
          const int mt = mt0 + a;
          wbase[a] = (mt % p.tiles_w) * p.Wt * p.stride - p.pad_w;
          hbase[a] = ((mt / p.tiles_w) % p.tiles_h) * p.Ht * p.stride - p.pad_h;
          n0[a] = (mt / (p.tiles_w * p.tiles_h)) * p.Nt;
        }
        int cc = 0, kw = 0, kh = 0, sub = 0;   // (tap, channel chunk) of the next sub-tile, advanced without divisions
        for (int it = 0; it < num_iters; ++it) {
          ring.wait_empty();
          const int nsub = min(SUBS, p.total_sub - sub);
          const uint32_t full = ring.full();
          const uint32_t sbase = smem_base + (uint32_t)ring.slot * kStageBytes;
          mbar_expect_tx(full, (uint32_t)nsub * ((uint32_t)na * kASub + NB * kBSub));
#pragma unroll
          for (int j = 0; j < SUBS; ++j) {
            if (j < nsub) {
#pragma unroll
              for (int a = 0; a < NA; ++a)
                if (a < na)
                  tma_load_5d(sbase + (uint32_t)(j * NA + a) * kASub, &tmA, cc * KB, wbase[a] + kw * p.dil_w,
                              hbase[a] + kh * p.dil_h, n0[a], 0, full);
#pragma unroll
              for (int b = 0; b < NB; ++b)
                tma_load_3d(sbase + kBRegion + (uint32_t)(j * NB + b) * kBSub, &tmB,
                            (kh * p.KW + kw) * p.CinPadTC + cc * KB, (nt0 + b) * BN, 0, full);
              ++sub;
              if (++cc == p.cchunks) {
                cc = 0;
                if (++kw == p.KW) {
                  kw = 0;
                  ++kh;
                }
              }
            }
          }
          ring.advance();
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumer warpgroups: wgmma into registers, then the epilogue =====================
    const int half = (warp >> 2) & 1;   // pixels [64 half, 64 half + 64) of its m-tile
    const int pair = warp >> 3;         // which m-tile (PAIR_M) or N tile (PAIR_N) of the unit
    const int a_sel = MODE == PAIR_M ? pair : 0, b_sel = MODE == PAIR_N ? pair : 0;
    const float slope = act_slope(p.act);
    const uint32_t dhi = desc_hi(8 * KB * 2, kLayout);
    MbarRing ring(smem_u32(&bar_full[0]), smem_u32(&bar_empty[0]), 0, p.stages);
    float acc[BN / 2];
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
      const int nt = unit % n_units * NB + b_sel;
      const int mt = unit / n_units * NA + a_sel;
      if (mt >= p.m_tiles) {
        // the missing second m-tile of a PAIR_M unit: release every stage unread, store nothing
        for (int it = 0; it < num_iters; ++it) {
          ring.wait_full();
          warp_arrive(ring.empty(), lane);
          ring.advance();
        }
        continue;
      }
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      HeldSlot held;
      for (int it = 0; it < num_iters; ++it) {
        const int nsub = min(SUBS, p.total_sub - it * SUBS);
        ring.wait_full();
        const uint32_t sdesc = desc_lo(smem_base + (uint32_t)ring.slot * kStageBytes);
        wg_fence();
#pragma unroll
        for (int j = 0; j < SUBS; ++j) {
          if (j < nsub) {
            const uint32_t a_hi = sdesc + (((j * NA + a_sel) * kASub + (uint32_t)half * (kAPlane / 2)) >> 4);
            const uint32_t a_lo = a_hi + (kAPlane >> 4);
            const uint32_t b_hi = sdesc + ((kBRegion + (j * NB + b_sel) * kBSub) >> 4);
            const uint32_t b_lo = b_hi + (kBPlane >> 4);
#pragma unroll
            for (int k = 0; k < kSteps; ++k)
              wgmma_split3<BN>(acc, a_hi + 2u * k, a_lo + 2u * k, b_hi + 2u * k, b_lo + 2u * k, dhi);
          }
        }
        wg_commit();
        wg_wait<1>();   // the group of the previous stage has read its operands: hand that slot back
        held.release(ring, lane);
        held.hold(ring);
        ring.advance();
      }
      wg_wait<0>();
      held.release_last(ring, lane);

      const int w0 = (mt % p.tiles_w) * p.Wt;
      const int h0 = ((mt / p.tiles_w) % p.tiles_h) * p.Ht;
      const int n0 = (mt / (p.tiles_w * p.tiles_h)) * p.Nt;
      // 16-byte stores where the variant allows them (generic_vec16); rows past the batch store nothing
      constexpr bool kVec16 = generic_vec16(MODE, BN);
      EpiDest d{p.out_hi, p.out_lo, {0, 0}, {false, false}, nt * BN, p.Cout, kVec16 && p.vec16};
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int row = 64 * half + 16 * (warp & 3) + (lane >> 2) + 8 * hr;
        const int dw = row % p.Wt;
        const int dh = (row / p.Wt) % p.Ht;
        const int n = n0 + row / (p.Wt * p.Ht);
        d.obase[hr] = (int64_t)n * p.osn + (int64_t)(h0 + dh) * p.osh + (int64_t)(w0 + dw) * p.osw;
        d.keep[hr] = n < p.N;
      }
      epilogue_store<BN>(acc, bias_s, slope, lane, d);
    }
  }
}

// every (KB, BN, MODE) instantiation the host can launch.  The paired variants take KB = min(KB, 32) (pair_KB), and
// PAIR_N the BN of two N tiles (129 to 256 output channels) at KB = 32.
#define VR_TC_FOR_BN(X, KB, M) \
  X(KB, 16, M) X(KB, 32, M) X(KB, 48, M) X(KB, 64, M) X(KB, 80, M) X(KB, 96, M) X(KB, 112, M) X(KB, 128, M)
#define VR_TC_FOR_ALL(X)                                                                                   \
  VR_TC_FOR_BN(X, 64, PAIR_NONE) VR_TC_FOR_BN(X, 32, PAIR_NONE) VR_TC_FOR_BN(X, 16, PAIR_NONE)             \
  VR_TC_FOR_BN(X, 32, PAIR_M) VR_TC_FOR_BN(X, 16, PAIR_M)                                                  \
  X(32, 80, PAIR_N) X(32, 96, PAIR_N) X(32, 112, PAIR_N) X(32, 128, PAIR_N)


// ------------------------------------------------------------------------------------------------
// host side
TcDebug g_debug;
TcLastConv g_last_conv;

static constexpr int kMaxDevices = 64;
const TcDevice& tc_device() {
  static TcDevice table[kMaxDevices];
  static TcDevice none;
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return none;
  TcDevice& d = table[dev];
  if (!d.ok) {
    if (cudaDeviceGetAttribute(&d.max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&d.num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      return none;
#define VR_TC_SET_SMEM(KB, BN, M) \
  cudaFuncSetAttribute(conv_tc_kernel<KB, BN, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, d.max_smem - kStaticSmem);
    VR_TC_FOR_ALL(VR_TC_SET_SMEM)
#undef VR_TC_SET_SMEM
    tc_rows_set_attributes(d.max_smem);
    tc_halo_set_attributes(d.max_smem);
    d.ok = true;
  }
  return d;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tc_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

static CUtensorMapSwizzle swizzle_for(int KB) {
  return KB == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : KB == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
}

static uint16_t tc_f2bf(float f) {   // round-to-nearest-even, same as __float2bfloat16_rn for finite values
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  uint32_t r = 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)((u + r) >> 16);
}
static float tc_bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

struct TileGeom {
  int Wt, Ht, Nt;
  bool ok;
};
static TileGeom tile_geom(int Ho, int Wo) {
  TileGeom g{0, 0, 0, false};
  if (Wo <= 0 || Ho <= 0) return g;
  if (Wo >= 128) {
    if (Wo % 128) return g;
    g.Wt = 128; g.Ht = 1; g.Nt = 1;
  } else {
    if (128 % Wo) return g;
    g.Wt = Wo;
    g.Ht = 128 / Wo < Ho ? 128 / Wo : Ho;
    if (Ho % g.Ht) return g;
    if ((128 / Wo) % g.Ht) return g;
    g.Nt = 128 / (g.Wt * g.Ht);
  }
  g.ok = true;
  return g;
}

// output-channel tiles of the row kernel (rows) or of the generic and halo kernels
struct NTiling {
  int BN, n_tiles;
};
static NTiling n_tiling(const ConvLayer& L, bool rows, bool rows_wide) {
  const int cout16 = round_up(L.Cout, 16);
  if (rows) {
    // 64 output channels per tile for the decoder layers with a fused upsample: one N = 64 MMA per product and output
    // row instead of two N = 32 ones (half the A-operand reads from shared memory) and every input row is interpolated
    // once instead of once per N tile.  Plain TMA layers stay at 32: the 64-wide tile has a single accumulator set (no
    // epilogue overlap) and only four operand slots next to its 147 KB of weights, and measured slower there.
    const int BN = cout16 == 16 ? 16 : (rows_wide && cout16 % 64 == 0 ? 64 : 32);
    return {BN, ceil_div(cout16, BN)};
  }
  const int n_tiles = ceil_div(cout16, 128);
  return {round_up(ceil_div(cout16, n_tiles), 16), n_tiles};
}

// The kernel of a layer whose output maps are H x W: the row kernel where it applies, else the halo kernel, else the
// generic one.  All three kernels stage the bias of every N tile in 256 floats of shared memory, so a layer with more
// output channels than that stays on the CUDA-core kernel.
TcKind tc_choose(const ConvLayer& L, int H, int W, bool rows_wide) {
  if (!(L.k == 1 || L.k == 3) || !(L.stride == 1 || L.stride == 2) || L.Cout < 4) return TC_NONE;
  const TileGeom g = tile_geom(H, W);
  if (!g.ok || g.Wt * L.stride > 256 || g.Ht * L.stride > 256) return TC_NONE;
  const bool k3s1 = L.k == 3 && L.stride == 1 && L.dil_h == 1 && L.dil_w == 1;
  const NTiling r = n_tiling(L, true, rows_wide), t = n_tiling(L, false, false);
  // whole 128-pixel row tiles of 2, 4 or 8 rows (rows_per_tile, conv_tc_rows.cu)
  if (k3s1 && W % 128 == 0 && H % 8 == 0 && tc_rows_has(r.BN) && r.n_tiles * r.BN <= 256) return TC_ROWS;
  // whole tiles of 128 / W rows (MB = 1)
  if (k3s1 && (W == 16 || W == 32 || W == 64) && H % (128 / W) == 0 && tc_halo_has(t.BN) &&
      t.n_tiles * t.BN <= 256 && g_debug.halo != 1)
    return TC_HALO;
  if (t.n_tiles * t.BN > 256) return TC_NONE;
  return TC_GENERIC;
}

// The folded fp32 weights w [tap][L.CinPad][L.CoutPad] split into bf16 hi / lo planes of rows x K; at(co, tap, ci) =
// row * K + k of one weight.
template <class At>
static std::vector<uint16_t> split_bf16(const ConvLayer& L, const float* wp, int rows, int K, At at) {
  std::vector<uint16_t> planes((size_t)2 * rows * K, 0);
  const size_t lo = (size_t)rows * K;
  for (int co = 0; co < L.Cout; ++co)
    for (int t = 0; t < L.k * L.k; ++t)
      for (int ci = 0; ci < L.CinPad; ++ci) {
        const float w = wp[((size_t)t * L.CinPad + ci) * L.CoutPad + co];
        const uint16_t hi = tc_f2bf(w);
        const size_t i = at(co, t, ci);
        planes[i] = hi;
        planes[lo + i] = tc_f2bf(w - tc_bf2f(hi));
      }
  return planes;
}

// which 8-channel input groups carry any weight at all (the lstm / pad groups of the concat layouts do not)
static unsigned long long weight_group_mask(const ConvLayer& L, const float* wp, int CinPad) {
  if (CinPad / 8 > 64) return ~0ull;
  unsigned long long m = 0x3ull;   // k-step 0 of chunk 0 initialises the accumulators: never skipped
  for (int ci = 0; ci < L.CinPad; ++ci) {
    bool any = false;
    for (int t = 0; t < L.k * L.k && !any; ++t)
      for (int co = 0; co < L.Cout && !any; ++co) any = wp[((size_t)t * L.CinPad + ci) * L.CoutPad + co] != 0.f;
    if (any) m |= 1ull << (ci / 8);
  }
  return m;
}

// TMA map of the packed weights [2][rows][K]: boxes of kb channels x box_rows rows, both planes
static bool encode_weight_map(const TcConv& tc, CUtensorMap* map, int kb, int rows, int K, int box_rows,
                              std::string& err, const std::string& name) {
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, 2};
  cuuint64_t strides[2] = {(cuuint64_t)K * 2, (cuuint64_t)rows * K * 2};
  cuuint32_t box[3] = {(cuuint32_t)kb, (cuuint32_t)box_rows, 2};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = tc_encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, tc.w_planes.get(), dims, strides, box, es,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(kb), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    err = "cuTensorMapEncodeTiled(weights) failed for " + name + " code " + std::to_string((int)r);
    return false;
  }
  return true;
}

const CUtensorMap* tc_activation_map(TcConv& tc, const ActView& v, int bw, int bh, int bn, int es, std::string& err,
                                     const std::string& name, int kb) {
  if (kb == 0) kb = tc.KB;
  const ViewKey key = std::make_tuple((const void*)v.hi, (const void*)v.lo, v.N, v.H, v.W, v.C, bw, bh, bn, kb);
  auto it = tc.map_a.find(key);
  if (it != tc.map_a.end()) return &it->second;
  // TMA reads 16-byte aligned rows; the lo plane is the box's outermost dimension
  const int64_t plane = (const char*)v.lo - (const char*)v.hi;
  if (v.sw % 8 || v.sh % 8 || v.sn % 8 || (reinterpret_cast<uintptr_t>(v.hi) & 15) || plane <= 0 || plane % 16) {
    err = "internal: the input of " + name + " is not 16-byte aligned or its lo plane does not follow its hi plane";
    return nullptr;
  }
  cuuint64_t dims[5] = {(cuuint64_t)v.C, (cuuint64_t)v.W, (cuuint64_t)v.H, (cuuint64_t)v.N, 2};
  cuuint64_t strides[4] = {(cuuint64_t)v.sw * 2, (cuuint64_t)v.sh * 2, (cuuint64_t)v.sn * 2, (cuuint64_t)plane};
  cuuint32_t box[5] = {(cuuint32_t)kb, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn, 2};
  cuuint32_t estr[5] = {1, (cuuint32_t)es, (cuuint32_t)es, 1, 1};
  CUtensorMap m;
  CUresult r = tc_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)v.hi, dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(kb), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    err = "cuTensorMapEncodeTiled(activations) failed for " + name + " code " + std::to_string((int)r);
    return nullptr;
  }
  return &tc.map_a.emplace(key, m).first->second;
}

bool tc_prepare(ConvLayer& L, const float* w, const float* b, int H, int W, bool rows_wide, std::string& err) {
  const TcKind kind = tc_choose(L, H, W, rows_wide);
  if (kind == TC_NONE) return true;   // stays on the CUDA-core kernel
  if (!tc_encode_fn()) {
    err = "cuTensorMapEncodeTiled is not available from the driver";
    return false;
  }
  auto tc = std::make_shared<TcConv>();
  tc->kind = kind;
  tc->H = H; tc->W = W;
  const NTiling nt = n_tiling(L, kind == TC_ROWS, rows_wide);
  const int BN = nt.BN, cin16 = round_up(L.CinPad, 16);
  tc->BN = BN; tc->n_tiles = nt.n_tiles;
  tc->KB = kind != TC_GENERIC ? 32 : cin16 % 64 == 0 ? 64 : cin16 % 32 == 0 ? 32 : 16;
  const int CinPad = round_up(L.CinPad, tc->KB);
  tc->CinPad = CinPad;
  tc->chunks = CinPad / tc->KB;
  tc->kmask = weight_group_mask(L, w, CinPad);
  const int rows = nt.n_tiles * BN;
  std::vector<uint16_t> planes;
  int brows, K;
  if (kind == TC_ROWS) {
    // B[plane][nt*3*BN + (2-kh)*BN + co][kw*CinPad + ci]: the three kh taps stacked along the MMA N dimension
    brows = 3 * rows;
    K = 3 * CinPad;
    planes = split_bf16(L, w, brows, K, [&](int co, int t, int ci) {
      return (size_t)(co / BN * 3 * BN + (2 - t / 3) * BN + co % BN) * K + (size_t)(t % 3) * CinPad + ci;
    });
  } else {
    // B[plane][co][tap*CinPad + ci]: every tap padded to whole chunks, so no chunk reads another tap's weights
    brows = rows;
    K = L.k * L.k * CinPad;
    planes = split_bf16(L, w, brows, K, [&](int co, int t, int ci) { return (size_t)co * K + (size_t)t * CinPad + ci; });
  }
  std::vector<float> bias((size_t)rows, 0.f);
  for (int co = 0; co < L.Cout; ++co) bias[(size_t)co] = b[co];
  if (tc->w_planes.alloc(planes.size() * 2) != cudaSuccess || tc->bias.alloc(bias.size() * 4) != cudaSuccess) {
    err = "cudaMalloc failed while packing tensor-core weights for " + L.name;
    return false;
  }
  if (!upload(tc->w_planes.get(), planes.data(), planes.size() * 2, err) ||
      !upload(tc->bias.get(), bias.data(), bias.size() * 4, err) ||
      !encode_weight_map(*tc, &tc->map_b, tc->KB, brows, K, kind == TC_ROWS ? 3 * BN : BN, err, L.name))
    return false;
  if (kind == TC_GENERIC) {
    // the paired variants stage 32 channels of K: a KB = 64 layer runs them in 32-channel boxes.  The k-steps, and so
    // every accumulator's sum order, are the same in either box width.
    tc->pair_KB = tc->KB < 32 ? tc->KB : 32;
    tc->pair = tc->n_tiles == 2 && tc->pair_KB == 32 ? PAIR_N : PAIR_M;
    if (!encode_weight_map(*tc, &tc->map_b_pair, tc->pair_KB, brows, K, BN, err, L.name)) return false;
  }
  L.tc = tc;
  return true;
}

// The pairing of one generic-kernel launch.  Only layers with at most 32 channels per chunk and per N tile pair
// automatically: on an H100 at 700 W (profiles/generic_conv.py, DESIGN 5.3) those ran 10-30 % faster paired, while the
// wider layers ran from 6 % faster to 24 % slower, the KB = 64 ones (moved to 32-channel boxes) slowest.  A paired unit does the work of two tiles and takes about 1.9x as long
// as one (the halo kernel's 256-pixel tiles measured the same), so pair only where that does not lose to the last wave
// of the persistent grid: 1.9 x the paired waves <= the unpaired waves.  vr_debug_set(8, 1 / 2 / 3) pins none /
// PAIR_M / PAIR_N where the layer allows it.
bool tc_vec16(const ActView& out) {
  return g_debug.pair_stores != 1 &&
         ((reinterpret_cast<uintptr_t>(out.hi) | reinterpret_cast<uintptr_t>(out.lo)) & 15) == 0 && out.sn % 8 == 0 &&
         out.sh % 8 == 0 && out.sw % 8 == 0;
}

static TcPair launch_pairing(const TcConv& tc, int m_tiles, int num_sms) {
  if (g_debug.pair == 1) return PAIR_NONE;
  if (g_debug.pair == 2) return PAIR_M;
  if (g_debug.pair == 3) return tc.pair == PAIR_N ? PAIR_N : PAIR_NONE;
  if (tc.KB > 32 || tc.BN > 32) return PAIR_NONE;
  const int units = tc.pair == PAIR_N ? m_tiles : ceil_div(m_tiles, 2) * tc.n_tiles;
  const int waves1 = ceil_div(m_tiles * tc.n_tiles, num_sms), waves2 = ceil_div(units, num_sms);
  return 19 * waves2 <= 10 * waves1 ? tc.pair : PAIR_NONE;
}

cudaError_t tc_launch(const ConvLayer& L, const ActView& in, const ActView& out, cudaStream_t s, std::string& err,
                      const ConvFusion& f) {
  TcConv& tc = *L.tc;
  if (out.H != tc.H || out.W != tc.W || (in.H - 1) / L.stride + 1 != out.H || (in.W - 1) / L.stride + 1 != out.W) {
    err = "internal: " + L.name + " is launched on maps of another size than it was prepared for";
    return cudaErrorInvalidValue;
  }
  if (tc.kind == TC_ROWS) return tc_rows_launch(L, tc, in, out, s, err, f);
  if (!f.empty()) {
    err = "tc_launch: fused work is only implemented in the row-streaming kernel";
    return cudaErrorInvalidValue;
  }
  if (tc.kind == TC_HALO) return tc_halo_launch(L, tc, in, out, s, err);
  const TcDevice& dv = tc_device();
  if (!dv.ok) {
    err = "tc_launch: cannot query the current device";
    return cudaErrorInvalidValue;
  }
  const TileGeom g = tile_geom(out.H, out.W);
  TcParams p;
  p.N = out.N; p.Ho = out.H; p.Wo = out.W;
  p.Wt = g.Wt; p.Ht = g.Ht; p.Nt = g.Nt;
  p.tiles_w = out.W / g.Wt; p.tiles_h = out.H / g.Ht;
  p.m_tiles = p.tiles_w * p.tiles_h * ceil_div(out.N, g.Nt);
  p.n_tiles = tc.n_tiles;
  p.stride = L.stride; p.dil_h = L.dil_h; p.dil_w = L.dil_w;
  p.pad_h = L.dil_h * (L.k / 2); p.pad_w = L.dil_w * (L.k / 2);
  p.KW = L.k;
  p.CinPadTC = tc.CinPad; p.Cout = L.Cout; p.act = L.act;
  const TcPair mode = launch_pairing(tc, p.m_tiles, dv.num_sms);
  const int KB = mode == PAIR_NONE ? tc.KB : tc.pair_KB;
  p.cchunks = tc.CinPad / KB; p.total_sub = L.k * L.k * p.cchunks;
  const CUtensorMap* map_a = tc_activation_map(tc, in, g.Wt * L.stride, g.Ht * L.stride, g.Nt, L.stride, err, L.name, KB);
  if (!map_a) return cudaErrorInvalidValue;
  const CUtensorMap& map_b = mode == PAIR_NONE ? tc.map_b : tc.map_b_pair;
  const int na = mode == PAIR_M ? 2 : 1, nb = mode == PAIR_N ? 2 : 1;
  const int stage_bytes = stage_k(mode) / KB * (na * 2 * 128 * KB * 2 + nb * 2 * tc.BN * KB * 2);
  const int dyn = dv.max_smem - kStaticSmem;
  p.stages = (dyn - 1024) / stage_bytes;
  if (p.stages > kMaxStages) p.stages = kMaxStages;
  if (p.stages < 2) {
    err = "tc_launch: shared memory too small for two pipeline stages";
    return cudaErrorInvalidValue;
  }
  p.out_hi = out.hi; p.out_lo = out.lo;
  p.osn = out.sn; p.osh = out.sh; p.osw = out.sw;
  p.vec16 = tc_vec16(out);
  p.bias = tc.bias.get();
  const int total_units = ceil_div(p.m_tiles, na) * (p.n_tiles / nb);
  const int grid = total_units < dv.num_sms ? total_units : dv.num_sms;
  const TcLastConv launched{TC_GENERIC, KB, tc.BN, tc.n_tiles, mode, 0, 0, generic_vec16(mode, tc.BN) && p.vec16};
#define VR_TC_LAUNCH(KB_, BN_, M_)                                                          \
  if (KB == KB_ && tc.BN == BN_ && mode == M_) {                                            \
    g_last_conv = launched;                                                                 \
    conv_tc_kernel<KB_, BN_, M_><<<grid, tc_threads(M_), dyn, s>>>(*map_a, map_b, p);       \
    return cudaGetLastError();                                                              \
  }
  VR_TC_FOR_ALL(VR_TC_LAUNCH)
#undef VR_TC_LAUNCH
  err = "tc_launch: no kernel instantiation for this channel tile";
  return cudaErrorInvalidValue;
}

}  // namespace vr
