// Halo-tile wgmma convolution: 3x3, stride 1, dilation 1, output width 16, 32 or 64.
//
// The generic kernel (conv_tc.cu) fetches one shifted 128-pixel box per (tap, channel chunk), so every activation
// crosses L2->SM nine times per N tile.  Here a CTA tile is Ht x W output pixels (Ht * W = 128 * MB) x BN output
// channels, and for every 32-channel chunk the TMA warp loads ONE two-plane box of (Ht + 2) x Wb pixels: the tile with
// its +-1 halo, zero-filled outside the image (= the conv padding).  Wb = W + 2 rounded up to 8 pixels keeps each
// plane a whole number of 512-byte SWIZZLE_64B periods, so the lo plane of the box starts on a period as well.
//   * The nine taps are the SAME shared-memory tile: for tap (kh, kw) each consumer warp gathers the A fragments of its
//     16 pixels (one image row, since 16 | W) with ldmatrix.x4 at halo pixels (h + kh, w + kw).  ldmatrix takes one row
//     address per lane, so shifted rows, rows of the next image row and the padding need no data movement.
//   * The wgmma take A from those registers (hi*hi + lo*hi + hi*lo, as everywhere) and B (BN x 32 channels of one tap,
//     hi + lo) from a ring of per-tap weight stages that the TMA warp streams next to the halo slots.
//   * Each of the two consumer warpgroups owns MB m64 blocks of the tile.  The weights of a chunk (9 taps x BN x 32
//     channels, hi + lo) are read once per tile, so they outweigh the halo box at MB = 1 (BN = 128: 144 KB against
//     36 KB per 128 pixels); MB = 2 halves them per pixel, at twice the accumulators (setmaxnreg, below).
// L2->SM traffic per output pixel: (Ht + 2) * Wb / (Ht * W) activation fetches instead of 9.
#include <stdio.h>

#include "engine.h"
#include "tc_common.cuh"
#include "tc_plan.h"

namespace vr {

static constexpr int kConsumerWarps = 8;   // two warpgroups
static constexpr int kProducerWarps = 4;   // the TMA warp and three idle warps: one warpgroup, so that it can give
                                           // its registers to the consumers (setmaxnreg acts on whole warpgroups)
static constexpr int kThreads = 32 * (kConsumerWarps + kProducerWarps);
// MB = 2 at BN = 128 holds 128 accumulator and 2 x 16 fragment registers per thread, more than the 168 a 12-warp block
// launches with (65536 / 384, rounded down to a multiple of 8): at 168 ptxas spills and serialises its wgmma (C7512).
// setmaxnreg moves registers from the producer warpgroup to the consumers.  setmaxnreg.inc waits until the block's
// pool, which holds what the block was launched with, can grant the request: the budgets must add up to no more.
static constexpr int kLaunchRegs = 168;
static constexpr int kConsumerRegs = 232;
static constexpr int kProducerRegs = 40;
static_assert(kConsumerWarps * kConsumerRegs + kProducerWarps * kProducerRegs <=
                  (kConsumerWarps + kProducerWarps) * kLaunchRegs,
              "setmaxnreg.inc would wait forever for registers the block does not own");
static constexpr int kStaticSmem = 2048;   // shared memory not given to the dynamic part: barriers and staged bias
static constexpr int kMaxHSlots = 4;
static constexpr int kMaxWStages = 18;      // two chunks of nine taps
static constexpr uint32_t kKB = 32;         // channels per chunk (SWIZZLE_64B rows of 64 bytes)
static constexpr uint32_t kRowB = kKB * 2;  // bytes of one pixel of a chunk

template <int BN>
struct HaloGeom {
  static constexpr uint32_t kBPlane = BN * kRowB;    // hi -> lo plane of one tap's weights
  static constexpr uint32_t kWStage = 2 * kBPlane;   // one tap of one chunk, both planes
};

struct HaloParams {
  int N, H, W, lw, Ht, Wb, tiles_h, n_tiles, total_tiles;
  int chunks, CinPadH, Cout, act;
  int n_hslots, n_wstages;
  uint32_t hplane, hslot;   // bytes of one plane / both planes of a halo box
  unsigned long long kmask;   // bit g: some weight on input channels [8g, 8g+8) is non-zero (all ones = no skipping)
  bf16* out_hi;
  bf16* out_lo;
  int64_t osn, osh;
  int osw;
  int vec16;   // 16-byte stores of 8 channels (tc_vec16)
  const float* bias;
};

// The consumers' positions in the halo ring and the weight ring, and the weight stage still held
struct HaloConsumer {
  MbarRing h, w;
  HeldSlot held_w;
};

// One channel chunk.  Each (tap, k-step) is one commit group: the warp loads the 16 x 16 hi and lo fragments of its MB
// pixel blocks with ldmatrix, then issues the group's wgmma from registers.  The fragments of two consecutive groups
// live in the two halves of fr (k-step 0 / 1), and a group's fragments are overwritten only after `wait_group 1` has
// retired it.  The halo slot is free once the last group's ldmatrix have returned, a weight stage once the last group
// that read it has completed.  Every accumulator receives its products in the order chunk, kh, kw, k-step, hi*hi,
// lo*hi, hi*lo.  Unlike the row kernel, the k-steps of a chunk are not skipped one by one: with that branch ptxas
// serialises the wgmma of the BN = 128 tile (C7512) and spills at BN = 96.  Chunks without weights are skipped whole.
// q0[b]: halo pixel of this lane's ldmatrix row (tap 0, 0) in block b.
template <int BN, int MB>
__device__ __forceinline__ void consume_halo(HaloConsumer& st, const HaloParams& p, float* acc,
                                             uint32_t (&fr)[2][MB * 8], const uint32_t* q0, uint32_t h_base,
                                             uint32_t w_base, uint32_t dhi, int lane) {
  typedef HaloGeom<BN> G;
  st.h.wait_full();
  const uint32_t slot = h_base + (uint32_t)st.h.slot * p.hslot;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int kh = t / 3, kw = t % 3;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      uint32_t* f = fr[ks];
#pragma unroll
      for (int b = 0; b < MB; ++b) {
        const uint32_t q = q0[b] + (uint32_t)(kh * p.Wb + kw);
        // SWIZZLE_64B: 16-byte chunk j of 64-byte row q sits at chunk j ^ ((q >> 1) & 3) (planes are 512-byte aligned)
        const uint32_t a = slot + (q << 6) + ((((uint32_t)(2 * ks) + ((uint32_t)lane >> 4)) ^ ((q >> 1) & 3u)) << 4);
        ldsm_x4(f + 8 * b, a);
        ldsm_x4(f + 8 * b + 4, a + p.hplane);
      }
      if (ks == 0) st.w.wait_full();
      const uint32_t b_hi = desc_lo(w_base + (uint32_t)st.w.slot * G::kWStage) + (uint32_t)(ks * 32 >> 4);
      wg_fence();
#pragma unroll
      for (int b = 0; b < MB; ++b)
        wgmma_split3_rs<BN>(acc + b * (BN / 2), f + 8 * b, f + 8 * b + 4, b_hi, b_hi + (G::kBPlane >> 4), dhi);
      wg_commit();
      if (t == 8 && ks == 1) warp_arrive(st.h.empty(), lane);
      wg_wait<1>();   // every group but this one is complete: its fragments and the weights it read can be reused
      st.held_w.release(st.w, lane);
    }
    st.held_w.hold(st.w);   // released after the next group, once this tap's k-step 1 group has completed
    st.w.advance();
  }
  st.h.advance();
}

template <int BN, int MB>
__global__ void __launch_bounds__(kThreads, 1)
    conv_tc_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                        const HaloParams p) {
  typedef HaloGeom<BN> G;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_hfull[kMaxHSlots];
  __shared__ __align__(8) uint64_t bar_hempty[kMaxHSlots];
  __shared__ __align__(8) uint64_t bar_wfull[kMaxWStages];
  __shared__ __align__(8) uint64_t bar_wempty[kMaxWStages];
  __shared__ float bias_s[256];   // folded-BN bias of every N tile, staged once

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);   // provably warp-uniform: keeps wgmma unserialised
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t h_base = smem_base;
  const uint32_t w_base = smem_base + (uint32_t)p.n_hslots * p.hslot;
  MbarRing hring(smem_u32(&bar_hfull[0]), smem_u32(&bar_hempty[0]), 0, p.n_hslots);
  MbarRing wring(smem_u32(&bar_wfull[0]), smem_u32(&bar_wempty[0]), 0, p.n_wstages);

  if (warp == kConsumerWarps && lane == 0) {
    tma_prefetch(&tmA);
    tma_prefetch(&tmB);
    hring.init(1, kConsumerWarps);
    wring.init(1, kConsumerWarps);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < p.n_tiles * BN; i += blockDim.x) bias_s[i] = __ldg(p.bias + i);
  __syncthreads();

  // Consumers and producers split first: all four producer warps execute the one setmaxnreg.dec, as setmaxnreg requires
  // of every thread of a warpgroup, and ptxas allocates the consumer code for kConsumerRegs.
  if (warp >= kConsumerWarps) {
    setmaxnreg_dec<kProducerRegs>();
    // ===================== TMA producer: one elected lane of warp 8 runs the whole loop nest =====================
    if (warp == kConsumerWarps && elect_one_sync()) {
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int nt = tile % p.n_tiles;
        const int mt = tile / p.n_tiles;
        const int h0 = (mt % p.tiles_h) * p.Ht;
        const int n = mt / p.tiles_h;
        for (int cc = 0; cc < p.chunks; ++cc) {
          if (!chunk_groups(p.kmask, cc)) continue;   // no weights on this chunk: the consumers skip it too
          hring.wait_empty();
          mbar_expect_tx(hring.full(), p.hslot);
          tma_load_5d(h_base + (uint32_t)hring.slot * p.hslot, &tmA, cc * (int)kKB, -1, h0 - 1, n, 0, hring.full());
          hring.advance();
          for (int t = 0; t < 9; ++t) {
            wring.wait_empty();
            mbar_expect_tx(wring.full(), G::kWStage);
            tma_load_3d(w_base + (uint32_t)wring.slot * G::kWStage, &tmB, t * p.CinPadH + cc * (int)kKB, nt * BN, 0,
                        wring.full());
            wring.advance();
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumer warpgroups: wgmma into registers, then the epilogue =====================
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2;   // m64 blocks [MB wg, MB wg + MB) of the tile
    const float slope = act_slope(p.act);
    const uint32_t dhi = desc_hi(8 * kRowB, 2u);   // SWIZZLE_64B, 8-row groups of 64-byte rows
    uint32_t q0[MB];
#pragma unroll
    for (int b = 0; b < MB; ++b) {
      const int px = 64 * (MB * wg + b) + 16 * (warp & 3) + (lane & 15);
      q0[b] = (uint32_t)((px >> p.lw) * p.Wb + (px & (p.W - 1)));
    }
    HaloConsumer st{hring, wring};
    float acc[MB * BN / 2];
    uint32_t fr[2][MB * 8];
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
#pragma unroll
      for (int i = 0; i < MB * BN / 2; ++i) acc[i] = 0.f;
      for (int cc = 0; cc < p.chunks; ++cc) {
        // a chunk whose weights are all zero is not issued: exact, since the products would be 0
        if (!chunk_groups(p.kmask, cc)) continue;
        consume_halo<BN, MB>(st, p, acc, fr, q0, h_base, w_base, dhi, lane);
      }
      wg_wait<0>();
      st.held_w.release_last(st.w, lane);

      const int nt = tile % p.n_tiles;
      const int mt = tile / p.n_tiles;
      const int h0 = (mt % p.tiles_h) * p.Ht;
      const int n = mt / p.tiles_h;
      // 16-byte stores except at MB = 2, BN = 128, whose 128 accumulators leave too few registers for the transposes
      // (they spill, DESIGN 5.7): that variant stores each pixel with 8-byte stores
      constexpr bool kVec16 = !(MB == 2 && BN == 128);
#pragma unroll
      for (int b = 0; b < MB; ++b) {
        EpiDest d{p.out_hi, p.out_lo, {0, 0}, {true, true}, nt * BN, p.Cout, p.vec16 != 0};
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int px = 64 * (MB * wg + b) + 16 * (warp & 3) + (lane >> 2) + 8 * hr;
          d.obase[hr] = (int64_t)n * p.osn + (int64_t)(h0 + (px >> p.lw)) * p.osh + (int64_t)(px & (p.W - 1)) * p.osw;
          if constexpr (!kVec16)
            epilogue_pixel8<BN>(acc + b * (BN / 2) + 2 * hr, bias_s, nt * BN, p.Cout, slope, lane,
                                p.out_hi + d.obase[hr], p.out_lo + d.obase[hr], d.vec16);
        }
        if constexpr (kVec16) epilogue_store<BN>(acc + b * (BN / 2), bias_s, slope, lane, d);
      }
    }
  }
}

// every (BN, MB) instantiation the host can launch, and so the BN values tc_choose accepts for these layers
#define VR_HALO_FOR_MB(X, BN) X(BN, 1) X(BN, 2)
#define VR_HALO_FOR_ALL(X) \
  VR_HALO_FOR_MB(X, 16) VR_HALO_FOR_MB(X, 32) VR_HALO_FOR_MB(X, 48) VR_HALO_FOR_MB(X, 64) VR_HALO_FOR_MB(X, 96) \
  VR_HALO_FOR_MB(X, 128)

bool tc_halo_has(int BN) {
#define VR_HALO_HAS(BN_, MB_) if (BN == BN_) return true;
  VR_HALO_FOR_ALL(VR_HALO_HAS)
#undef VR_HALO_HAS
  return false;
}

// ------------------------------------------------------------------------------------------------
cudaError_t tc_halo_launch(const ConvLayer& L, TcConv& tc, const ActView& in, const ActView& out, cudaStream_t s,
                           std::string& err) {
  const TcDevice& dv = tc_device();
  if (!dv.ok) {
    err = "tc_halo_launch: cannot query the current device";
    return cudaErrorInvalidValue;
  }
  // MB = 2 halves the weight traffic per pixel but also the number of tiles, so the last wave of the persistent grid
  // weighs twice as much.  A 256-pixel tile takes about 1.9x a 128-pixel one (H100, per-layer times of both): MB = 2
  // where 1.9 x its waves are no more than MB = 1's (vr_debug_set(3, 2 / 3) pins MB = 1 / 2).
  const int ht1 = 128 / out.W;
  const bool mb2_tiles = out.H % (2 * ht1) == 0;
  const int tiles1 = out.N * (out.H / ht1) * tc.n_tiles;
  const int waves1 = ceil_div(tiles1, dv.num_sms), waves2 = ceil_div(tiles1 / 2, dv.num_sms);
  int MB = mb2_tiles && 19 * waves2 <= 10 * waves1 ? 2 : 1;
  if (g_debug.halo == 2) MB = 1;
  if (g_debug.halo == 3 && mb2_tiles) MB = 2;
  HaloParams p;
  p.N = out.N; p.H = out.H; p.W = out.W;
  p.lw = out.W == 16 ? 4 : out.W == 32 ? 5 : 6;
  p.Ht = MB * ht1;
  p.Wb = round_up(out.W + 2, 8);
  p.tiles_h = out.H / p.Ht;
  p.n_tiles = tc.n_tiles;
  p.total_tiles = out.N * p.tiles_h * p.n_tiles;
  p.chunks = tc.chunks; p.CinPadH = tc.CinPad; p.Cout = L.Cout; p.act = L.act;
  p.hplane = (uint32_t)((p.Ht + 2) * p.Wb) * kRowB;
  p.hslot = 2 * p.hplane;
  p.kmask = g_debug.kskip == 1 ? tc.kmask : ~0ull;
  p.out_hi = out.hi; p.out_lo = out.lo;
  p.osn = out.sn; p.osh = out.sh; p.osw = out.sw;
  p.vec16 = tc_vec16(out);
  p.bias = tc.bias.get();
  // the halo tile, both planes
  const CUtensorMap* map_a = tc_activation_map(tc, in, p.Wb, p.Ht + 2, 1, 1, err, L.name);
  if (!map_a) return cudaErrorInvalidValue;
  // shared memory: up to kMaxHSlots halo slots next to one chunk's nine weight stages, the rest to weight stages
  const int w_stage = tc.BN * 2 * (int)kRowB;
  const int dyn = dv.max_smem - kStaticSmem;
  const int avail = dyn - 1024;
  p.n_hslots = (avail - 9 * w_stage) / (int)p.hslot;
  if (p.n_hslots > kMaxHSlots) p.n_hslots = kMaxHSlots;
  if (p.n_hslots < 2) p.n_hslots = 2;
  p.n_wstages = (avail - p.n_hslots * (int)p.hslot) / w_stage;
  if (p.n_wstages > kMaxWStages) p.n_wstages = kMaxWStages;
  if (p.n_wstages < 2) {
    err = "tc_halo_launch: shared memory too small for two halo slots and two weight stages";
    return cudaErrorInvalidValue;
  }
  const int grid = p.total_tiles < dv.num_sms ? p.total_tiles : dv.num_sms;   // persistent: one CTA per SM
  const TcLastConv launched{TC_HALO, (int)kKB, tc.BN, tc.n_tiles, PAIR_NONE, MB, 0, p.vec16};
#define VR_HALO_LAUNCH(BN_, MB_)                                                        \
  if (tc.BN == BN_ && MB == MB_) {                                                      \
    g_last_conv = launched;                                                             \
    conv_tc_halo_kernel<BN_, MB_><<<grid, kThreads, dyn, s>>>(*map_a, tc.map_b, p);     \
    return cudaGetLastError();                                                          \
  }
  VR_HALO_FOR_ALL(VR_HALO_LAUNCH)
#undef VR_HALO_LAUNCH
  err = "tc_halo_launch: no kernel instantiation for this channel tile";
  return cudaErrorInvalidValue;
}


// cudaFuncSetAttribute is per device: called by tc_device() the first time a device is used (conv_tc.cu)
void tc_halo_set_attributes(int max_smem) {
#define VR_HALO_SET(BN_, MB_) \
  cudaFuncSetAttribute(conv_tc_halo_kernel<BN_, MB_>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - kStaticSmem);
  VR_HALO_FOR_ALL(VR_HALO_SET)
#undef VR_HALO_SET
}

}  // namespace vr
