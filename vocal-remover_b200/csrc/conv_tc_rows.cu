// Row-streaming wgmma convolution: 3x3, stride 1, dilation 1, output width a multiple of 128.
//
// The generic kernel (conv_tc.cu) re-fetches every input pixel from L2 once per tap (9x) and is bound
// by L2->SM bandwidth on the wide, shallow layers (enc1, enc2.conv2, dec2, dec1 of every BaseNet).
// Here one CTA owns a block of R output rows x 128 pixels x BN couts with R accumulators resident in
// registers, and streams the R+2 input rows it needs through shared memory ONCE per 32-channel chunk:
//   * each input row (130 pixels incl. the +-1 halo, 32 channels, hi and lo plane) is one TMA load of
//     a two-plane box; out-of-image rows / columns are zero-filled by TMA = the conv padding;
//   * a row feeds up to three output rows (kh = 0,1,2) and, for each, the three kw taps are the SAME
//     shared-memory tile read with ldmatrix at rows shifted by kw pixels - no data movement per tap.  Each A
//     fragment is loaded into registers once per (row, kw, k-step) and serves every wgmma of the row;
//   * the weights of the three kh taps are stacked ([kh=2 | kh=1 | kh=0] x BN couts) and each of the R output rows
//     has its own BN-column block of the accumulator fragment; input row r issues one N = BN wgmma per output row
//     r-2, r-1, r it feeds (see consume_rows for why they are not one N = 3*BN wgmma);
//   * the 9-tap weight slab of the chunk (3 kw x [3*BN] x 32, hi+lo) is double-buffered in shared memory.
// L2->SM traffic per output pixel drops from 9 to (R+2)/R operand fetches.
//
// Two consumer warpgroups (warps 0-7) each own 64 of the 128 pixels; warp 8 is the TMA producer.  R is chosen per BN
// so that the R * BN / 2 accumulator registers of a thread fit the consumers' register budget.
//
// Fused decoder upsample (optional, Decoder of lib/layers.py:51-64): the leading `up_chunks` channel chunks of the
// input are F.interpolate(x2, bilinear, align_corners=True) of a tensor at half resolution.  Instead of reading a
// materialised up-sampled copy (4x the bytes, and the decoder layers are HBM-bound), ten producer warps
// interpolate each 130-pixel row from half-resolution rows into the swizzled operand slot
// (plain stores + mbarrier arrive; the consumers read the slot with ldmatrix), bit-identical to upsample2x_kernel up to the
// order of the two blends.
//
// Fused output layer (optional, stage 3's dec1 only): the tiles cover only the columns [col0, W - col0) whose mask
// frames the network keeps (lib/nets.py:127-129), and the epilogue applies the 1x1 output convolution and the sigmoid
// (mask_out_kernel) instead of storing the layer.  A runtime branch of the BN <= 32 instantiations with the fused
// upsample, like the fused single-channel dot product, so that no other instantiation changes.
#include <stdio.h>

#include "engine.h"
#include "tc_common.cuh"
#include "tc_plan.h"

namespace vr {

static constexpr int kInterpWarps = 10;             // each covers 7 staged source pixels (+1 neighbour): 70 >= kSrcPx
static constexpr int kConsumerWarps = 8;            // two warpgroups: pixels [0,64) and [64,128) of the tile
static constexpr int kTmaWarp = kConsumerWarps;
static constexpr int kInterpWarp0 = kConsumerWarps + 1;
// output rows per tile: R * BN / 2 accumulator registers per consumer thread, next to 32 registers of A fragments.
// The warps of a block are spread over the four SM sub-partitions, each with 512 registers per lane.  Without the
// fused upsample the block is 9 warps (3 per sub-partition: 168 registers per thread).  With it the block is five
// warpgroups (the TMA warp, the ten interpolation warps and one idle warp make three producer warpgroups; 5 warps
// per sub-partition, 96 registers at launch), and setmaxnreg moves registers from the producer warpgroups to the
// consumers.  setmaxnreg.inc waits until the block's pool, which holds what the block was launched with, can grant
// the request: the budgets must add up to no more than 20 warps x 96 registers.
__host__ __device__ constexpr int rows_per_tile(int BN) { return BN == 64 ? 2 : BN == 32 ? 4 : 8; }
static constexpr int kUpProducerWarps = 12;
static constexpr int kUpConsumerRegs = 128;
static constexpr int kUpProducerRegs = 72;
static constexpr int kUpLaunchRegs = 96;   // 65536 / 640 threads, rounded down to a multiple of 8
static_assert(kConsumerWarps * kUpConsumerRegs + kUpProducerWarps * kUpProducerRegs <=
                  (kConsumerWarps + kUpProducerWarps) * kUpLaunchRegs,
              "setmaxnreg.inc would wait forever for registers the block does not own");
__host__ __device__ constexpr int rows_threads(bool up) { return 32 * (kConsumerWarps + (up ? kUpProducerWarps : 1)); }
static constexpr int kRowPx = 130;                 // 128 + 2 halo pixels
static constexpr int kBoxPx = 136;                 // pixels per TMA row box: makes one plane 17 x 512 B, so that the lo plane
                                                   // of the two-plane box starts on the SWIZZLE_64B repeat (8 rows x 64 B)
static constexpr int kMaxASlots = 8;
static constexpr int kStaticSmem = 3072;           // shared memory not given to the dynamic part: barriers, bias, dot_s
static constexpr int kSrcPx = 68;                  // half-resolution pixels a 130-pixel row interpolates from (fused upsample)
static constexpr uint32_t kKB = 32;                 // channels per chunk (SWIZZLE_64B rows of 64 bytes)
static constexpr uint32_t kRowB = kKB * 2;          // bytes of one pixel of a chunk
static constexpr uint32_t kAPlane = kBoxPx * kRowB; // 8704: hi plane, then lo plane (one two-plane TMA box per row)
static constexpr uint32_t kASlot = 2 * kAPlane;     // 17408 = 17 KiB

// Optional timeline of CTA 0 (builds with -DVR_TRACE only: vr_debug_set(0, 1), read back with vr_debug_trace): clock64 stamps of the three producer /
// consumer loops, to see which of them the others wait for.  [role][event index][3] : role 0 is not recorded, role 1 =
// TMA producer (before the slot wait, after the load was issued, 0), role 2 = interpolation warp 0 (row start, after the
// slot wait, after the arrive).
static constexpr int kTraceEvents = 2048;
__device__ unsigned long long g_rows_trace[3 * kTraceEvents * 3];

template <int BN>
struct RowsGeom {
  static constexpr uint32_t kBPlane = 3 * BN * kRowB;   // hi -> lo plane inside one kw slab ([kh=2|kh=1|kh=0] x BN rows)
  static constexpr uint32_t kBKw = 2 * kBPlane;         // one kw slab, both planes
  static constexpr uint32_t kBBuf = 3 * kBKw;           // the three kw slabs of a chunk
};

struct RowsParams {
  int N, H, W, tiles_w, tiles_h, n_tiles, total_tiles;
  int col0;   // first output column computed: tiles cover columns [col0, col0 + 128 tiles_w) of the W-wide image
  int chunks, CinPadR, Cout, act;
  int n_aslots;
  bf16* out_hi;
  bf16* out_lo;
  int64_t osn, osh;
  int osw;
  int vec16;   // 16-byte stores of 8 channels (tc_vec16)
  const float* bias;
  // fused bilinear x2 producer for the first up_chunks chunks (0: everything comes from the TMA map)
  int up_chunks, xH, xW;
  const bf16* x_hi;   // half-resolution source (NHWC split-bf16), read with plain 16-byte loads by the producer warps
  const bf16* x_lo;
  int64_t xsn, xsh;
  int xsw;
  int trace;   // 1: CTA 0 records its timeline in g_rows_trace
  unsigned long long kmask;   // bit g: some weight on input channels [8g, 8g+8) is non-zero (all ones = no skipping)
  int a_c_off;   // channel coordinate of chunk 0 in the TMA map (negative: the map holds only the skip tensor)
  int l_chunk;   // >= 0: this chunk is read through the second activation map (tmL) from channel 0 (dec1's up-sampled
                 // LSTM channel group, kept in a buffer of its own so that the skip tensor stays dense)
  int n_uslots;   // A slots [0, n_uslots) form the ring of the interpolation warps, [n_uslots, n_aslots) the TMA ring:
                  // one producer per ring (two producers sharing one ring can lap each other: the 1-bit phase
                  // parity cannot tell 'two uses behind' from 'up to date')
  float up_sh, up_sw;
  // fused 1x1 convolution to ONE channel (the LSTM branch's input convolution, lib/layers.py:112,126): every output pixel
  // adds sum_c dot_w[c] * y[c] over this tile's output channels to dot_out[(n * H + h) * W + w] (pre-zeroed fp32 plane)
  const float* dot_w;
  float* dot_out;
  // fused output layer of the network (mask_out_kernel, elementwise.cu) when mask.out is set: the consumers apply the
  // 1x1 convolution to two channels and the sigmoid to each computed pixel, column w being kept frame w - col0, and
  // store no activation.  mask.f3 is not used.
  MaskOutParams mask;
};

// The tile decomposition, shared by the consumers, the TMA producer and the interpolation warps: N tile fastest,
// then the 128-pixel column tile, the R-row tile and the image.
struct RowsTile {
  int nt, w0, h0, n;
};
template <int R>
__device__ __forceinline__ RowsTile rows_tile(const RowsParams& p, int tile) {
  RowsTile t;
  t.nt = tile % p.n_tiles;
  int mt = tile / p.n_tiles;
  t.w0 = p.col0 + (mt % p.tiles_w) * 128;
  mt /= p.tiles_w;
  t.h0 = (mt % p.tiles_h) * R;
  t.n = mt / p.tiles_h;
  return t;
}

// The consumers' positions in the two A rings (one per producer, see RowsParams::n_uslots) and in the weight ring,
// and the weight buffer still held
struct RowsConsumer {
  MbarRing a_up, a_tma, b;
  HeldSlot held_b;
};

// Input row r of one chunk.  For each kw tap the warp loads its 16 x 16 A fragments (hi and lo plane, both k-steps) of
// the slot once with ldmatrix, rows shifted by kw pixels, and every wgmma that needs them reads them from registers:
// one N = BN product per output row o_lo..o_hi the row feeds, each into that row's own column block of the accumulator
// fragment (merging the kh taps into one N = cnt * BN wgmma would make the accumulator windows of consecutive rows
// overlap at different offsets, and ptxas then serialises every wgmma, C7511).  Each kw tap is one commit group; the
// fragments of two consecutive groups live in the two halves of fr, so a group's fragments are overwritten only after
// `wait_group 1` has retired it.  The wgmma read only weights from shared memory: the A slot is free once the last
// ldmatrix of the row has returned.  Every accumulator receives its products in the order chunk, row, kw, k-step,
// hi*hi, lo*hi, hi*lo.
// a: the A ring this chunk's rows come from; returned advanced past them.  ksm: k-steps (16 channels) of the chunk that
// carry weights (bit 0 / 1).  lrow: shared-memory address of this lane's ldmatrix row (pixel 64 wg + 16 (warp % 4) +
// lane % 16) in slot 0; bsrc: descriptor low word of the weight buffer.
template <int BN, int R, int r>
__device__ __forceinline__ MbarRing consume_rows(MbarRing a, RowsConsumer& st, float* acc, uint32_t (&fr)[2][16],
                                                 uint32_t lrow, uint32_t bsrc, uint32_t dhi, uint32_t ksm, int lane) {
  constexpr int o_lo = r - 2 < 0 ? 0 : r - 2;
  constexpr int o_hi = r > R - 1 ? R - 1 : r;
  a.wait_full();
  const uint32_t row = lrow + (uint32_t)a.slot * kASlot;
#pragma unroll
  for (int kw = 0; kw < 3; ++kw) {
    uint32_t* f = fr[(3 * r + kw) & 1];
    // SWIZZLE_64B: 16-byte chunk j of 64-byte row q sits at chunk j ^ ((q >> 1) & 3) (planes are 512-byte aligned)
    const uint32_t q = (row >> 6) + (uint32_t)kw;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      if (!((ksm >> ks) & 1u)) continue;
      const uint32_t a = (q << 6) + ((((uint32_t)(2 * ks) + ((uint32_t)lane >> 4)) ^ ((q >> 1) & 3u)) << 4);
      ldsm_x4(f + 8 * ks, a);
      ldsm_x4(f + 8 * ks + 4, a + kAPlane);
    }
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      if (!((ksm >> ks) & 1u)) continue;
      const uint32_t bo = (uint32_t)(kw * RowsGeom<BN>::kBKw + ks * 32) >> 4;
#pragma unroll
      for (int o = o_lo; o <= o_hi; ++o) {
        const uint32_t b_row = bsrc + (((uint32_t)((2 - (r - o)) * BN) * kRowB) >> 4) + bo;   // tap kh = r - o
        wgmma_split3_rs<BN>(acc + o * (BN / 2), f + 8 * ks, f + 8 * ks + 4, b_row,
                            b_row + (RowsGeom<BN>::kBPlane >> 4), dhi);
      }
    }
    wg_commit();
    if (kw == 2) warp_arrive(a.empty(), lane);
    wg_wait<1>();   // every group but this one is complete: its fragments and the weights it read can be reused
    st.held_b.release(st.b, lane);
  }
  a.advance();
  if constexpr (r + 1 < R + 2)
    return consume_rows<BN, R, r + 1>(a, st, acc, fr, lrow, bsrc, dhi, ksm, lane);
  else
    return a;
}

// w[c] * act(v0 + bias[c]) + w[c + 1] * act(v1 + bias[c + 1]): this thread's share of the fused single-channel 1x1
// convolution on the fp32 activations of one pixel (weights past Cout are zero)
__device__ __forceinline__ float dot_pair(float v0, float v1, const float* bias_s, const float* dot_s, int c, float slope) {
  const float t0 = v0 + bias_s[c], t1 = v1 + bias_s[c + 1];
  return fmaf(fmaxf(t0, 0.f) + slope * fminf(t0, 0.f), dot_s[c], (fmaxf(t1, 0.f) + slope * fminf(t1, 0.f)) * dot_s[c + 1]);
}

// The fused output layer on pixel (n, bin, w) of a one-N-tile layer (BN = Cout = nout), with mask_out_kernel's exact
// arithmetic.  v holds this lane's accumulators of the pixel, channels 8 j + 2 (lane % 4) + {0, 1}: the quad of lanes
// that shares the pixel holds all of its channels.  Each channel becomes act(acc + bias) split to hi / lo bf16 as
// epilogue_pair stores it, then hi + lo: the value mask_out_kernel reads back.  The quad gathers the values in channel
// order by shuffle; lanes 0 / 1 (mod 4) take the dot product with row 0 / 1 of out.weight (mask_s) and write that mask
// channel, lanes 2 / 3 write the same value into the replicated Nyquist row (lib/nets.py:111-115).
template <int BN>
__device__ __forceinline__ void mask_pixel(const RowsParams& p, const float* v, const float* bias_s,
                                           const float* mask_s, float slope, int lane, int n, int bin, int w) {
  float x[BN / 4];
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = 8 * j + 2 * (lane & 3);
    const float t0 = v[4 * j] + bias_s[c], t1 = v[4 * j + 1] + bias_s[c + 1];
    const float y0 = fmaxf(t0, 0.f) + slope * fminf(t0, 0.f);
    const float y1 = fmaxf(t1, 0.f) + slope * fminf(t1, 0.f);
    const float2 hf = bf2_to_f2(f2_to_bf2(y0, y1));
    const float2 lf = bf2_to_f2(f2_to_bf2(y0 - hf.x, y1 - hf.y));
    x[2 * j] = hf.x + lf.x;
    x[2 * j + 1] = hf.y + lf.y;
  }
  const float* wm = mask_s + (lane & 1) * BN;
  float a = 0.f;
#pragma unroll
  for (int c = 0; c < BN; ++c)
    a = fmaf(__shfl_sync(0xffffffffu, x[2 * (c >> 3) + (c & 1)], (lane & ~3) | ((c >> 1) & 3)), wm[c], a);
  const float m = 1.f / (1.f + expf(-a));
  const int tr = w - p.col0;
  const int64_t t = p.mask.t_base0 + (int64_t)n * p.mask.roi_t + tr;
  const bool nyquist = (lane & 2) != 0;
  if (t < 0 || t >= p.mask.t_limit || (nyquist && bin != p.H - 1)) return;
  float* d = p.mask.out + (int64_t)n * p.mask.stride_n + (int64_t)(nyquist ? bin + 1 : bin) * p.mask.stride_bin +
             p.mask.t_base0 + tr + ((lane & 1) ? p.mask.stride_c : 0);
  *d = p.mask.accumulate ? (*d + m) * 0.5f : m;
}

template <int BN, bool UP>
__global__ void __launch_bounds__(rows_threads(UP), 1)
    conv_tc_rows_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                        const __grid_constant__ CUtensorMap tmL, const RowsParams p) {
  typedef RowsGeom<BN> G;
  constexpr int R = rows_per_tile(BN);
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_afull[kMaxASlots];
  __shared__ __align__(8) uint64_t bar_aempty[kMaxASlots];
  __shared__ __align__(8) uint64_t bar_bfull[2];
  __shared__ __align__(8) uint64_t bar_bempty[2];
  __shared__ float bias_s[256];   // folded-BN bias of every N tile, staged once (a global load per use stalled the epilogue)
  __shared__ float dot_s[256];    // weights of the fused single-channel 1x1 convolution (zeros past Cout)

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);   // provably warp-uniform: keeps wgmma unserialised
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = smem_base + (uint32_t)p.n_aslots * kASlot;
  // the A slots hold one ring per producer: [0, n_uslots) for the interpolation warps, [n_uslots, n_aslots) for TMA
  MbarRing a_up(smem_u32(&bar_afull[0]), smem_u32(&bar_aempty[0]), 0, p.n_uslots);
  MbarRing a_tma(smem_u32(&bar_afull[0]), smem_u32(&bar_aempty[0]), p.n_uslots, p.n_aslots);
  MbarRing b_ring(smem_u32(&bar_bfull[0]), smem_u32(&bar_bempty[0]), 0, 2);

  if (warp == kTmaWarp && lane == 0) {
    tma_prefetch(&tmA);
    tma_prefetch(&tmB);
    // an interpolation slot is filled by kInterpWarps producers (one arrive each), a TMA slot by one box
    a_up.init(kInterpWarps, kConsumerWarps);
    a_tma.init(1, kConsumerWarps);
    b_ring.init(1, kConsumerWarps);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < p.n_tiles * BN; i += blockDim.x) {
    bias_s[i] = __ldg(p.bias + i);
    dot_s[i] = p.dot_out && i < p.Cout ? __ldg(p.dot_w + i) : 0.f;
  }
  // the fused output layer only exists where stage 3's dec1 can run (kMaskable); dot_s then holds out.weight [2][BN]
  constexpr bool kMaskable = UP && BN <= 32;
  if constexpr (kMaskable) {
    if (p.mask.out)
      for (int i = threadIdx.x; i < 2 * BN; i += blockDim.x) dot_s[i] = __ldg(p.mask.w + i);
  }
  __syncthreads();
  // Consumers and producers split first: each producer warpgroup (with UP: the TMA warp with interpolation warps 0-2,
  // interpolation warps 3-6, interpolation warps 7-9 with the idle warp) executes the one setmaxnreg.dec below, as
  // setmaxnreg requires of all threads of a warpgroup, and ptxas allocates the consumer code for kUpConsumerRegs
  // because no producer path reaches it.
  if (warp < kConsumerWarps) {
    // ===================== consumer warpgroups: wgmma into registers, then the epilogue =====================
    if constexpr (UP) setmaxnreg_inc<kUpConsumerRegs>();
    const int wg = warp >> 2;   // pixels [64 wg, 64 wg + 64) of the tile
    const float slope = act_slope(p.act);
    const uint32_t dhi = desc_hi(8 * kRowB, 2u);   // SWIZZLE_64B, 8-row groups of 64-byte rows
    const uint32_t lrow = a_base + (uint32_t)(64 * wg + 16 * (warp & 3) + (lane & 15)) * kRowB;
    RowsConsumer st{a_up, a_tma, b_ring};
    float acc[R * BN / 2];
    uint32_t fr[2][16];
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
#pragma unroll
      for (int i = 0; i < R * BN / 2; ++i) acc[i] = 0.f;
      for (int cc = 0; cc < p.chunks; ++cc) {
        st.b.wait_full();
        const uint32_t bsrc = desc_lo(b_base + (uint32_t)st.b.slot * G::kBBuf);
        const bool up = cc < p.up_chunks;
        // k-steps (16 channels = two groups) whose weights are all zero are not issued: exact, since the products
        // would be 0 (lstm / pad channel groups of the concat layouts)
        const uint32_t gm = chunk_groups(p.kmask, cc);
        const uint32_t ksm = ((gm & 0x3u) ? 1u : 0u) | ((gm & 0xCu) ? 2u : 0u);
        // The chosen ring goes by value and its position comes back by select: a ring chosen through a reference can be
        // placed in local memory, and writing back whole rings (the barrier addresses and ranges never change) costs
        // ptxas 8 to 13 more consumer registers.
        const MbarRing a = consume_rows<BN, R, 0>(up ? st.a_up : st.a_tma, st, acc, fr, lrow, bsrc, dhi, ksm, lane);
        st.a_up.slot = up ? a.slot : st.a_up.slot;
        st.a_up.phase = up ? a.phase : st.a_up.phase;
        st.a_tma.slot = up ? st.a_tma.slot : a.slot;
        st.a_tma.phase = up ? st.a_tma.phase : a.phase;
        st.held_b.hold(st.b);   // released with the last row's slot, once the next group has been committed
        st.b.advance();
      }
      wg_wait<0>();
      st.held_b.release_last(st.b, lane);

      const RowsTile tl = rows_tile<R>(p, tile);
      const int w0 = tl.w0, h0 = tl.h0, n = tl.n;
      const int c_lane = tl.nt * BN + 2 * (lane & 3);
      // this thread's share of the fused single-channel 1x1 convolution on pixel px of output row orow
      auto dot = [&](const float* v, int orow, int px) {
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) d += dot_pair(v[4 * j], v[4 * j + 1], bias_s, dot_s, c_lane + 8 * j, slope);
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        d += __shfl_xor_sync(0xffffffffu, d, 2);
        if ((lane & 3) == 0) atomicAdd(p.dot_out + ((int64_t)n * p.H + (h0 + orow)) * p.W + (w0 + px), d);
      };
      const int px0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // pixel of fragment row m; row m + 8 is px0 + 8
#pragma unroll
      for (int orow = 0; orow < R; ++orow) {
        if constexpr (UP) {
          // With the fused upsample the consumers hold 128 registers, next to the interpolation warps, and the
          // transposes of the 16-byte stores spill there (DESIGN 5.2): these variants store each pixel with 8-byte stores,
          // except at BN = 16, whose decoders (dec1 of stages 1 and 2) measured slower with them than with channel pairs.
          constexpr bool kPixel8 = BN > 16;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int px = px0 + 8 * hr;
            const float* v = acc + orow * (BN / 2) + 2 * hr;
            if constexpr (kMaskable) {
              if (p.mask.out) {
                mask_pixel<BN>(p, v, bias_s, dot_s, slope, lane, n, h0 + orow, w0 + px);
                continue;
              }
            }
            if (p.dot_out) dot(v, orow, px);
            const int64_t obase = (int64_t)n * p.osn + (int64_t)(h0 + orow) * p.osh + (int64_t)(w0 + px) * p.osw;
            epilogue_pixel8<BN>(v, bias_s, tl.nt * BN, p.Cout, slope, lane, p.out_hi + obase, p.out_lo + obase,
                                kPixel8 && p.vec16 != 0);
          }
        } else {
          const float* v = acc + orow * (BN / 2);
          if (p.dot_out) {
            dot(v, orow, px0);
            dot(v + 2, orow, px0 + 8);
          }
          const int64_t obase = (int64_t)n * p.osn + (int64_t)(h0 + orow) * p.osh + (int64_t)(w0 + px0) * p.osw;
          const EpiDest d{p.out_hi, p.out_lo, {obase, obase + 8 * (int64_t)p.osw}, {true, true}, tl.nt * BN, p.Cout,
                          p.vec16 != 0};
          epilogue_store<BN>(v, bias_s, slope, lane, d);
        }
      }
    }
  } else {
    if constexpr (UP) setmaxnreg_dec<kUpProducerRegs>();
    if (warp == kTmaWarp) {
      // ===================== TMA producer: one elected lane runs the whole loop nest =====================
      if (elect_one_sync()) {
#ifdef VR_TRACE
        const bool tr = p.trace && blockIdx.x == 0;
#else
        constexpr bool tr = false;
#endif
        int tn = 0;
        for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
          const RowsTile tl = rows_tile<R>(p, tile);
          const int nt = tl.nt, w0 = tl.w0, h0 = tl.h0, n = tl.n;
          for (int cc = 0; cc < p.chunks; ++cc) {
            b_ring.wait_empty();
            const uint32_t bdst = b_base + (uint32_t)b_ring.slot * G::kBBuf;
            mbar_expect_tx(b_ring.full(), G::kBBuf);
#pragma unroll
            for (int kw = 0; kw < 3; ++kw)
              tma_load_3d(bdst + (uint32_t)kw * G::kBKw, &tmB, kw * p.CinPadR + cc * (int)kKB, nt * 3 * BN, 0,
                          b_ring.full());
            b_ring.advance();
            if (cc < p.up_chunks) continue;   // rows of this chunk are produced by the interpolation warps
            const bool from_l = cc == p.l_chunk;
            const int c0 = from_l ? 0 : cc * (int)kKB + p.a_c_off;
            for (int r = 0; r < R + 2; ++r) {
              const unsigned long long t0 = tr ? clock64() : 0ull;
              a_tma.wait_empty();
              mbar_expect_tx(a_tma.full(), kASlot);
              tma_load_5d(a_base + (uint32_t)a_tma.slot * kASlot, from_l ? &tmL : &tmA, c0, w0 - 1, h0 - 1 + r, n, 0,
                          a_tma.full());
              if (tr && tn < kTraceEvents) {
                g_rows_trace[(1 * kTraceEvents + tn) * 3 + 0] = t0;
                g_rows_trace[(1 * kTraceEvents + tn) * 3 + 1] = clock64();
                g_rows_trace[(1 * kTraceEvents + tn) * 3 + 2] = 0ull;
                ++tn;
              }
              a_tma.advance();
            }
          }
        }
      }
      __syncwarp();
    } else if (UP && warp < kInterpWarp0 + kInterpWarps) {
      // ===================== bilinear x2 producer (kInterpWarps autonomous warps) =====================
      // align_corners=True bilinear x2 (ATen upsample_bilinear2d / upsample2x_kernel weights; the vertical blend is done
      // first here).  Warp k owns the source pixels xs + [7k, 7k+7) of the row (+ pixel 7k+7 as right neighbour): lane =
      // (source pixel, 8-channel group) reads its two source rows (hi and lo plane: four 16-byte global loads, issued one
      // row AHEAD so that their latency overlaps the previous row's arithmetic), blends them vertically in registers,
      // fetches the right neighbour's blend by shuffle and emits the 2-3 output pixels whose left source pixel it is,
      // split to hi/lo, straight into the SWIZZLE_64B slot.  Which output pixels those are (and their horizontal weights
      // and slot offsets) depends only on the tile: computed once per tile.  No block-wide barrier and no shared-memory
      // staging (it would add shared-memory traffic next to the consumers' operand reads): every warp waits for
      // the slot (released by the consumer warps) itself and arrives on the slot's mbarrier (count = kInterpWarps).
      if (p.up_chunks > 0) {
        const int wk = warp - kInterpWarp0;
        const int xi = lane >> 2, j = lane & 3;
        const int sx = 7 * wk + xi;              // source pixel of this lane, relative to xs
        const bool emit = xi < 7 && sx < kSrcPx; // xi == 7 only provides the neighbour of xi == 6
        const float inv_sw = p.up_sw > 0.f ? 1.f / p.up_sw : 0.f;
#ifdef VR_TRACE
        const bool tr = p.trace && blockIdx.x == 0 && wk == 0;
#else
        constexpr bool tr = false;
#endif
        int tn = 0;
        const int my_tiles = (p.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
        const int fills = my_tiles * p.up_chunks * (R + 2);
        // iteration state of the NEXT row to fetch (one ahead of the row being written); the tile decomposition
        // (divisions) is redone only when the fetch moves on to another tile
        int f_tile = blockIdx.x, f_cc = 0, f_r = 0, f_h0 = 0, f_X = 0;
        int64_t f_base = 0;
        bool f_px = false;
        auto fetch_tile = [&]() {
          const RowsTile tl = rows_tile<R>(p, f_tile);
          f_h0 = tl.h0 - 1;
          f_X = (int)(p.up_sw * (tl.w0 > 0 ? tl.w0 - 1 : 0)) + sx;
          f_px = sx < kSrcPx && f_X < p.xW;
          f_base = (int64_t)tl.n * p.xsn + (int64_t)f_X * p.xsw + j * 8;
        };
        fetch_tile();
        // Two rows are in flight: the loads of row k+2 are issued right after row k has been stored and announced, so
        // that they have the whole of row k+1 to land.  q* = row k+1, n* = row k+2.
        bf16x8 qah, qch, qal, qcl, nah, nch, nal, ncl;   // rows y0 / y1 of the hi plane, rows y0 / y1 of the lo plane
        float q_ly = 0.f, n_ly = 0.f;
        qah = qch = qal = qcl = nah = nch = nal = ncl = make_uint4(0, 0, 0, 0);
        auto fetch = [&]() {
          qah = nah; qch = nch; qal = nal; qcl = ncl;
          q_ly = n_ly;
          const int h = f_h0 + f_r;
          const bool grp = (chunk_groups(p.kmask, f_cc) >> j) & 1u;   // channel group without weights: zeros are written
          // a row without source data (image border, past the last tile, no weights) keeps all-zero registers, which
          // blend to +0 exactly: no flag has to travel with the row
          if (f_tile < p.total_tiles && h >= 0 && h < p.H && grp && f_px) {
            const float fy = p.up_sh * h;
            const int y0 = (int)fy;
            n_ly = fy - (float)y0;
            const int64_t o0 = f_base + (int64_t)y0 * p.xsh + f_cc * 32;
            const int64_t o1 = o0 + (y0 < p.xH - 1 ? p.xsh : 0);
            nah = ld128(p.x_hi + o0);
            nch = ld128(p.x_hi + o1);
            nal = ld128(p.x_lo + o0);
            ncl = ld128(p.x_lo + o1);
          } else {
            nah = nch = nal = ncl = make_uint4(0, 0, 0, 0);
          }
          if (++f_r == R + 2) {
            f_r = 0;
            if (++f_cc == p.up_chunks) {
              f_cc = 0;
              f_tile += gridDim.x;
              if (f_tile < p.total_tiles) fetch_tile();
            }
          }
        };
        if (fills > 0) {
          fetch();   // row 0
          fetch();   // row 1 (row 0 moves to q*)
        }
        for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
          const int w0 = rows_tile<R>(p, tile).w0;
          const int X = (int)(p.up_sw * (w0 > 0 ? w0 - 1 : 0)) + sx;   // absolute source pixel
          // the output pixels w with (int)(up_sw * w) == X lie in [wc - 1, wc + 3] and there are at most 3 of them
          int e_off[3];
          float e_lx[3];
#pragma unroll
          for (int k = 0; k < 3; ++k) e_off[k] = -1;
          if (emit) {
            const int wc = (int)((float)X * inv_sw);
            int cnt = 0;
#pragma unroll
            for (int dw = -1; dw <= 3; ++dw) {
              const int w = wc + dw;
              const float fx = p.up_sw * (float)w;
              if (w < 0 || w >= p.W || (int)fx != X || w < w0 - 1 || w > w0 + 128) continue;
              const int q = w - (w0 - 1);
              // SWIZZLE_64B (same pattern TMA writes and the consumers' ldmatrix reads): 16-byte chunk j of 64-byte row q sits at chunk
              // j ^ ((q >> 1) & 3) because the XOR takes address bits [7,9) and the planes are 512-byte aligned
              const int off = q * 64 + ((j ^ ((q >> 1) & 3)) << 4);
              const float lx = fx - (float)X;
              if (cnt == 0) { e_off[0] = off; e_lx[0] = lx; }
              else if (cnt == 1) { e_off[1] = off; e_lx[1] = lx; }
              else if (cnt == 2) { e_off[2] = off; e_lx[2] = lx; }
              ++cnt;
            }
          }
          // conv padding columns of the row: slot pixel 0 at the left image border, slot pixel 129 at the right one
          int z_off = -1;
          if (wk == 0 && lane < 8) {
            const int q = lane < 4 ? 0 : kRowPx - 1;
            const int w = w0 - 1 + q;
            if (w < 0 || w >= p.W) z_off = q * 64 + ((j ^ ((q >> 1) & 3)) << 4);
          }
          const bool last_px = X >= p.xW - 1;   // x1 = x0 on the last source pixel (upsample2x_kernel)
          for (int cc = 0; cc < p.up_chunks; ++cc) {
            for (int r = 0; r < R + 2; ++r) {
              const unsigned long long t0 = tr ? clock64() : 0ull;
              float v[8];
              {
                float a[8], c[8];
                unpack8(qah, qal, a);
                unpack8(qch, qcl, c);
                const float ly = q_ly, hy = 1.f - q_ly;
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = hy * a[i] + ly * c[i];
              }
              float nv[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float t = __shfl_down_sync(0xffffffffu, v[i], 4);
                nv[i] = last_px ? v[i] : t;
              }
              const unsigned long long t1 = tr ? clock64() : 0ull;
              a_up.wait_empty();
              const unsigned long long t2 = tr ? clock64() : 0ull;
              uint8_t* slot = smem_raw + (a_base - smem_u32(smem_raw)) + (size_t)a_up.slot * kASlot;
#pragma unroll
              for (int k = 0; k < 3; ++k) {
                if (e_off[k] < 0) continue;
                const float lx = e_lx[k], hx = 1.f - lx;
                float y[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) y[i] = hx * v[i] + lx * nv[i];
                bf16x8 oh, ol;
                split8(y, oh, ol);
                *reinterpret_cast<uint4*>(slot + e_off[k]) = oh;
                *reinterpret_cast<uint4*>(slot + kAPlane + e_off[k]) = ol;
              }
              if (z_off >= 0) {
                *reinterpret_cast<uint4*>(slot + z_off) = make_uint4(0, 0, 0, 0);
                *reinterpret_cast<uint4*>(slot + kAPlane + z_off) = make_uint4(0, 0, 0, 0);
              }
              // no fence.proxy.async: the slot is read by the consumers' ldmatrix (generic proxy), never by wgmma or TMA;
              // the arrive's release and the consumers' acquiring wait order the stores before those reads
              warp_arrive(a_up.full(), lane);
              fetch();   // row k+2 (after the arrive, see above); past the last row it only shifts the pipeline
              if (tr && lane == 0 && tn < kTraceEvents) {
                g_rows_trace[(2 * kTraceEvents + tn) * 3 + 0] = t0;
                g_rows_trace[(2 * kTraceEvents + tn) * 3 + 1] = t2 - t1;   // cycles spent waiting for the slot
                g_rows_trace[(2 * kTraceEvents + tn) * 3 + 2] = clock64();
              }
              ++tn;
              a_up.advance();
            }
          }
        }
      }
      }
  }
}

// every (BN, UP) instantiation the host can launch, and so the BN values tc_choose accepts for this kernel
#define VR_ROWS_FOR_ALL(X) X(16, true) X(16, false) X(32, true) X(32, false) X(64, true) X(64, false)

// bytes of the two weight buffers of the BN instantiations; 0 if there are none
static int rows_b_bytes(int BN) {
#define VR_ROWS_B(BN_, UP_) if (BN == BN_) return (int)(2 * RowsGeom<BN_>::kBBuf);
  VR_ROWS_FOR_ALL(VR_ROWS_B)
#undef VR_ROWS_B
  return 0;
}

bool tc_rows_has(int BN) { return rows_b_bytes(BN) > 0; }

// ------------------------------------------------------------------------------------------------
// f: the fused work (ConvFusion), checked against what the plan can do (TcConv::fuses_*)
cudaError_t tc_rows_launch(const ConvLayer& L, TcConv& tc, const ActView& in, const ActView& out, cudaStream_t s,
                           std::string& err, const ConvFusion& f) {
  const ActView* up_src = f.up;
  if (up_src && (!tc.fuses_upsample(up_src->C) || up_src->H * 2 != in.H || up_src->W * 2 != in.W || up_src->sw % 8)) {
    err = "tc_rows_launch: fused upsample needs a half-resolution source of 32k channels";
    return cudaErrorInvalidValue;
  }
  if (up_src && up_src->C + in.C > tc.CinPad) {
    err = "tc_rows_launch: with a fused upsample the input must hold only the channels after the up-sampled ones";
    return cudaErrorInvalidValue;
  }
  const ActView* last = f.last_chunk;
  if (last && (last->H != in.H || last->W != in.W || last->N != in.N || last->C > tc.KB)) {
    err = "tc_rows_launch: the last-chunk tensor must match the input geometry and fit one chunk";
    return cudaErrorInvalidValue;
  }
  // both planes of one row in one box
  const CUtensorMap* map_a = tc_activation_map(tc, in, kBoxPx, 1, 1, 1, err, L.name);
  const CUtensorMap* map_l = last ? tc_activation_map(tc, *last, kBoxPx, 1, 1, 1, err, L.name) : map_a;
  if (!map_a || !map_l) return cudaErrorInvalidValue;
  // with the fused output layer only the kept columns [offset, W - offset) are computed
  if (f.mask && !tc.fuses_mask(L.Cout, f.mask->offset, up_src != nullptr)) {
    err = "tc_rows_launch: the fused output layer needs a fused upsample, one N tile of Cout <= 32 channels and a "
          "kept width that is a multiple of 128";
    return cudaErrorInvalidValue;
  }
  const int col0 = f.mask ? f.mask->offset : 0;
  RowsParams p;
  p.N = out.N; p.H = out.H; p.W = out.W;
  const bool up = up_src != nullptr;
  p.col0 = col0;
  p.tiles_w = (out.W - 2 * col0) / 128; p.tiles_h = out.H / rows_per_tile(tc.BN); p.n_tiles = tc.n_tiles;
  p.total_tiles = p.tiles_w * p.tiles_h * out.N * tc.n_tiles;
  p.chunks = tc.chunks; p.CinPadR = tc.CinPad; p.Cout = L.Cout; p.act = L.act;
  p.out_hi = out.hi; p.out_lo = out.lo;
  p.osn = out.sn; p.osh = out.sh; p.osw = out.sw;
  p.vec16 = tc_vec16(out);
  p.bias = tc.bias.get();
  p.up_chunks = 0; p.xH = p.xW = 0;
  p.x_hi = p.x_lo = nullptr; p.xsn = p.xsh = 0; p.xsw = 0;
  p.trace = g_debug.trace == 1 ? 1 : 0;
  p.up_sh = p.up_sw = 0.f;
  p.dot_w = f.dot_w; p.dot_out = f.dot_w ? f.dot_out : nullptr;
  p.mask = f.mask ? *f.mask : MaskOutParams{};
  p.a_c_off = 0;
  p.l_chunk = last ? tc.chunks - 1 : -1;
  p.kmask = g_debug.kskip == 1 ? tc.kmask : ~0ull;   // VR_KSKIP=0 issues the all-zero-weight channel groups too
  if (up_src) {
    p.a_c_off = -up_src->C;   // `in` starts at reduction channel up_src->C
    p.up_chunks = up_src->C / 32;
    p.xH = up_src->H; p.xW = up_src->W;
    p.x_hi = up_src->hi; p.x_lo = up_src->lo;
    p.xsn = up_src->sn; p.xsh = up_src->sh; p.xsw = up_src->sw;
    if ((reinterpret_cast<uintptr_t>(up_src->hi) | reinterpret_cast<uintptr_t>(up_src->lo)) & 15) {
      err = "tc_rows_launch: upsample source planes must be 16-byte aligned";
      return cudaErrorInvalidValue;
    }
    p.up_sh = in.H > 1 ? (float)(up_src->H - 1) / (float)(in.H - 1) : 0.f;   // as launch_upsample2x
    p.up_sw = in.W > 1 ? (float)(up_src->W - 1) / (float)(in.W - 1) : 0.f;
  }
  const TcDevice& dv = tc_device();
  if (!dv.ok) {
    err = "tc_rows_launch: cannot query the current device";
    return cudaErrorInvalidValue;
  }
  const int b_bytes = rows_b_bytes(tc.BN);
  p.n_aslots = (dv.max_smem - kStaticSmem - 1024 - b_bytes) / (int)kASlot;
  if (p.n_aslots > kMaxASlots) p.n_aslots = kMaxASlots;
  if (p.n_aslots < (p.up_chunks > 0 ? 4 : 2)) {
    err = "tc_rows_launch: shared memory too small";
    return cudaErrorInvalidValue;
  }
  // the interpolation ring gets the larger share: most chunks of the decoder layers are up-sampled
  p.n_uslots = p.up_chunks > 0 ? p.n_aslots - p.n_aslots / 2 : 0;
  if (p.up_chunks > 0 && p.n_aslots - p.n_uslots < 2) p.n_uslots = p.n_aslots - 2;
  const int dyn = p.n_aslots * (int)kASlot + b_bytes + 1024;
  const int grid = p.total_tiles < dv.num_sms ? p.total_tiles : dv.num_sms;   // persistent: one CTA per SM
  const int threads = rows_threads(up);
  const TcLastConv launched{TC_ROWS, (int)kKB, tc.BN, tc.n_tiles, PAIR_NONE, 0, up ? 1 : 0, p.vec16};
#define VR_ROWS_LAUNCH(BN_, UP_)                                                              \
  if (tc.BN == BN_ && up == UP_) {                                                            \
    g_last_conv = launched;                                                                   \
    conv_tc_rows_kernel<BN_, UP_><<<grid, threads, dyn, s>>>(*map_a, tc.map_b, *map_l, p);    \
    return cudaGetLastError();                                                                \
  }
  VR_ROWS_FOR_ALL(VR_ROWS_LAUNCH)
#undef VR_ROWS_LAUNCH
  err = "tc_rows_launch: no kernel instantiation for this channel tile";
  return cudaErrorInvalidValue;
}


// copies the timeline of the last traced launch (vr_debug_set(0, 1)) to the host: 3 roles x kTraceEvents x 3 stamps
int tc_rows_read_trace(unsigned long long* out, long long capacity) {
  const long long n = 3LL * kTraceEvents * 3;
  if (capacity < n) return -1;
  if (cudaMemcpyFromSymbol(out, g_rows_trace, sizeof(unsigned long long) * (size_t)n) != cudaSuccess) return -1;
  return (int)n;
}

// cudaFuncSetAttribute is per device: called by tc_device() the first time a device is used (conv_tc.cu)
void tc_rows_set_attributes(int max_smem) {
#define VR_ROWS_SET(BN_, UP_)                                                                        \
  cudaFuncSetAttribute(conv_tc_rows_kernel<BN_, UP_>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                       max_smem - kStaticSmem);                                                      \
  cudaFuncSetAttribute(conv_tc_rows_kernel<BN_, UP_>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  VR_ROWS_FOR_ALL(VR_ROWS_SET)
#undef VR_ROWS_SET
}

}  // namespace vr
