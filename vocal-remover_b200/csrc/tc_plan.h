// Host-side plan of one convolution layer for the wgmma kernels (conv_tc.cu, conv_tc_rows.cu, conv_tc_halo.cu).
// tc_prepare (conv_tc.cu) chooses the kernel of a layer once, from its fixed geometry (k, stride, dilation, channels and
// the H x W of its output maps), and packs the weights once, in that kernel's layout.  The launches read the plan; only
// the halo kernel's MB, which depends on the batch size, is chosen per launch.
#pragma once
#include <cuda.h>

#include <map>
#include <tuple>

#include "engine.h"

namespace vr {

enum TcKind {
  TC_NONE,      // CUDA-core kernel (conv_simt.cu)
  TC_GENERIC,   // one shifted pixel box per (tap, channel chunk) (conv_tc.cu)
  TC_ROWS,      // row streaming: 3x3, stride 1, dilation 1, W % 128 == 0, H % 8 == 0 (conv_tc_rows.cu)
  TC_HALO,      // halo tile: 3x3, stride 1, dilation 1, W in {16, 32, 64} (conv_tc_halo.cu)
};

// How the generic kernel's four-warpgroup variants pair work in one CTA (conv_tc.cu, DESIGN §5.3):
// PAIR_M: two adjacent 128-pixel m-tiles share each weight box; PAIR_N: both N tiles of a layer share each activation box.
enum TcPair { PAIR_NONE = 0, PAIR_M = 1, PAIR_N = 2 };

// activation view (hi, lo, N, H, W, C), TMA box (W, H, N extents) and channels per box
typedef std::tuple<const void*, const void*, int, int, int, int, int, int, int, int> ViewKey;

struct TcConv {
  TcKind kind = TC_NONE;
  int H = 0, W = 0;   // output maps the kernel was chosen for
  // KB: channels per chunk (generic: 64 / 32 / 16, rows and halo: 32); CinPad: input channels padded to whole chunks
  int KB = 0, CinPad = 0, chunks = 0, BN = 0, n_tiles = 0;
  unsigned long long kmask = ~0ull;   // bit g: input channels [8g, 8g+8) carry a non-zero weight (rows and halo)
  // weights, hi plane then lo plane: generic / halo [2][n_tiles*BN][taps*CinPad] (tap-major K), rows
  // [2][n_tiles*3*BN][3*CinPad] (the three kh taps of an N tile stacked along N, kw-major K)
  DevPtr<bf16> w_planes;
  DevPtr<float> bias;   // [n_tiles*BN]
  CUtensorMap map_b;
  std::map<ViewKey, CUtensorMap> map_a;
  // generic kernel only: the pairing a launch considers (PAIR_N where n_tiles == 2 and KB >= 32, else PAIR_M; whether
  // it pays depends on the batch, so tc_launch decides), and the weights in the paired variants' boxes of pair_KB
  // channels.  PAIR_M is legal for every generic layer.
  TcPair pair = PAIR_NONE;
  int pair_KB = 0;
  CUtensorMap map_b_pair;
  // What a launch of this plan can fuse (ConvFusion); the launchers reject anything else.
  // the row kernel can produce the leading up_C channels of its input as the x2 upsample of a half-resolution tensor
  bool fuses_upsample(int up_C) const { return kind == TC_ROWS && up_C % 32 == 0 && up_C <= CinPad; }
  // the row kernel can accumulate a 1x1 convolution to one channel in its epilogue
  bool fuses_dot() const { return kind == TC_ROWS; }
  // the row kernel can compute only the columns [offset, W - offset), in whole 128-pixel tiles, and apply the network's
  // output layer (mask_out_kernel) there in its epilogue: one quad of lanes must hold all Cout channels of a pixel, and
  // only the BN <= 32 instantiations with a fused upsample (up) carry that epilogue
  bool fuses_mask(int Cout, int offset, bool up) const {
    const int kept = W - 2 * offset;
    return kind == TC_ROWS && up && n_tiles == 1 && BN <= 32 && BN == Cout && offset >= 0 && kept > 0 &&
           kept % 128 == 0;
  }
};

TcKind tc_choose(const ConvLayer& L, int H, int W, bool rows_wide);
// tensor map of an activation view: both split-bf16 planes in one box of {kb, bw, bh, bn, 2} elements (kb = 0:
// tc.KB), element stride es along W and H; cached in the plan.  nullptr (err set) if TMA cannot read the view.
const CUtensorMap* tc_activation_map(TcConv& tc, const ActView& v, int bw, int bh, int bn, int es, std::string& err,
                                     const std::string& name, int kb = 0);

// conv_tc_rows.cu
cudaError_t tc_rows_launch(const ConvLayer& L, TcConv& tc, const ActView& in, const ActView& out, cudaStream_t s,
                           std::string& err, const ConvFusion& f);
void tc_rows_set_attributes(int max_smem);
bool tc_rows_has(int BN);   // the row kernel is instantiated for this BN
int tc_rows_read_trace(unsigned long long* out, long long capacity);

// conv_tc_halo.cu
cudaError_t tc_halo_launch(const ConvLayer& L, TcConv& tc, const ActView& in, const ActView& out, cudaStream_t s,
                           std::string& err);
void tc_halo_set_attributes(int max_smem);
bool tc_halo_has(int BN);   // the halo kernel is instantiated for this BN

// Properties of the CURRENT device, cached per device ordinal.  The first use on a device also opts the tensor-core
// kernels in to their dynamic shared memory there (cudaFuncSetAttribute is per device, so a process that drives
// several GPUs - one context per GPU - must do it on each of them).
struct TcDevice {
  bool ok = false;
  int num_sms = 0, max_smem = 0;
};
const TcDevice& tc_device();

// validation switches, set with vr_debug_set(key, value)
struct TcDebug {
  int trace = 0;       // key 0 = 1: CTA 0 of the row kernel records a timeline (-DVR_TRACE builds, vr_debug_trace)
  int rows_wide = 0;   // key 2 = 1: vr_debug_conv uses the row kernel's 64-wide tile
  int halo = 0;        // key 3 = 1: layers prepared from then on go to the generic kernel instead of the halo kernel;
                       // 2 / 3: the halo kernel uses MB = 1 / 2 (where the height tiles) in every launch
  int kskip = 1;       // key 6 = 1 (default): the row and halo kernels skip channel groups whose weights are all zero
  int crop_mask = 1;   // key 7 = 1 (default): stage 3's dec1 computes only the kept frames and applies the output layer
                       // in its epilogue where it can; 0: it computes every frame into f3_, then mask_out_kernel runs
  int pair = 0;        // key 8: generic kernel pairing, 0 = automatic, 1 = never (two warpgroups), 2 / 3 = PAIR_M /
                       // PAIR_N in every launch where the layer allows it
  int pair_stores = 0;   // key 9: 0 = 16-byte epilogue stores wherever the launch allows them, 1 = epilogue_pair's
                         // 4-byte channel-pair stores in every launch
};
extern TcDebug g_debug;

// The last convolution launch of this process, as the launchers decided it (vr_debug_last_conv): kind (TcKind), KB,
// BN, n_tiles, pairing (TcPair, generic kernel), MB (halo kernel), fused upsample (row kernel) and whether the epilogue
// stores 8 channels with 16-byte stores.  Fields a kernel does not have are 0.
struct TcLastConv {
  int kind = TC_NONE, KB = 0, BN = 0, n_tiles = 0, pair = PAIR_NONE, MB = 0, up = 0, vec16 = 0;
};
extern TcLastConv g_last_conv;

// The epilogue of a launch into `out` may store 8 channels with one 16-byte store per plane (epilogue_store,
// tc_common.cuh): both planes are 16-byte aligned, every stride is a multiple of 8 channels, and key 9 is not 1.
bool tc_vec16(const ActView& out);

}  // namespace vr
