// Host-side plan of one convolution layer for the wgmma kernels (conv_tc.cu, conv_tc_rows.cu).
#pragma once
#include <cuda.h>

#include <map>
#include <tuple>

#include "engine.h"

namespace vr {

typedef std::tuple<const void*, const void*, int, int, int, int> ViewKey;

struct TcRowsPlan {   // row-streaming variant: 3x3, stride 1, dilation 1, W % 128 == 0 (conv_tc_rows.cu)
  bool ok = false;
  int KB = 32, CinPadR = 0, chunks = 0, BN = 0, n_tiles = 0;
  unsigned long long kmask = ~0ull;   // bit g: input channels [8g, 8g+8) carry a non-zero weight
  bf16* w_planes = nullptr;   // [2][n_tiles*BN][9*CinPadR]
  float* bias = nullptr;      // [n_tiles*BN]
  CUtensorMap map_b;
  std::map<ViewKey, CUtensorMap> map_a;
  std::map<ViewKey, CUtensorMap> map_l;   // second activation map (the chunk read from its own buffer)
};

struct TcHaloPlan {   // halo-tile variant: 3x3, stride 1, dilation 1, W in {16, 32, 64} (conv_tc_halo.cu)
  bool ok = false;
  int CinPadH = 0, chunks = 0;   // BN, n_tiles and the bias are the generic plan's
  unsigned long long kmask = ~0ull;   // bit g: input channels [8g, 8g+8) carry a non-zero weight
  bf16* w_planes = nullptr;   // [2][n_tiles*BN][9*CinPadH]
  CUtensorMap map_b;
  std::map<ViewKey, CUtensorMap> map_a[2];   // per MB (the halo box height depends on it)
};

struct TcConv {
  int CinPadTC = 0, KB = 0, cchunks = 0, SUBS = 0, taps = 0, Ktot = 0, CoutPadN = 0, BN = 0, n_tiles = 0;
  bf16* w_planes = nullptr;   // [2][CoutPadN][Ktot]
  float* bias = nullptr;      // [n_tiles*BN]
  CUtensorMap map_b;
  std::map<ViewKey, CUtensorMap> map_a;
  TcRowsPlan rows;
  TcHaloPlan halo;
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tc_encode_fn();
uint16_t tc_f2bf(float f);
float tc_bf2f(uint16_t h);

// conv_tc_rows.cu
bool tc_rows_prepare(ConvLayer& L, TcConv& tc, std::string& err, std::vector<void*>& allocs);
bool tc_rows_supported(const ConvLayer& L, const TcConv& tc, const ActView& in, const ActView& out);
cudaError_t tc_rows_launch(ConvLayer& L, TcConv& tc, const ActView& in, const ActView& out, cudaStream_t s,
                           std::string& err, const ActView* up_src = nullptr, const ActView* extra = nullptr);
void tc_rows_set_attributes(int max_smem);
int tc_rows_read_trace(unsigned long long* out, long long capacity);

// conv_tc_halo.cu
bool tc_halo_prepare(ConvLayer& L, TcConv& tc, std::string& err, std::vector<void*>& allocs);
bool tc_halo_supported(const ConvLayer& L, const TcConv& tc, const ActView& in, const ActView& out);
cudaError_t tc_halo_launch(ConvLayer& L, TcConv& tc, const ActView& in, const ActView& out, cudaStream_t s,
                           std::string& err);
void tc_halo_set_attributes(int max_smem);

// Properties of the CURRENT device, cached per device ordinal.  The first use on a device also opts the tensor-core
// kernels in to their dynamic shared memory there (cudaFuncSetAttribute is per device, so a process that drives
// several GPUs - one context per GPU - must do it on each of them).
struct TcDevice {
  bool ok = false;
  int num_sms = 0, max_smem = 0;
};
const TcDevice& tc_device();

// validation knobs (vr_debug_set): [0] = 1: CTA 0 of the row kernel records a timeline (vr_debug_trace), [2] = 1: vr_debug_conv uses the 64-wide row tile, [1] = 1 disables the row kernel, [4] = k: k of the row slots feed the interpolation
// warps (default half), [5] = 1 (default): decoder upsample fused into the row kernel, [6] = 1 (default): the row
// and halo kernels skip channel groups whose weights are all zero, [3] = 1: the layers of the halo kernel go to the
// per-tap kernel instead, [3] = 2 / 3: the halo kernel uses MB = 1 / 2 (where the height tiles) for every layer;
// the other entries are unused
extern int g_tc_debug[8];

}  // namespace vr
