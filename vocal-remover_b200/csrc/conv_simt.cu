// fp32 CUDA-core implicit-GEMM convolution with fused folded-BN bias + activation.
//
// Replaces one reference Conv2DBNActiv (lib/layers.py:8-26: Conv2d(bias=False) -> BatchNorm2d(eval)
// -> ReLU | LeakyReLU) for ANY geometry on the path: 3x3 / 1x1, stride 1 / 2, dilation (dh, dw),
// arbitrary channel counts and channel-sliced inputs / outputs (concats are written in place).
// It is (a) the on-device numerical yardstick the wgmma kernel (conv_tc.cu) is validated against
// and (b) the kernel used for the geometries that do not map onto a 128-row wgmma tile
// (tiny feature maps, Cout in {1,2}).  Math is exact fp32 FMA over the 16-bit-significand
// split-bf16 activations.
#include "common.cuh"
#include "kernels.h"

namespace vr {

template <int PX>
__global__ void __launch_bounds__(128) conv_simt_kernel(ConvParams p, int Ho, int Wo, int64_t P) {
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int co0 = (blockIdx.y * 4 + warp) * 8;
  if (co0 >= p.CoutPad) return;
  const int64_t pix0 = (int64_t)blockIdx.x * (32 * PX) + lane;

  int n[PX], ho[PX], wo[PX];
  bool pv[PX];
#pragma unroll
  for (int j = 0; j < PX; ++j) {
    int64_t q = pix0 + 32 * j;
    pv[j] = q < P;
    if (!pv[j]) q = 0;
    wo[j] = (int)(q % Wo);
    int64_t r = q / Wo;
    ho[j] = (int)(r % Ho);
    n[j] = (int)(r / Ho);
  }

  float acc[PX][8];
#pragma unroll
  for (int j = 0; j < PX; ++j)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[j][c] = 0.f;

  for (int kh = 0; kh < p.KH; ++kh) {
    for (int kw = 0; kw < p.KW; ++kw) {
      const bf16* ph[PX];
      const bf16* pl[PX];
      bool ok[PX];
#pragma unroll
      for (int j = 0; j < PX; ++j) {
        int hi_ = ho[j] * p.stride - p.pad_h + kh * p.dil_h;
        int wi_ = wo[j] * p.stride - p.pad_w + kw * p.dil_w;
        ok[j] = pv[j] && hi_ >= 0 && hi_ < p.in.H && wi_ >= 0 && wi_ < p.in.W;
        int64_t off = ok[j] ? (int64_t)n[j] * p.in.sn + (int64_t)hi_ * p.in.sh + (int64_t)wi_ * p.in.sw : 0;
        ph[j] = p.in.hi + off;
        pl[j] = p.in.lo + off;
      }
      const float* wt = p.w + (size_t)((kh * p.KW + kw) * p.CinPad) * p.CoutPad + co0;
      for (int ci = 0; ci < p.CinPad; ci += 8) {
        float x[PX][8];
#pragma unroll
        for (int j = 0; j < PX; ++j) {
          if (ok[j]) {
            load8(ph[j] + ci, pl[j] + ci, x[j]);
          } else {
#pragma unroll
            for (int c = 0; c < 8; ++c) x[j][c] = 0.f;
          }
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float4 w0 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)(ci + c) * p.CoutPad));
          const float4 w1 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)(ci + c) * p.CoutPad + 4));
#pragma unroll
          for (int j = 0; j < PX; ++j) {
            float xv = x[j][c];
            acc[j][0] = fmaf(xv, w0.x, acc[j][0]);
            acc[j][1] = fmaf(xv, w0.y, acc[j][1]);
            acc[j][2] = fmaf(xv, w0.z, acc[j][2]);
            acc[j][3] = fmaf(xv, w0.w, acc[j][3]);
            acc[j][4] = fmaf(xv, w1.x, acc[j][4]);
            acc[j][5] = fmaf(xv, w1.y, acc[j][5]);
            acc[j][6] = fmaf(xv, w1.z, acc[j][6]);
            acc[j][7] = fmaf(xv, w1.w, acc[j][7]);
          }
        }
      }
    }
  }

  const int cnt = min(8, p.Cout - co0);
  if (cnt <= 0) return;
  float b[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) b[c] = __ldg(p.bias + co0 + c);
#pragma unroll
  for (int j = 0; j < PX; ++j) {
    if (!pv[j]) continue;
    float y[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) y[c] = act_apply(acc[j][c] + b[c], p.act);
    int64_t off = (int64_t)n[j] * p.out.sn + (int64_t)ho[j] * p.out.sh + (int64_t)wo[j] * p.out.sw + co0;
    store_split(p.out.hi + off, p.out.lo + off, y, cnt);
  }
}

cudaError_t launch_conv_simt(const ConvParams& p, cudaStream_t stream) {
  const int Ho = p.out.H, Wo = p.out.W;
  const int64_t P = (int64_t)p.out.N * Ho * Wo;
  if (P == 0) return cudaSuccess;
  constexpr int PX = 4;
  dim3 grid((unsigned)((P + 32 * PX - 1) / (32 * PX)), (unsigned)ceil_div(p.CoutPad, 32));
  conv_simt_kernel<PX><<<grid, 128, 0, stream>>>(p, Ho, Wo, P);
  return cudaGetLastError();
}

}  // namespace vr
