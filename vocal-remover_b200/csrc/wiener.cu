// Multichannel Wiener filter refined by expectation-maximisation (--wiener_iterations): norbert 0.2's
// wiener(v, x, iterations, use_softmask=False) for 2 channels and 2 sources, with the masked spectrograms as the initial
// estimates.  DESIGN.md §11 is the contract; tests/wiener_oracle.py restates it in float64 numpy.
//
// Per iteration: a statistics kernel sums, per (bin, frame slice), the 4 real second moments of each source over the
// slice's frames in fp64; a second kernel adds the slices of a bin in order and turns the sums into the spatial
// covariances R_j(f); the apply kernel then filters every (bin, frame) in fp64 and writes the estimates in place.  No
// float atomics (the scale's max is an integer max of non-negative floats), so repeated calls give identical bits.
#include "kernels.h"

namespace vr {

constexpr int WIENER_SLICES = 16;
constexpr int WIENER_THREADS = 256;
// per bin: {sum |y0|^2, sum |y1|^2, Re sum y0 conj(y1), Im sum y0 conj(y1)} of the instruments, then of the vocals;
// after the slice sum the same slots hold {R00, R11, Re R01, Im R01} of each source
constexpr int WIENER_STATS = 8;
constexpr double WIENER_EPS = 1.1920928955078125e-07;    // 2^-23, float32 machine epsilon
constexpr double WIENER_REG = 3.4526698300124393e-04;    // sqrt(2^-23)

// s = max(1, max|X| / 10): the scale norbert divides the mixture and the estimates by
__device__ __forceinline__ double wiener_scale(const float* absmax) { return fmax(1.0, (double)*absmax / 10.0); }

// an estimate as the iteration sees it: the complex64 value stored between iterations, which is y / s rounded to
// complex64 when the buffer still holds the caller's unscaled estimate
__device__ __forceinline__ double2 wiener_load(const float2* p, int64_t i, bool scaled, double s) {
  float2 a = p[i];
  if (!scaled) a = make_float2((float)((double)a.x / s), (float)((double)a.y / s));
  return make_double2(a.x, a.y);
}

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }

__device__ __forceinline__ double2 cscale(double k, double2 a) { return make_double2(k * a.x, k * a.y); }

// grid (bins, WIENER_SLICES): slice k of bin f takes the frames t = k * THREADS + lane (mod SLICES * THREADS)
__global__ void __launch_bounds__(WIENER_THREADS) wiener_stats_kernel(const float2* __restrict__ y,
                                                                      const float2* __restrict__ v, int bins,
                                                                      int64_t T, int scaled,
                                                                      const float* __restrict__ absmax,
                                                                      double* __restrict__ partial) {
  const int f = blockIdx.x;
  const int64_t plane = (int64_t)bins * T;
  const double s = wiener_scale(absmax);
  double acc[WIENER_STATS];
#pragma unroll
  for (int k = 0; k < WIENER_STATS; ++k) acc[k] = 0.0;
  for (int64_t t = (int64_t)blockIdx.y * WIENER_THREADS + threadIdx.x; t < T;
       t += (int64_t)WIENER_SLICES * WIENER_THREADS) {
    const int64_t i = (int64_t)f * T + t;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float2* src = j == 0 ? y : v;
      const double2 a = wiener_load(src, i, scaled, s), b = wiener_load(src, plane + i, scaled, s);
      acc[4 * j + 0] += a.x * a.x + a.y * a.y;
      acc[4 * j + 1] += b.x * b.x + b.y * b.y;
      acc[4 * j + 2] += a.x * b.x + a.y * b.y;
      acc[4 * j + 3] += a.y * b.x - a.x * b.y;
    }
  }
  __shared__ double warp_sum[WIENER_THREADS / 32][WIENER_STATS];
#pragma unroll
  for (int k = 0; k < WIENER_STATS; ++k) {
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5][k] = acc[k];
  }
  __syncthreads();
  if (threadIdx.x < WIENER_STATS) {
    double sum = 0.0;
#pragma unroll
    for (int w = 0; w < WIENER_THREADS / 32; ++w) sum += warp_sum[w][threadIdx.x];
    partial[((int64_t)f * WIENER_SLICES + blockIdx.y) * WIENER_STATS + threadIdx.x] = sum;
  }
}

// one thread per bin: the slices added in order, then R_j = sums_j / (eps + sum_t v_j), sum_t v_j = (S0 + S1) / 2
__global__ void wiener_covariance_kernel(const double* __restrict__ partial, int bins, double* __restrict__ R) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= bins) return;
  double S[WIENER_STATS];
#pragma unroll
  for (int k = 0; k < WIENER_STATS; ++k) {
    double sum = 0.0;
    for (int sl = 0; sl < WIENER_SLICES; ++sl) sum += partial[((int64_t)f * WIENER_SLICES + sl) * WIENER_STATS + k];
    S[k] = sum;
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const double w = WIENER_EPS + 0.5 * (S[4 * j + 0] + S[4 * j + 1]);
#pragma unroll
    for (int k = 0; k < 4; ++k) R[(int64_t)f * WIENER_STATS + 4 * j + k] = S[4 * j + k] / w;
  }
}

// one thread per (bin, frame): C = sum_j v_j R_j + reg I, u = C^-1 x by the adjugate, y_j = v_j R_j u, in place
__global__ void wiener_apply_kernel(const float2* __restrict__ spec, float2* __restrict__ y, float2* __restrict__ v,
                                    const double* __restrict__ R, int bins, int64_t T, int scaled, int last,
                                    const float* __restrict__ absmax) {
  const int64_t plane = (int64_t)bins * T;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= plane) return;
  const int64_t f = i / T;
  const double s = wiener_scale(absmax);
  const float2 X0 = spec[i], X1 = spec[plane + i];
  const double2 x0 = make_double2((double)X0.x / s, (double)X0.y / s);
  const double2 x1 = make_double2((double)X1.x / s, (double)X1.y / s);
  float2* dst[2] = {y, v};
  double vj[2];
  double2 Rj[2][2][2];   // [source][row][column]
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const double2 a = wiener_load(dst[j], i, scaled, s), b = wiener_load(dst[j], plane + i, scaled, s);
    vj[j] = 0.5 * ((a.x * a.x + a.y * a.y) + (b.x * b.x + b.y * b.y));
    const double* r = R + f * WIENER_STATS + 4 * j;
    Rj[j][0][0] = make_double2(r[0], 0.0);
    Rj[j][1][1] = make_double2(r[1], 0.0);
    Rj[j][0][1] = make_double2(r[2], r[3]);
    Rj[j][1][0] = make_double2(r[2], -r[3]);
  }
  const double c00 = vj[0] * Rj[0][0][0].x + vj[1] * Rj[1][0][0].x + WIENER_REG;
  const double c11 = vj[0] * Rj[0][1][1].x + vj[1] * Rj[1][1][1].x + WIENER_REG;
  const double2 c01 = cadd(cscale(vj[0], Rj[0][0][1]), cscale(vj[1], Rj[1][0][1]));
  const double2 c10 = make_double2(c01.x, -c01.y);
  const double rdet = 1.0 / (c00 * c11 - (c01.x * c01.x + c01.y * c01.y));
  // u = C^-1 x = adj(C) x / det, both rows in the same form
  const double2 u0 = cscale(rdet, cadd(cmul(make_double2(c11, 0.0), x0), cmul(make_double2(-c01.x, -c01.y), x1)));
  const double2 u1 = cscale(rdet, cadd(cmul(make_double2(-c10.x, -c10.y), x0), cmul(make_double2(c00, 0.0), x1)));
#pragma unroll
  for (int j = 0; j < 2; ++j) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const double2 g = cscale(vj[j], cadd(cmul(Rj[j][c][0], u0), cmul(Rj[j][c][1], u1)));
      float2 out = make_float2((float)g.x, (float)g.y);   // complex64 storage between iterations
      if (last) out = make_float2((float)(s * (double)out.x), (float)(s * (double)out.y));
      dst[j][c * plane + i] = out;
    }
  }
}

int64_t wiener_scratch(int bins) { return (int64_t)bins * WIENER_STATS * (WIENER_SLICES + 1) + 1; }

cudaError_t launch_wiener(const float2* spec, float2* y, float2* v, int bins, int64_t T, int iterations,
                          double* scratch, cudaStream_t stream) {
  if (iterations <= 0 || T <= 0) return cudaSuccess;
  double* partial = scratch;
  double* R = scratch + (int64_t)bins * WIENER_STATS * WIENER_SLICES;
  float* absmax = reinterpret_cast<float*>(R + (int64_t)bins * WIENER_STATS);
  const int64_t plane = (int64_t)bins * T;
  cudaError_t e = launch_absmax(spec, 2 * plane, absmax, stream);
  for (int it = 0; it < iterations && e == cudaSuccess; ++it) {
    const int scaled = it > 0;
    wiener_stats_kernel<<<dim3((unsigned)bins, WIENER_SLICES), WIENER_THREADS, 0, stream>>>(y, v, bins, T, scaled,
                                                                                          absmax, partial);
    if ((e = cudaGetLastError()) != cudaSuccess) break;
    wiener_covariance_kernel<<<(unsigned)((bins + 127) / 128), 128, 0, stream>>>(partial, bins, R);
    if ((e = cudaGetLastError()) != cudaSuccess) break;
    wiener_apply_kernel<<<(unsigned)((plane + 255) / 256), 256, 0, stream>>>(spec, y, v, R, bins, T, scaled,
                                                                            it == iterations - 1, absmax);
    e = cudaGetLastError();
  }
  return e;
}

}  // namespace vr
