// LSTM branch of BaseNet (reference lib/layers.py:108-133, wired at lib/nets.py:23,38):
//   1x1 conv (2n -> 1) + BN + ReLU  ->  (T, N, bins)  ->  BiLSTM(hidden = nout_lstm/2, gate order i,f,g,o)
//   -> Linear(nout_lstm -> bins) + BatchNorm1d(eval) + ReLU -> one extra channel of the dec1 input.
// 0.18 % of the FLOPs but a 128-step sequential dependency on the critical path between dec2 and dec1: the 1x1
// convolution is accumulated by dec2's epilogue (conv_tc_rows.cu; lstm_inconv_kernel only when dec2 runs elsewhere), the
// input projection is hoisted into one GEMM, the recurrence runs as one persistent CTA per (window, direction) with its
// W_hh row held in registers and h exchanged through shared memory, and the dense layer is the same GEMM computed
// transposed into an fp32 plane.  All math fp32 with accurate expf/tanhf.
#include "common.cuh"
#include "kernels.h"

namespace vr {

// ------------------------------------------------------------------------------------------------
__global__ void lstm_inconv_kernel(ActView in, const float* __restrict__ w, float* __restrict__ out) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = (int64_t)in.N * in.H * in.W;
  if (idx >= total) return;
  int t = (int)(idx % in.W);
  int64_t r = idx / in.W;
  int bin = (int)(r % in.H);
  int n = (int)(r / in.H);
  int64_t o = (int64_t)n * in.sn + (int64_t)bin * in.sh + (int64_t)t * in.sw;
  float acc = 0.f;
  for (int c = 0; c < in.C; c += 8) {
    float x[8];
    load8(in.hi + o + c, in.lo + o + c, x);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc = fmaf(x[i], __ldg(w + c + i), acc);
  }
  out[idx] = acc;   // [n][bin][t] pre-activation sums; the input projection applies the folded BN bias + ReLU
}

cudaError_t launch_lstm_inconv(ActView in, const float* w, float* out, cudaStream_t stream) {
  int64_t total = (int64_t)in.N * in.H * in.W;
  if (total == 0) return cudaSuccess;
  lstm_inconv_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, w, out);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// C[M][N] = f(A)[M][K] * B[N][K]^T on a 128x64 tile (256 threads x 8x4 outputs, 16-deep k slab, register prefetch of the
// next slab, double-buffered shared memory: one barrier per slab), fp32 FMA.  The two GEMMs of the branch:
//   input projection  xp[(n,t)][gate] = relu(l0[n][:][t] + b0) . wih[gate][:] + bias[gate]
//                     (ATRANS: A is stored [n][K][T] - the 1x1 convolution's pre-activation sums, t contiguous - and the
//                      folded BatchNorm bias + ReLU of that convolution are applied while the slab is loaded)
//   dense + BN + ReLU y[bin][(n,t)]   = relu(scale[bin] * (wd[bin][:] . hs[(n,t)][:]) + shift[bin])
//                     (computed transposed, so that the (n,t) index, contiguous in the consumer, runs along the store lanes)
struct GemmArgs {
  const float* A;
  const float* B;
  float* C;
  int M, N, K;
  int T;              // ATRANS: row m = (n, t) = (m / T, m % T) of A lives at A[(n * K + k) * T + t]
  float a_bias;       // ATRANS: f(a) = max(a + a_bias, 0)
  const float* col_bias;
  const float* row_scale;
  const float* row_shift;
  int relu;
};

template <bool ATRANS>
__global__ void __launch_bounds__(256) gemm_nt_128x64_kernel(const GemmArgs g) {
  __shared__ __align__(16) float As[2][16][128 + 4];
  __shared__ __align__(16) float Bs[2][16][64 + 4];
  const float* __restrict__ A = g.A;
  const float* __restrict__ B = g.B;
  const int M = g.M, N = g.N, K = g.K;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * 128, n0 = blockIdx.x * 64;
  // slab loads.  B (and A when it is row-major): row lr (+64), four k from lk.  ATRANS: k row ak (+8), four m from am.
  const int lr = tid >> 2, lk = (tid & 3) * 4;
  const int ak = tid >> 5, am = (tid & 31) * 4;
  const bool vec_k = (K & 3) == 0 && ((reinterpret_cast<uintptr_t>(B) | (ATRANS ? 0 : reinterpret_cast<uintptr_t>(A))) & 15) == 0;
  const bool vec_m = ATRANS && (g.T & 3) == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0;
  auto a_at = [&](int m, int k) -> float {   // guarded scalar access, any layout
    if (m >= M || k >= K) return 0.f;
    if (!ATRANS) return A[(int64_t)m * K + k];
    const int n = m / g.T, t = m - n * g.T;
    return fmaxf(A[((int64_t)n * K + k) * g.T + t] + g.a_bias, 0.f);
  };
  auto a_quad_k = [&](int m, int k) -> float4 {   // row-major A: four consecutive k
    if (vec_k) return m < M && k < K ? *reinterpret_cast<const float4*>(A + (int64_t)m * K + k) : make_float4(0.f, 0.f, 0.f, 0.f);
    return make_float4(a_at(m, k), a_at(m, k + 1), a_at(m, k + 2), a_at(m, k + 3));
  };
  auto a_quad_m = [&](int m, int k) -> float4 {   // ATRANS: four consecutive m (same image when T % 4 == 0)
    if (vec_m) {
      if (m >= M || k >= K) return make_float4(0.f, 0.f, 0.f, 0.f);   // M = n * T is a multiple of 4 as well
      const int n = m / g.T, t = m - n * g.T;
      const float4 x = *reinterpret_cast<const float4*>(A + ((int64_t)n * K + k) * g.T + t);
      return make_float4(fmaxf(x.x + g.a_bias, 0.f), fmaxf(x.y + g.a_bias, 0.f), fmaxf(x.z + g.a_bias, 0.f),
                         fmaxf(x.w + g.a_bias, 0.f));
    }
    return make_float4(a_at(m, k), a_at(m + 1, k), a_at(m + 2, k), a_at(m + 3, k));
  };
  auto b_quad = [&](int n, int k) -> float4 {
    if (vec_k) return n < N && k < K ? *reinterpret_cast<const float4*>(B + (int64_t)n * K + k) : make_float4(0.f, 0.f, 0.f, 0.f);
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = n < N && k + i < K ? B[(int64_t)n * K + k + i] : 0.f;
    return make_float4(v[0], v[1], v[2], v[3]);
  };
  float4 ra0, ra1, rb;
  auto gload = [&](int k0) {
    if (ATRANS) {
      ra0 = a_quad_m(m0 + am, k0 + ak);
      ra1 = a_quad_m(m0 + am, k0 + ak + 8);
    } else {
      ra0 = a_quad_k(m0 + lr, k0 + lk);
      ra1 = a_quad_k(m0 + lr + 64, k0 + lk);
    }
    rb = b_quad(n0 + lr, k0 + lk);
  };
  auto sstore = [&](int buf) {
    if (ATRANS) {
      *reinterpret_cast<float4*>(&As[buf][ak][am]) = ra0;
      *reinterpret_cast<float4*>(&As[buf][ak + 8][am]) = ra1;
    } else {
      As[buf][lk + 0][lr] = ra0.x; As[buf][lk + 1][lr] = ra0.y; As[buf][lk + 2][lr] = ra0.z; As[buf][lk + 3][lr] = ra0.w;
      As[buf][lk + 0][lr + 64] = ra1.x; As[buf][lk + 1][lr + 64] = ra1.y;
      As[buf][lk + 2][lr + 64] = ra1.z; As[buf][lk + 3][lr + 64] = ra1.w;
    }
    Bs[buf][lk + 0][lr] = rb.x; Bs[buf][lk + 1][lr] = rb.y; Bs[buf][lk + 2][lr] = rb.z; Bs[buf][lk + 3][lr] = rb.w;
  };
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  gload(0);
  sstore(0);
  __syncthreads();
  const int nk = (K + 15) >> 4;
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload((kt + 1) << 4);
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    if (kt + 1 < nk) sstore(buf ^ 1);
    __syncthreads();
  }
  const int gn = n0 + tx * 4;
  float cb[4] = {0.f, 0.f, 0.f, 0.f};
  if (g.col_bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (gn + j < N) cb[j] = g.col_bias[gn + j];
  }
  const bool vec_c = (N & 3) == 0 && (reinterpret_cast<uintptr_t>(g.C) & 15) == 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + ty * 8 + i;
    if (gm >= M) continue;
    const float sc = g.row_scale ? g.row_scale[gm] : 1.f, sf = g.row_scale ? g.row_shift[gm] : 0.f;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[j] = fmaf(acc[i][j] + cb[j], sc, sf);
      if (g.relu) v[j] = fmaxf(v[j], 0.f);
    }
    float* dst = g.C + (int64_t)gm * N + gn;
    if (vec_c && gn + 3 < N) {
      *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (gn + j < N) dst[j] = v[j];
    }
  }
}

cudaError_t launch_lstm_input_projection(const float* l0, float conv_bias, const float* wih, const float* bih, float* xp,
                                         int N, int T, int bins, int gates, cudaStream_t stream) {
  if (N == 0 || T == 0 || gates == 0) return cudaSuccess;
  GemmArgs g{l0, wih, xp, N * T, gates, bins, T, conv_bias, bih, nullptr, nullptr, 0};
  dim3 grid((unsigned)ceil_div(gates, 64), (unsigned)ceil_div(N * T, 128));
  gemm_nt_128x64_kernel<true><<<grid, 256, 0, stream>>>(g);
  return cudaGetLastError();
}

cudaError_t launch_lstm_dense(const float* hs, const float* wd, const float* scale, const float* shift, int NT, int K,
                              int bins, float* y, cudaStream_t stream) {
  if (NT == 0 || bins == 0) return cudaSuccess;
  GemmArgs g{wd, hs, y, bins, NT, K, 0, 0.f, nullptr, scale, shift, 1};
  dim3 grid((unsigned)ceil_div(NT, 64), (unsigned)ceil_div(bins, 128));
  gemm_nt_128x64_kernel<false><<<grid, 256, 0, stream>>>(g);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoid_acc(float x) { return 1.f / (1.f + expf(-x)); }

// grid (N, 2 directions), block 4*HID threads.  Thread j owns gate row j of W_hh (registers).
template <int HID>
__global__ void __launch_bounds__(4 * HID) lstm_recurrence_kernel(const float* __restrict__ xp,
                                                                  const float* __restrict__ whh,
                                                                  float* __restrict__ hs, int T) {
  const int n = blockIdx.x, dir = blockIdx.y, j = threadIdx.x;
  __shared__ float h_s[HID];
  __shared__ float g_s[4 * HID];
  float wrow[HID];
#pragma unroll
  for (int k = 0; k < HID; ++k) wrow[k] = whh[((int64_t)dir * 4 * HID + j) * HID + k];
  if (j < HID) h_s[j] = 0.f;
  float c = 0.f;
  __syncthreads();
  const float* xp_n = xp + (int64_t)n * T * 8 * HID + dir * 4 * HID + j;
  int t = dir ? T - 1 : 0;
  float xnext = xp_n[(int64_t)t * 8 * HID];
  for (int s = 0; s < T; ++s) {
    const int tn = dir ? t - 1 : t + 1;
    // four independent partial sums: the 4-cycle FMA latency chain is HID/4 long instead of HID
    float g0 = xnext, g1 = 0.f, g2 = 0.f, g3 = 0.f;
    if (s + 1 < T) xnext = xp_n[(int64_t)tn * 8 * HID];
#pragma unroll
    for (int k = 0; k < HID; k += 4) {
      g0 = fmaf(wrow[k], h_s[k], g0);
      g1 = fmaf(wrow[k + 1], h_s[k + 1], g1);
      g2 = fmaf(wrow[k + 2], h_s[k + 2], g2);
      g3 = fmaf(wrow[k + 3], h_s[k + 3], g3);
    }
    // every thread applies its own gate's non-linearity (i, f, o: sigmoid; g: tanh) - one transcendental per thread in
    // parallel instead of five in sequence on the HID combining threads
    const float pre = (g0 + g1) + (g2 + g3);
    g_s[j] = (j >= 2 * HID && j < 3 * HID) ? tanhf(pre) : sigmoid_acc(pre);
    __syncthreads();
    if (j < HID) {
      const float ig = g_s[j], fg = g_s[HID + j], gg = g_s[2 * HID + j], og = g_s[3 * HID + j];
      c = fg * c + ig * gg;
      float h = og * tanhf(c);
      h_s[j] = h;
      hs[((int64_t)n * T + t) * 2 * HID + dir * HID + j] = h;
    }
    __syncthreads();
    t = tn;
  }
}

cudaError_t launch_lstm_recurrence(const float* xp, const float* whh, float* hs, int N, int T, int hid,
                                   cudaStream_t stream) {
  if (N == 0) return cudaSuccess;
  dim3 grid((unsigned)N, 2);
  switch (hid) {
    case 8: lstm_recurrence_kernel<8><<<grid, 32, 0, stream>>>(xp, whh, hs, T); break;
    case 16: lstm_recurrence_kernel<16><<<grid, 64, 0, stream>>>(xp, whh, hs, T); break;
    case 32: lstm_recurrence_kernel<32><<<grid, 128, 0, stream>>>(xp, whh, hs, T); break;
    case 64: lstm_recurrence_kernel<64><<<grid, 256, 0, stream>>>(xp, whh, hs, T); break;
    case 128: lstm_recurrence_kernel<128><<<grid, 512, 0, stream>>>(xp, whh, hs, T); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace vr
