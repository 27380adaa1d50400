// BSS Eval images with time-invariant distortion filters ("v4": one set of filters per track) on the device: the SDR,
// ISR, SIR and SAR of lib/bsseval.py, restated in float64 numpy by oracle/bsseval_oracle.py.  DESIGN.md section 10
// states the contract; the pipeline is
//
//   bss_corr_kernel         r[a][b](l) = sum_u s_a(u) * y_b(u + l), l < L, y = the M references then the M estimates
//                           (M = K * C signals): the Toeplitz blocks of the Gram matrix G and the right-hand sides d
//   bss_corr_reduce_kernel  the per-group partial sums of the above, added in group order
//   bss_assemble_kernel     G + eps I (all K*C*L unknowns) and its K per-source diagonal blocks, and the right-hand sides
//   chol_*_kernel           blocked Cholesky of each system (64 x 64 tiles) and its two triangular solves; a system
//                           whose factorisation meets a non-positive pivot is assembled and factored again with a
//                           larger eps (the loading schedule of DESIGN.md section 10)
//   bss_coef_kernel         the solutions as the FIR taps of each estimate channel
//   bss_project_kernel      P_all and P_j of every sample (FIRs of K*C*L and C*L taps) and the eight per-sample energies
//                           the four ratios need, summed per task (a piece of one frame segment); nothing but these sums
//                           is written
//   bss_frames_kernel       the task sums of every frame, over the source's channels
//
// Every sum is float64 and reduced in a fixed order (no atomics), so two calls give identical bits.
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/vr_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace vr {
namespace {

constexpr int BR = 16;   // register block: lags per thread (correlation), samples per thread (projection)

// Shared-memory signal layout: 16 doubles, then one pad.  A lane whose 16-sample block starts 16 samples after its
// neighbour's then reads 17 doubles further on, so the 16 lanes of a half-warp hit 16 different bank pairs.
__host__ __device__ constexpr int spad(int p) { return p + (p >> 4); }

// ---- correlations ------------------------------------------------------------------------------------------------
constexpr int CORR_THREADS = 256;             // 8 warps; warp w owns lags lt * CORR_LT + 16 w + [0, 16)
constexpr int CORR_LT = 128;                  // lags per CTA
constexpr int CORR_NB = 4;                    // 16-sample blocks per lane per chunk
constexpr int CORR_TC = 32 * BR * CORR_NB;    // samples per chunk (2048)
constexpr int CORR_GROUPS = 64;               // CTAs along time per (a, b, lag tile): the partial sums kept

// grid: x = lag tile + Lc / CORR_LT * (b + 2M * a), y = time group.  part[g][a][b][Lc].
__global__ void __launch_bounds__(CORR_THREADS, 2)
bss_corr_kernel(const float* __restrict__ refs, const float* __restrict__ ests, int M, int64_t N, int Lc,
                int64_t nchunks, double* __restrict__ part) {
  __shared__ double s_a[spad(CORR_TC)];
  __shared__ double s_y[spad(CORR_TC + CORR_LT)];
  const int ntile = Lc / CORR_LT;
  int bid = blockIdx.x;
  const int lt = bid % ntile;
  bid /= ntile;
  const int b = bid % (2 * M);
  const int a = bid / (2 * M);
  const int g = blockIdx.y, groups = gridDim.y;
  const float* sa = refs + (int64_t)a * N;
  const float* yb = b < M ? refs + (int64_t)b * N : ests + (int64_t)(b - M) * N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t c0 = nchunks * g / groups, c1 = nchunks * (g + 1) / groups;

  double acc[BR];
#pragma unroll
  for (int e = 0; e < BR; ++e) acc[e] = 0.0;
  for (int64_t c = c0; c < c1; ++c) {
    const int64_t t0 = c * CORR_TC;
    const int64_t ty0 = t0 + (int64_t)lt * CORR_LT;
    __syncthreads();
    for (int i = threadIdx.x; i < CORR_TC; i += CORR_THREADS) {
      const int64_t t = t0 + i;
      s_a[spad(i)] = t < N ? (double)sa[t] : 0.0;
    }
    for (int i = threadIdx.x; i < CORR_TC + CORR_LT; i += CORR_THREADS) {
      const int64_t t = ty0 + i;
      s_y[spad(i)] = t < N ? (double)yb[t] : 0.0;
    }
    __syncthreads();
#pragma unroll 1
    for (int nb = 0; nb < CORR_NB; ++nb) {
      const int ub = lane + 32 * nb;                 // this lane's 16-sample block u = t0 + 16 ub + r
      const double* pa = s_a + ub * 17;
      const double* py = s_y + (ub + warp) * 17;     // y(u + lt * 128 + 16 warp + e) = s_y[16 (ub + warp) + r + e]
      double w[2 * BR - 1];
#pragma unroll
      for (int k = 0; k < 2 * BR - 1; ++k) w[k] = py[k + (k >> 4)];
#pragma unroll
      for (int r = 0; r < BR; ++r) {
        const double x = pa[r];
#pragma unroll
        for (int e = 0; e < BR; ++e) acc[e] = fma(x, w[r + e], acc[e]);
      }
    }
  }
#pragma unroll
  for (int e = 0; e < BR; ++e) {
    double v = acc[e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    acc[e] = v;
  }
  if (lane == 0) {
    double* out = part + (((int64_t)g * M + a) * 2 * M + b) * Lc + lt * CORR_LT + warp * BR;
#pragma unroll
    for (int e = 0; e < BR; ++e) out[e] = acc[e];
  }
}

__global__ void bss_corr_reduce_kernel(const double* __restrict__ part, int groups, int64_t total,
                                       double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  double s = 0.0;
  for (int g = 0; g < groups; ++g) s += part[(int64_t)g * total + i];
  out[i] = s;
}

// ---- the linear systems ------------------------------------------------------------------------------------------
constexpr int NB = 64;   // Cholesky tile
// diagonal loading eps = scale * max diag G: first scale, factor between tries, last scale tried
constexpr double BSS_LOADING_FIRST = 0x1p-40, BSS_LOADING_STEP = 0x1p8, BSS_LOADING_LAST = 0x1p-20;
constexpr int CHOL_TILES_SMEM = 2 * NB * (NB + 1) * (int)sizeof(double);

struct AssembleArgs {
  const double* R;    // [M][2M][Lc]
  int K, C, M, L, Lc;
  int np, nbp;        // padded orders of the full system and of one source block (multiples of NB)
  double* G;          // [np][np]
  double* Gb;         // [K][nbp][nbp]
  double* B;          // [np][M]
  double* Bb;         // [K][nbp][C]
  double scale[1 + BSS_EVAL_MAX_SIGNALS];   // eps = scale[s] * max diag G of system s (0: all unknowns, 1 + j: source j)
};

// G[(a, t), (b, t')] = r[a][b](t - t') (r[b][a](t' - t) for negative lags), + eps on the diagonal; rows and columns
// past K*C*L (C*L for a block) are the identity, their right-hand sides zero, so their unknowns solve to zero.
__global__ void bss_assemble_kernel(AssembleArgs p) {
  const int64_t n_g = (int64_t)p.np * p.np, n_gb = (int64_t)p.K * p.nbp * p.nbp;
  const int64_t n_b = (int64_t)p.np * p.M, n_bb = (int64_t)p.K * p.nbp * p.C;
  const int64_t total = n_g + n_gb + n_b + n_bb;
  double dmax = 0.0;
  for (int a = 0; a < p.M; ++a) dmax = fmax(dmax, p.R[((int64_t)a * 2 * p.M + a) * p.Lc]);
  const double eps = dmax * p.scale[0];
  auto corr = [&](int a, int b, int t, int t2) {
    const int l = t - t2;
    return l >= 0 ? p.R[((int64_t)a * 2 * p.M + b) * p.Lc + l] : p.R[((int64_t)b * 2 * p.M + a) * p.Lc - l];
  };
  const int n = p.M * p.L, nb = p.C * p.L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < n_g) {
      const int r = (int)(i / p.np), c = (int)(i % p.np);
      double v;
      if (r >= n || c >= n) v = r == c ? 1.0 : 0.0;
      else v = corr(r / p.L, c / p.L, r % p.L, c % p.L) + (r == c ? eps : 0.0);
      p.G[i] = v;
    } else if (i < n_g + n_gb) {
      const int64_t k = i - n_g;
      const int j = (int)(k / ((int64_t)p.nbp * p.nbp));
      const int64_t q = k % ((int64_t)p.nbp * p.nbp);
      const int r = (int)(q / p.nbp), c = (int)(q % p.nbp);
      double v;
      if (r >= nb || c >= nb) v = r == c ? 1.0 : 0.0;
      else v = corr(j * p.C + r / p.L, j * p.C + c / p.L, r % p.L, c % p.L) + (r == c ? dmax * p.scale[1 + j] : 0.0);
      p.Gb[k] = v;
    } else if (i < n_g + n_gb + n_b) {
      const int64_t k = i - n_g - n_gb;
      const int r = (int)(k / p.M), e = (int)(k % p.M);
      p.B[k] = r < n ? p.R[((int64_t)(r / p.L) * 2 * p.M + p.M + e) * p.Lc + r % p.L] : 0.0;
    } else {
      const int64_t k = i - n_g - n_gb - n_b;
      const int j = (int)(k / ((int64_t)p.nbp * p.C));
      const int64_t q = k % ((int64_t)p.nbp * p.C);
      const int r = (int)(q / p.C), ci = (int)(q % p.C);
      p.Bb[k] = r < nb ? p.R[((int64_t)(j * p.C + r / p.L) * 2 * p.M + p.M + j * p.C + ci) * p.Lc + r % p.L] : 0.0;
    }
  }
}

// Right-looking blocked Cholesky, lower triangle in place, of a batch of n x n row-major matrices (blockIdx.z or x
// selects one, stride n * n).  Step k: factor diagonal tile k, solve the panel below it, update the trailing tiles.
// status[z] receives 1 + the first row whose pivot is not positive (a NaN pivot included) and is left alone otherwise.
__global__ void __launch_bounds__(256) chol_diag_kernel(double* A, int n, int k, int* status) {
  __shared__ double t[NB][NB + 1];
  double* a = A + (int64_t)blockIdx.x * n * n;
  const int r0 = k * NB, tid = threadIdx.x;
  for (int i = tid; i < NB * NB; i += 256) t[i / NB][i % NB] = a[(int64_t)(r0 + i / NB) * n + r0 + i % NB];
  __syncthreads();
  for (int c = 0; c < NB; ++c) {
    const double piv = t[c][c];
    if (tid == 0 && !(piv > 0.0) && status[blockIdx.x] == 0) status[blockIdx.x] = r0 + c + 1;
    const double d = sqrt(piv);   // NaN past a failed pivot: the caller reports the status, never the numbers
    __syncthreads();
    if (tid == 0) t[c][c] = d;
    for (int r = c + 1 + tid; r < NB; r += 256) t[r][c] /= d;
    __syncthreads();
    for (int i = tid; i < NB * NB; i += 256) {
      const int r = i / NB, r2 = i % NB;
      if (r2 > c && r2 <= r) t[r][r2] -= t[r][c] * t[r2][c];
    }
    __syncthreads();
  }
  for (int i = tid; i < NB * NB; i += 256)
    if (i % NB <= i / NB) a[(int64_t)(r0 + i / NB) * n + r0 + i % NB] = t[i / NB][i % NB];
}

// tile row k + 1 + blockIdx.x of column k: X L_kk^T = A_ik, one thread per row
__global__ void __launch_bounds__(NB) chol_panel_kernel(double* A, int n, int k) {
  extern __shared__ double chol_smem[];   // two padded tiles (CHOL_TILES_SMEM bytes)
  double(*l)[NB + 1] = reinterpret_cast<double(*)[NB + 1]>(chol_smem);
  double(*x)[NB + 1] = l + NB;
  double* a = A + (int64_t)blockIdx.y * n * n;
  const int r0 = k * NB, i0 = (k + 1 + blockIdx.x) * NB, tid = threadIdx.x;
  for (int i = tid; i < NB * NB; i += NB) {
    l[i / NB][i % NB] = a[(int64_t)(r0 + i / NB) * n + r0 + i % NB];
    x[i / NB][i % NB] = a[(int64_t)(i0 + i / NB) * n + r0 + i % NB];
  }
  __syncthreads();
  for (int c = 0; c < NB; ++c) {
    const double v = x[tid][c] / l[c][c];
    x[tid][c] = v;
    for (int c2 = c + 1; c2 < NB; ++c2) x[tid][c2] -= v * l[c2][c];
  }
  __syncthreads();
  for (int i = tid; i < NB * NB; i += NB) a[(int64_t)(i0 + i / NB) * n + r0 + i % NB] = x[i / NB][i % NB];
}

// trailing tile (k + 1 + blockIdx.y, k + 1 + blockIdx.x) -= A_ik A_jk^T, lower tiles only; 4 x 4 outputs per thread
__global__ void __launch_bounds__(256) chol_update_kernel(double* A, int n, int k) {
  const int ti = k + 1 + blockIdx.y, tj = k + 1 + blockIdx.x;
  if (tj > ti) return;
  extern __shared__ double chol_smem[];
  double(*sa)[NB + 1] = reinterpret_cast<double(*)[NB + 1]>(chol_smem);
  double(*sb)[NB + 1] = sa + NB;
  double* a = A + (int64_t)blockIdx.z * n * n;
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  for (int i = tid; i < NB * NB; i += 256) {
    sa[i / NB][i % NB] = a[(int64_t)(ti * NB + i / NB) * n + k * NB + i % NB];
    sb[i / NB][i % NB] = a[(int64_t)(tj * NB + i / NB) * n + k * NB + i % NB];
  }
  __syncthreads();
  double acc[4][4] = {};
#pragma unroll 4
  for (int kk = 0; kk < NB; ++kk) {
    double x[4], y[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) x[m] = sa[ty + 16 * m][kk];
#pragma unroll
    for (int q = 0; q < 4; ++q) y[q] = sb[tx + 16 * q][kk];
#pragma unroll
    for (int m = 0; m < 4; ++m)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[m][q] = fma(x[m], y[q], acc[m][q]);
  }
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int q = 0; q < 4; ++q) a[(int64_t)(ti * NB + ty + 16 * m) * n + tj * NB + tx + 16 * q] -= acc[m][q];
}

struct SolveSys {
  const double* L;   // n x n, the factor in the lower triangle
  double* B;         // [n][nr]: right-hand sides in, solutions out
  int n, nr;         // nr <= 8
};
struct SolveArgs {
  SolveSys s[9];
};

// L L^T x = b for one system per CTA: forward then backward substitution, tile by tile.  One warp solves each 64 x 64
// triangle; all warps then update the rest of the right-hand sides.
constexpr int SOLVE_THREADS = 512;
__global__ void __launch_bounds__(SOLVE_THREADS) chol_solve_kernel(SolveArgs args) {
  const SolveSys sys = args.s[blockIdx.x];
  __shared__ double t[NB][NB + 1];
  __shared__ double xb[NB][8];
  const int n = sys.n, nr = sys.nr, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int T = n / NB;
  for (int k = 0; k < T; ++k) {   // forward: L y = b
    const int r0 = k * NB;
    for (int i = tid; i < NB * NB; i += SOLVE_THREADS) t[i / NB][i % NB] = sys.L[(int64_t)(r0 + i / NB) * n + r0 + i % NB];
    for (int i = tid; i < NB * nr; i += SOLVE_THREADS) xb[i / nr][i % nr] = sys.B[(int64_t)(r0 + i / nr) * nr + i % nr];
    __syncthreads();
    if (warp == 0) {
      for (int c = 0; c < NB; ++c) {
        if (lane < nr) xb[c][lane] /= t[c][c];
        __syncwarp();
        for (int i = lane; i < (NB - 1 - c) * nr; i += 32) {
          const int r = c + 1 + i / nr, e = i % nr;
          xb[r][e] -= t[r][c] * xb[c][e];
        }
        __syncwarp();
      }
    }
    __syncthreads();
    for (int i = tid; i < NB * nr; i += SOLVE_THREADS) sys.B[(int64_t)(r0 + i / nr) * nr + i % nr] = xb[i / nr][i % nr];
    for (int r = r0 + NB + warp; r < n; r += SOLVE_THREADS / 32) {
      const double l0 = sys.L[(int64_t)r * n + r0 + lane], l1 = sys.L[(int64_t)r * n + r0 + 32 + lane];
      for (int e = 0; e < nr; ++e) {
        double v = l0 * xb[lane][e] + l1 * xb[lane + 32][e];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) sys.B[(int64_t)r * nr + e] -= v;
      }
    }
    __syncthreads();
  }
  for (int k = T - 1; k >= 0; --k) {   // backward: L^T x = y
    const int r0 = k * NB;
    for (int i = tid; i < NB * NB; i += SOLVE_THREADS) t[i / NB][i % NB] = sys.L[(int64_t)(r0 + i / NB) * n + r0 + i % NB];
    for (int i = tid; i < NB * nr; i += SOLVE_THREADS) xb[i / nr][i % nr] = sys.B[(int64_t)(r0 + i / nr) * nr + i % nr];
    __syncthreads();
    if (warp == 0) {
      for (int c = NB - 1; c >= 0; --c) {
        if (lane < nr) xb[c][lane] /= t[c][c];
        __syncwarp();
        for (int i = lane; i < c * nr; i += 32) {
          const int r = i / nr, e = i % nr;
          xb[r][e] -= t[c][r] * xb[c][e];
        }
        __syncwarp();
      }
    }
    __syncthreads();
    for (int i = tid; i < NB * nr; i += SOLVE_THREADS) sys.B[(int64_t)(r0 + i / nr) * nr + i % nr] = xb[i / nr][i % nr];
    for (int r = tid; r < r0; r += SOLVE_THREADS) {
      double acc[8] = {};
      for (int c = 0; c < NB; ++c) {
        const double l = sys.L[(int64_t)(r0 + c) * n + r];
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (e < nr) acc[e] = fma(l, xb[c][e], acc[e]);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (e < nr) sys.B[(int64_t)r * nr + e] -= acc[e];
    }
    __syncthreads();
  }
}

// the solutions as taps: ca[e][kc][Lp] from the full system, cs[e][c][Lp] from source j's (e = j * C + i), zero past L
__global__ void bss_coef_kernel(const double* __restrict__ X, const double* __restrict__ Xb, int K, int C, int L, int Lp,
                                int nbp, double* __restrict__ ca, double* __restrict__ cs) {
  const int M = K * C;
  const int64_t n_a = (int64_t)M * M * Lp, total = n_a + (int64_t)M * C * Lp;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < n_a) {
      const int tau = (int)(i % Lp), kc = (int)(i / Lp % M), e = (int)(i / Lp / M);
      ca[i] = tau < L ? X[((int64_t)kc * L + tau) * M + e] : 0.0;
    } else {
      const int64_t q = i - n_a;
      const int tau = (int)(q % Lp), c = (int)(q / Lp % C), e = (int)(q / Lp / C);
      const int j = e / C, ci = e % C;
      cs[q] = tau < L ? Xb[(int64_t)j * nbp * C + ((int64_t)c * L + tau) * C + ci] : 0.0;
    }
  }
}

// ---- projection and energies -------------------------------------------------------------------------------------
constexpr int PROJ_THREADS = 256;
constexpr int PROJ_TC = PROJ_THREADS * BR;   // samples per task at most (4096)

template <bool OWN>
__device__ __forceinline__ void fir_block(const double* __restrict__ pw, const double* __restrict__ ca,
                                          const double* __restrict__ cs, double (&pa)[BR], double (&pj)[BR]) {
  double w[2 * BR];
#pragma unroll
  for (int k = 1; k < 2 * BR; ++k) w[k] = pw[k + (k >> 4)];
#pragma unroll
  for (int e = 0; e < BR; ++e) {
    const double c1 = __ldg(ca + e);
    const double c2 = OWN ? __ldg(cs + e) : 0.0;
#pragma unroll
    for (int r = 0; r < BR; ++r) {
      pa[r] = fma(c1, w[r - e + BR], pa[r]);
      if (OWN) pj[r] = fma(c2, w[r - e + BR], pj[r]);
    }
  }
}

// grid: x = task, y = estimate channel e = j * C + i.  Thread b owns samples t = t_start + 16 b + [0, 16).
// part[e][task][8] = sums over the task's samples of s^2, (P_j - s)^2, (shat - s)^2, P_j^2, (P_all - P_j)^2, P_all^2,
// (shat - P_all)^2, shat^2, with s = s_e and shat = shat_e.
__global__ void __launch_bounds__(PROJ_THREADS, 1)
bss_project_kernel(const float* __restrict__ refs, const float* __restrict__ ests, int K, int C, int64_t N, int Lp,
                   const double* __restrict__ coef_all, const double* __restrict__ coef_src,
                   const int64_t* __restrict__ tasks, int ntask, double* __restrict__ part) {
  extern __shared__ double xs[];   // time t_start - Lp + p at spad(p), p < Lp + PROJ_TC
  __shared__ double red[PROJ_THREADS / 32][8];
  const int task = blockIdx.x, e = blockIdx.y, M = K * C, j = e / C;
  const int64_t t_start = tasks[2 * task], t_end = tasks[2 * task + 1];
  const int b = threadIdx.x;
  double pa[BR], pj[BR];
#pragma unroll
  for (int r = 0; r < BR; ++r) pa[r] = pj[r] = 0.0;
  for (int kc = 0; kc < M; ++kc) {
    const float* x = refs + (int64_t)kc * N;
    __syncthreads();
    for (int p = threadIdx.x; p < Lp + PROJ_TC; p += PROJ_THREADS) {
      const int64_t t = t_start - Lp + p;
      xs[spad(p)] = (t >= 0 && t < N) ? (double)x[t] : 0.0;
    }
    __syncthreads();
    const double* ca = coef_all + ((int64_t)e * M + kc) * Lp;
    const bool own = kc / C == j;
    const double* cs = coef_src + ((int64_t)e * C + (own ? kc - j * C : 0)) * Lp;
    // x(t - tau) for t = t_start + 16 b + r, tau = 16 tb + e' sits at p = Lp + 16 (b - tb - 1) + (r - e' + 16)
    if (own) {
#pragma unroll 1
      for (int tb = 0; tb < Lp / BR; ++tb)
        fir_block<true>(xs + (Lp / BR + b - tb - 1) * 17, ca + tb * BR, cs + tb * BR, pa, pj);
    } else {
#pragma unroll 1
      for (int tb = 0; tb < Lp / BR; ++tb)
        fir_block<false>(xs + (Lp / BR + b - tb - 1) * 17, ca + tb * BR, cs, pa, pj);
    }
  }
  double q[8] = {};
  const float* sr = refs + (int64_t)e * N;
  const float* se = ests + (int64_t)e * N;
#pragma unroll
  for (int r = 0; r < BR; ++r) {
    const int64_t t = t_start + (int64_t)BR * b + r;
    if (t < t_end) {
      const double s = sr[t], y = se[t], Pj = pj[r], Pa = pa[r];
      q[0] = fma(s, s, q[0]);
      q[1] = fma(Pj - s, Pj - s, q[1]);
      q[2] = fma(y - s, y - s, q[2]);
      q[3] = fma(Pj, Pj, q[3]);
      q[4] = fma(Pa - Pj, Pa - Pj, q[4]);
      q[5] = fma(Pa, Pa, q[5]);
      q[6] = fma(y - Pa, y - Pa, q[6]);
      q[7] = fma(y, y, q[7]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    double v = q[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    q[i] = v;
  }
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int i = 0; i < 8; ++i) red[threadIdx.x >> 5][i] = q[i];
  __syncthreads();
  if (threadIdx.x < 8) {
    double s = 0.0;
    for (int w = 0; w < PROJ_THREADS / 32; ++w) s += red[w][threadIdx.x];
    part[((int64_t)e * ntask + task) * 8 + threadIdx.x] = s;
  }
}

// frames[j][w][q] = sum over channels i, then over the tasks [lo_w, hi_w) of frame w, of part[j * C + i][task][q]
__global__ void bss_frames_kernel(const double* __restrict__ part, const int64_t* __restrict__ franges, int K, int C,
                                  int64_t nwin, int ntask, double* __restrict__ frames) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * nwin * 8) return;
  const int q = (int)(i % 8);
  const int64_t w = i / 8 % nwin;
  const int j = (int)(i / 8 / nwin);
  double s = 0.0;
  for (int c = 0; c < C; ++c)
    for (int64_t t = franges[2 * w]; t < franges[2 * w + 1]; ++t) s += part[((int64_t)(j * C + c) * ntask + t) * 8 + q];
  frames[i] = s;
}

// flag = 1 if any of the n samples of x or y is NaN or Inf (an integer OR: the result does not depend on the order)
__global__ void bss_finite_kernel(const float* __restrict__ x, const float* __restrict__ y, int64_t n, int* flag) {
  bool bad = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    bad |= !isfinite(x[i]) || !isfinite(y[i]);
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(flag, 1);
}

// ---- host plan ---------------------------------------------------------------------------------------------------
int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

struct Plan {
  int K, C, M, L, Lc, Lp, n, np, nb, nbp, groups;
  int64_t N, window, hop, nwin, nchunks;
  std::vector<int64_t> tasks;     // [ntask][2] sample ranges, each inside one frame segment, in time order
  std::vector<int64_t> franges;   // [nwin][2] task range of each frame
  // workspace offsets (bytes)
  size_t o_part, o_R, o_G, o_Gb, o_B, o_Bb, o_ca, o_cs, o_tasks, o_fr, o_ep, o_frames, o_status, bytes;
};

bool make_plan(int K, int C, int64_t N, int L, int64_t window, int64_t hop, Plan& p, std::string& err) {
  if (K < 1 || C < 1 || K * C > BSS_EVAL_MAX_SIGNALS) {
    err = "bss_eval: K * C must be in [1, " + std::to_string(BSS_EVAL_MAX_SIGNALS) + "] (sources x channels), got K = " +
          std::to_string(K) + ", C = " + std::to_string(C);
    return false;
  }
  if (L < 1 || L > BSS_EVAL_MAX_FILTER) {
    err = "bss_eval: filters_len must be in [1, " + std::to_string(BSS_EVAL_MAX_FILTER) + "], got " + std::to_string(L);
    return false;
  }
  if (window < 1 || hop < 1) {
    err = "bss_eval: window and hop must be positive";
    return false;
  }
  if (N < window) {
    err = "bss_eval: the signals (" + std::to_string(N) + " samples) are shorter than one window (" +
          std::to_string(window) + ")";
    return false;
  }
  p.K = K; p.C = C; p.M = K * C; p.L = L; p.N = N; p.window = window; p.hop = hop;
  p.Lc = (int)round_up(L, CORR_LT);
  p.Lp = (int)round_up(L, BR);
  p.n = p.M * L; p.np = (int)round_up(p.n, NB);
  p.nb = C * L; p.nbp = (int)round_up(p.nb, NB);
  p.nwin = (N - window + hop) / hop;
  p.nchunks = (N + CORR_TC - 1) / CORR_TC;
  p.groups = (int)std::min<int64_t>(CORR_GROUPS, p.nchunks);
  // segments: the pieces the frame starts and ends cut the timeline into; the tasks split the covered ones
  std::vector<int64_t> cuts;
  cuts.reserve(2 * p.nwin);
  for (int64_t w = 0; w < p.nwin; ++w) {
    cuts.push_back(w * hop);
    cuts.push_back(w * hop + window);
  }
  std::sort(cuts.begin(), cuts.end());
  cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
  p.tasks.clear();
  for (size_t m = 0; m + 1 < cuts.size(); ++m) {
    const int64_t a = cuts[m], b = cuts[m + 1];
    const int64_t w = std::min(a / hop, p.nwin - 1);   // the last frame starting at or before a
    if (a >= w * hop + window) continue;               // a gap between frames (hop > window)
    for (int64_t t = a; t < b; t += PROJ_TC) {
      p.tasks.push_back(t);
      p.tasks.push_back(std::min(b, t + PROJ_TC));
    }
  }
  const int64_t ntask = (int64_t)p.tasks.size() / 2;
  if (ntask > 0x7fffffff) {
    err = "bss_eval: too many frame pieces; use a longer hop";
    return false;
  }
  p.franges.resize(2 * p.nwin);
  std::vector<int64_t> starts(ntask);
  for (int64_t i = 0; i < ntask; ++i) starts[i] = p.tasks[2 * i];
  for (int64_t w = 0; w < p.nwin; ++w) {
    p.franges[2 * w] = std::lower_bound(starts.begin(), starts.end(), w * hop) - starts.begin();
    p.franges[2 * w + 1] = std::lower_bound(starts.begin(), starts.end(), w * hop + window) - starts.begin();
  }
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off += (bytes + 255) / 256 * 256;
    return o;
  };
  const int M = p.M;
  p.o_part = take(sizeof(double) * p.groups * M * 2 * M * p.Lc);
  p.o_R = take(sizeof(double) * M * 2 * M * p.Lc);
  p.o_G = take(sizeof(double) * p.np * p.np);
  p.o_Gb = take(sizeof(double) * K * p.nbp * p.nbp);
  p.o_B = take(sizeof(double) * p.np * M);
  p.o_Bb = take(sizeof(double) * K * p.nbp * C);
  p.o_ca = take(sizeof(double) * M * M * p.Lp);
  p.o_cs = take(sizeof(double) * M * C * p.Lp);
  p.o_tasks = take(sizeof(int64_t) * p.tasks.size());
  p.o_fr = take(sizeof(int64_t) * p.franges.size());
  p.o_ep = take(sizeof(double) * M * ntask * 8);
  p.o_frames = take(sizeof(double) * K * p.nwin * 8);
  p.o_status = take(sizeof(int) * (2 + K));   // one per system, then the non-finite input flag
  p.bytes = off;
  return true;
}

bool cuda_ok(cudaError_t e, const char* what, std::string& err) {
  if (e == cudaSuccess) return true;
  err = std::string("bss_eval: ") + what + ": " + cudaGetErrorString(e);
  return false;
}

bool cholesky(double* A, int n, int batch, int* status, cudaStream_t st, std::string& err) {
  const int T = n / NB;
  if (!cuda_ok(cudaFuncSetAttribute(chol_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CHOL_TILES_SMEM),
               "cudaFuncSetAttribute", err) ||
      !cuda_ok(cudaFuncSetAttribute(chol_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CHOL_TILES_SMEM),
               "cudaFuncSetAttribute", err))
    return false;
  for (int k = 0; k < T; ++k) {
    chol_diag_kernel<<<batch, 256, 0, st>>>(A, n, k, status);
    if (k + 1 < T) {
      chol_panel_kernel<<<dim3(T - k - 1, batch), NB, CHOL_TILES_SMEM, st>>>(A, n, k);
      chol_update_kernel<<<dim3(T - k - 1, T - k - 1, batch), 256, CHOL_TILES_SMEM, st>>>(A, n, k);
    }
  }
  return cuda_ok(cudaGetLastError(), "cholesky", err);
}

}  // namespace

int64_t bss_eval_workspace(int K, int C, int64_t N, int L, int64_t window, int64_t hop, std::string& err) {
  Plan p;
  if (!make_plan(K, C, N, L, window, hop, p, err)) return -1;
  return (int64_t)p.bytes;
}

bool bss_eval(const float* refs, const float* ests, int K, int C, int64_t N, int L, int64_t window, int64_t hop,
              void* workspace, int64_t workspace_bytes, double* frames_host, double* corr_host, double* loading_host,
              double* phase_ms, cudaStream_t st, std::string& err) {
  Plan p;
  if (!make_plan(K, C, N, L, window, hop, p, err)) return false;
  if (!refs || !ests || !workspace || !frames_host) {
    err = "bss_eval: null pointer";
    return false;
  }
  if (workspace_bytes < (int64_t)p.bytes) {
    err = "bss_eval: workspace of " + std::to_string(workspace_bytes) + " bytes, " + std::to_string(p.bytes) +
          " needed";
    return false;
  }
  char* ws = (char*)workspace;
  double* part = (double*)(ws + p.o_part);
  double* R = (double*)(ws + p.o_R);
  double* G = (double*)(ws + p.o_G);
  double* Gb = (double*)(ws + p.o_Gb);
  double* B = (double*)(ws + p.o_B);
  double* Bb = (double*)(ws + p.o_Bb);
  double* ca = (double*)(ws + p.o_ca);
  double* cs = (double*)(ws + p.o_cs);
  int64_t* d_tasks = (int64_t*)(ws + p.o_tasks);
  int64_t* d_fr = (int64_t*)(ws + p.o_fr);
  double* ep = (double*)(ws + p.o_ep);
  double* d_frames = (double*)(ws + p.o_frames);
  int* d_status = (int*)(ws + p.o_status);
  const int M = p.M, ntask = (int)(p.tasks.size() / 2);

  cudaEvent_t ev[4] = {};
  if (phase_ms)
    for (auto& e : ev)
      if (!cuda_ok(cudaEventCreate(&e), "cudaEventCreate", err)) return false;
  struct Events {
    cudaEvent_t* e;
    ~Events() {
      for (int i = 0; i < 4; ++i)
        if (e[i]) cudaEventDestroy(e[i]);
    }
  } guard{ev};
  if (phase_ms) cudaEventRecord(ev[0], st);

  if (!cuda_ok(cudaMemcpyAsync(d_tasks, p.tasks.data(), sizeof(int64_t) * p.tasks.size(), cudaMemcpyHostToDevice, st),
               "copy tasks", err) ||
      !cuda_ok(cudaMemcpyAsync(d_fr, p.franges.data(), sizeof(int64_t) * p.franges.size(), cudaMemcpyHostToDevice, st),
               "copy frame ranges", err) ||
      !cuda_ok(cudaMemsetAsync(d_status, 0, sizeof(int) * (2 + K), st), "clear status", err))
    return false;
  bss_finite_kernel<<<1024, 256, 0, st>>>(refs, ests, (int64_t)M * N, d_status + 1 + K);

  // correlations
  bss_corr_kernel<<<dim3(p.Lc / CORR_LT * M * 2 * M, p.groups), CORR_THREADS, 0, st>>>(refs, ests, M, N, p.Lc,
                                                                                      p.nchunks, part);
  const int64_t ncorr = (int64_t)M * 2 * M * p.Lc;
  bss_corr_reduce_kernel<<<(unsigned)((ncorr + 255) / 256), 256, 0, st>>>(part, p.groups, ncorr, R);
  if (!cuda_ok(cudaGetLastError(), "correlation", err)) return false;
  if (phase_ms) cudaEventRecord(ev[1], st);

  // systems: G is only positive semidefinite, so a system whose factorisation fails is assembled and factored again
  // with its loading raised by BSS_LOADING_STEP, up to BSS_LOADING_LAST; the systems that succeeded come out the same
  AssembleArgs aa{R, K, C, M, L, p.Lc, p.np, p.nbp, G, Gb, B, Bb, {}};
  for (int s = 0; s <= K; ++s) aa.scale[s] = BSS_LOADING_FIRST;
  std::vector<int> status(2 + K);
  for (;;) {
    bss_assemble_kernel<<<2048, 256, 0, st>>>(aa);
    if (!cuda_ok(cudaGetLastError(), "assemble", err)) return false;
    if (!cholesky(G, p.np, 1, d_status, st, err) || !cholesky(Gb, p.nbp, K, d_status + 1, st, err)) return false;
    if (!cuda_ok(cudaMemcpyAsync(status.data(), d_status, sizeof(int) * (2 + K), cudaMemcpyDeviceToHost, st),
                 "copy status", err) ||
        !cuda_ok(cudaStreamSynchronize(st), "synchronize", err))
      return false;
    if (status[1 + K]) {
      err = "bss_eval: the references or the estimates hold NaN or Inf";
      return false;
    }
    bool again = false;
    for (int s = 0; s <= K; ++s) {
      if (!status[s]) continue;
      if (aa.scale[s] * BSS_LOADING_STEP > BSS_LOADING_LAST) {
        err = "bss_eval: " + std::string(s == 0 ? "the Gram matrix of all references"
                                                : "the Gram matrix of source " + std::to_string(s - 1) + "'s references") +
              " is not positive definite even with a diagonal loading of 2^-20 of its largest diagonal value (pivot " +
              std::to_string(status[s]) + " of the Cholesky factorisation)";
        return false;
      }
      aa.scale[s] *= BSS_LOADING_STEP;
      again = true;
    }
    if (!again) break;
    if (!cuda_ok(cudaMemsetAsync(d_status, 0, sizeof(int) * (1 + K), st), "clear status", err)) return false;
  }
  if (loading_host)
    for (int s = 0; s <= K; ++s) loading_host[s] = aa.scale[s];
  SolveArgs sa{};
  sa.s[0] = SolveSys{G, B, p.np, M};
  for (int j = 0; j < K; ++j)
    sa.s[1 + j] = SolveSys{Gb + (int64_t)j * p.nbp * p.nbp, Bb + (int64_t)j * p.nbp * C, p.nbp, C};
  chol_solve_kernel<<<1 + K, SOLVE_THREADS, 0, st>>>(sa);
  bss_coef_kernel<<<256, 256, 0, st>>>(B, Bb, K, C, L, p.Lp, p.nbp, ca, cs);
  if (!cuda_ok(cudaGetLastError(), "solve", err)) return false;
  if (phase_ms) cudaEventRecord(ev[2], st);

  // projections and energies
  const size_t smem = sizeof(double) * spad(p.Lp + PROJ_TC);
  // (the longest filter needs more than the default 48 KB; the attribute belongs to the current device)
  if (!cuda_ok(cudaFuncSetAttribute(bss_project_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)(sizeof(double) * spad(BSS_EVAL_MAX_FILTER + PROJ_TC))),
               "cudaFuncSetAttribute", err))
    return false;
  if (ntask > 0) {
    bss_project_kernel<<<dim3(ntask, M), PROJ_THREADS, smem, st>>>(refs, ests, K, C, N, p.Lp, ca, cs, d_tasks, ntask,
                                                                   ep);
  }
  const int64_t nf = (int64_t)K * p.nwin * 8;
  bss_frames_kernel<<<(unsigned)((nf + 255) / 256), 256, 0, st>>>(ep, d_fr, K, C, p.nwin, ntask, d_frames);
  if (!cuda_ok(cudaGetLastError(), "projection", err)) return false;
  if (phase_ms) cudaEventRecord(ev[3], st);

  if (!cuda_ok(cudaMemcpyAsync(frames_host, d_frames, sizeof(double) * nf, cudaMemcpyDeviceToHost, st), "copy frames",
               err))
    return false;
  if (corr_host && !cuda_ok(cudaMemcpy2DAsync(corr_host, sizeof(double) * L, R, sizeof(double) * p.Lc,
                                              sizeof(double) * L, (size_t)M * 2 * M, cudaMemcpyDeviceToHost, st),
                            "copy correlations", err))
    return false;
  if (!cuda_ok(cudaStreamSynchronize(st), "synchronize", err)) return false;
  if (phase_ms) {
    float ms;
    for (int i = 0; i < 3; ++i) {
      cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
      phase_ms[i] = ms;
    }
    cudaEventElapsedTime(&ms, ev[0], ev[3]);
    phase_ms[3] = ms;
  }
  return true;
}

}  // namespace vr
