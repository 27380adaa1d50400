// FLAC encoding (RFC 9639) of float32 stems on the device: the encode behind `--output_format flac` (lib/flac.py drives
// it; oracle/flac_oracle.py decodes the result independently), and the PCM packer behind 24-bit WAV output.
//
// The stream has a fixed block size of 4096 (the last block is shorter), 16 or 24 bits per sample, one or two channels,
// and stays inside the streamable subset: LPC order <= 12, coefficient precision 15 with shift 0..15, Rice partition
// order <= 8, sample-rate and sample-size codes in every frame header.  The sample width BITS is a template parameter
// of both kernels: it sets the quantiser's scale, the element type of pcm (int16 / int32), the subframes' sample bits
// (BITS, and BITS + 1 for the side channel S = L - R, which spans 25 bits at 24), the sample-size code and the size of
// the pack kernel's bit buffer.  Everything downstream of the samples is width-blind: residuals are int32 (an LPC
// residual outside it, or INT32_MIN, which RFC 9639 forbids, rules that predictor out; FIXED order 4 of 25-bit
// samples reaches 29 bits), their zigzag is uint32, and sums of code lengths are 64-bit.
// Two kernels with a host step between them:
//   flac_analyse_kernel  one CTA per frame.  Quantises the frame (clip(rint(x * (2^(BITS-1) - 1))), NaN -> 0) into the
//                        interleaved pcm buffer and shared memory, then codes every signal (L, R, M = (L+R)>>1,
//                        S = L-R for stereo) as CONSTANT, VERBATIM, FIXED 0-4 or LPC 1-12 (Tukey(0.5)-windowed
//                        autocorrelation, Levinson-Durbin in fp64) and prices each predictor exactly: bit-plane counts of
//                        the zigzagged residual per finest partition give sum(u >> k) for every k and partition order,
//                        so the best Rice parameter (4- or 5-bit method) or escape of every partition and the best
//                        partition order are exact.  The channel assignment is the cheapest of the four in exact bits.
//                        Writes the frame's plan: its size in bytes, the subframe codings and each partition's parameter.
//   (host)               exclusive scan of the frame sizes: each frame's byte offset.
//   flac_pack_kernel     one CTA per frame.  Recomputes the chosen residuals, places every code by a block prefix sum
//                        of code lengths, ORs the codes into a shared bit buffer (the bits are disjoint, so the order of
//                        the ORs does not matter), copies the frame to its byte span and appends CRC-8 / CRC-16.
//   pcm_pack_kernel      the quantiser alone: x [channels][n] -> interleaved little-endian 2- or 3-byte PCM, what a WAV
//                        file's data chunk and the STREAMINFO MD5 read.  One thread per 16 samples, 16-byte stores.
// Every reduction is integer or in a fixed order and no float atomics are used: the bytes are the same on every run.
#include <type_traits>

#include "common.cuh"
#include "flac_common.cuh"
#include "kernels.h"

namespace vr {

namespace {

constexpr int kBlock = 4096;          // samples per frame (FLAC_ENCODE_BLOCK in include/vr_b200.h)
constexpr int kThreads = 256;
constexpr int kMaxPorder = 8;
constexpr int kMaxLpc = 12;
constexpr int kLpcPrecision = 15;
constexpr int kPlanInts = 192;        // FLAC_ENCODE_PLAN_INTS
constexpr int kSubBase = 8, kSubInts = 24, kParamBase = 64;
constexpr int kTreeRows = (2 << kMaxPorder) - 1;   // partitions of all orders 0..8
// words of the largest frame: a 16-byte header and two VERBATIM subframes
template <int BITS>
constexpr int kBufWords = (16 * 8 + 2 * (8 + (BITS + 1) * kBlock) + 31) / 32 + 2;
constexpr uint64_t kInf = ~0ull >> 2;

enum Kind { kConstant = 0, kVerbatim = 1, kFixed = 2, kLpc = 3 };

// plan row of a frame (int32): [0] frame bytes, [1] header bytes, [2] channel code, [3] block size,
// subframe c at kSubBase + c * kSubInts: kind, order, partition order, 5-bit Rice method, shift, sample bits,
// subframe bits, then kMaxLpc coefficients; partition parameters as bytes at int kParamBase: [c][256], k or 0x80 | raw
struct Choice {
  int kind, order, porder, rice5;
  uint64_t bits;
};

__host__ __device__ __forceinline__ int utf8_len(int64_t v) {
  if (v < 0x80) return 1;
  int n = 2;
  while (n < 7 && v >= (1ll << (5 * n + 1))) ++n;
  return n;
}

__device__ __forceinline__ int header_bytes(int f, int bs, int rate_code) {
  const int bs_extra = bs == kBlock ? 0 : (bs <= 256 ? 1 : 2);
  return 4 + utf8_len(f) + bs_extra + flac::rate_code_bytes(rate_code) + 1;
}

template <int BITS>
struct Pcm {
  static_assert(BITS == 16 || BITS == 24, "16 or 24 bits per sample");
  using type = typename std::conditional<BITS == 16, int16_t, int32_t>::type;
};

// the integers of every writer: clip(rint(v * (2^(BITS-1) - 1))) with the product rounded once in fp32, NaN -> 0
template <int BITS>
__device__ __forceinline__ typename Pcm<BITS>::type quantise(float v) {
  constexpr float kTop = (float)((1 << (BITS - 1)) - 1);
  if (v != v) return 0;
  const float s = rintf(__fmul_rn(v, kTop));
  return (typename Pcm<BITS>::type)fminf(fmaxf(s, -kTop - 1.0f), kTop);
}

// signal s of a frame from its two channels: 0 L (or mono), 1 R, 2 M = (L + R) >> 1, 3 S = L - R
__device__ __forceinline__ int32_t signal_at(int s, const int32_t* x0, const int32_t* x1, int j) {
  switch (s) {
    case 0: return x0[j];
    case 1: return x1[j];
    case 2: return (x0[j] + x1[j]) >> 1;
    default: return x0[j] - x1[j];
  }
}

// residual of sample j >= order; false when an LPC prediction leaves a residual outside int32 or equal to INT32_MIN
// (not a legal residual, RFC 9639 section 9.2.7.3)
__device__ __forceinline__ bool residual_at(const int32_t* __restrict__ sig, int j, int kind, int order,
                                            const int32_t* __restrict__ coef, int shift, int32_t& r) {
  if (kind == kFixed) {
    const int32_t s0 = sig[j];
    switch (order) {
      case 0: r = s0; break;
      case 1: r = s0 - sig[j - 1]; break;
      case 2: r = s0 - 2 * sig[j - 1] + sig[j - 2]; break;
      case 3: r = s0 - 3 * sig[j - 1] + 3 * sig[j - 2] - sig[j - 3]; break;
      default: r = s0 - 4 * sig[j - 1] + 6 * sig[j - 2] - 4 * sig[j - 3] + sig[j - 4]; break;
    }
    return true;
  }
  int64_t sum = 0;
  for (int i = 0; i < order; ++i) sum += (int64_t)coef[i] * sig[j - 1 - i];
  const int64_t v = (int64_t)sig[j] - (sum >> shift);
  r = (int32_t)v;
  return v == (int64_t)r && r != INT32_MIN;
}

__device__ __forceinline__ uint32_t zigzag(int32_t r) { return ((uint32_t)r << 1) ^ (uint32_t)(r >> 31); }

// finest partition order of a block: the largest p <= 8 with bs divisible by 2^p
__device__ __forceinline__ int finest_porder(int bs) {
  int p = 0;
  while (p < kMaxPorder && (bs & ((2 << p) - 1)) == 0) ++p;
  return p;
}

// cost of one partition of n residuals from its bit-plane counts: 4- or 5-bit Rice parameter (or escape) + codes
__device__ __forceinline__ uint64_t partition_cost(const uint16_t* cnt, int n, int rice5, int* param) {
  const int kmax = rice5 ? 30 : 14, pbits = rice5 ? 5 : 4;
  uint64_t S = 0, best = kInf;
  int width = 0, bk = 0;
  for (int b = 31; b >= 0; --b) {
    S = 2 * S + cnt[b];
    if (!width && cnt[b]) width = b + 1;
    if (b <= kmax) {
      const uint64_t c = S + (uint64_t)(b + 1) * n;
      if (c <= best) { best = c; bk = b; }
    }
  }
  if (width <= 31) {
    const uint64_t esc = 5 + (uint64_t)width * n;
    if (esc < best) { best = esc; bk = 0x80 | width; }
  }
  if (param) *param = bk;
  return best + pbits;
}

struct AnalyseSmem {
  int32_t x[2][kBlock];
  int32_t sig[kBlock];
  union {
    uint32_t tree[kTreeRows * 16];   // uint16 bit-plane counts [row][32], level p at rows 2^p - 1 ..
    double win[kBlock];              // windowed signal for the autocorrelation (fp64, two halves of the tree)
  };
  unsigned long long lvl[kMaxPorder + 1][2];
  double acf[kThreads / 32][kMaxLpc + 1];
  double lev_r[kMaxLpc + 1], lev_a[kMaxLpc + 1], lev_t[kMaxLpc + 1];   // Levinson-Durbin (thread 0)
  int32_t coef[4][kMaxLpc][kMaxLpc];
  int shift[4][kMaxLpc];   // -1: no LPC of that order
  Choice best[4];
  int res_porder, res_rice5;
  uint64_t res_bits;
};

// exact bits of the residual of one predictor (partition order and method chosen), or kInf when it does not fit int32;
// with params, also the chosen partitions' parameters
__device__ __forceinline__ uint64_t price_residual(AnalyseSmem& sm, int bs, int kind, int order, const int32_t* coef, int shift,
                                   int* porder_out, int* rice5_out, uint8_t* params) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int P = finest_porder(bs);
  const int psize = bs >> P;
  uint32_t* fine = sm.tree + ((1 << P) - 1) * 16;
  for (int i = tid; i < (16 << P); i += kThreads) fine[i] = 0;
  if (tid < 2 * (kMaxPorder + 1)) (&sm.lvl[0][0])[tid] = 0;
  __syncthreads();
  bool bad = false;
  for (int j0 = warp * 32; j0 < bs; j0 += kThreads) {
    const int j = j0 + lane;
    uint32_t u = 0;
    if (j >= order && j < bs) {
      int32_t r;
      bad |= !residual_at(sm.sig, j, kind, order, coef, shift, r);
      u = zigzag(r);
    }
    const uint32_t any = __reduce_or_sync(0xffffffffu, u);
    if (!any) continue;
    const int nb = 32 - __clz(any);
    uint32_t mine = 0;   // lane b: which of the 32 samples have bit b set
    for (int b = 0; b < nb; ++b) {
      const uint32_t m = __ballot_sync(0xffffffffu, (u >> b) & 1u);
      if (lane == b) mine = m;
    }
    if (lane < nb && mine) {
      const int last = min(j0 + 31, bs - 1);
      for (int p = j0 / psize; p <= last / psize; ++p) {
        const int lo = max(p * psize - j0, 0), hi = min((p + 1) * psize - j0, 32);
        const uint32_t seg = (hi == 32 ? 0xffffffffu : ((1u << hi) - 1)) & ~((1u << lo) - 1);
        const uint32_t c = __popc(mine & seg);
        if (c) atomicAdd(&fine[p * 16 + (lane >> 1)], c << ((lane & 1) * 16));
      }
    }
  }
  if (__syncthreads_or(bad)) return kInf;
  for (int p = P - 1; p >= 0; --p) {   // coarser orders: each partition is the sum of its two halves
    uint32_t* dst = sm.tree + ((1 << p) - 1) * 16;
    const uint32_t* src = sm.tree + ((2 << p) - 1) * 16;
    for (int i = tid; i < (16 << p); i += kThreads) {
      const int row = i >> 4, w = i & 15;
      dst[i] = src[(2 * row) * 16 + w] + src[(2 * row + 1) * 16 + w];   // uint16 halves: counts <= 4096, no carry
    }
    __syncthreads();
  }
  const uint16_t* cnt = reinterpret_cast<const uint16_t*>(sm.tree);
  for (int item = tid; item < (2 << P) - 1; item += kThreads) {
    const int p = 31 - __clz(item + 1), t = item + 1 - (1 << p);
    const int ps = bs >> p;
    if (ps <= order) continue;   // every partition keeps at least one residual
    const int n = ps - (t == 0 ? order : 0);
    atomicAdd(&sm.lvl[p][0], (unsigned long long)partition_cost(cnt + item * 32, n, 0, nullptr));
    atomicAdd(&sm.lvl[p][1], (unsigned long long)partition_cost(cnt + item * 32, n, 1, nullptr));
  }
  __syncthreads();
  if (tid == 0) {
    uint64_t best = kInf;
    int bp = 0, bm = 0;
    for (int p = 0; p <= P; ++p) {
      if ((bs >> p) <= order) break;
      for (int m = 0; m < 2; ++m)
        if (sm.lvl[p][m] < best) { best = sm.lvl[p][m]; bp = p; bm = m; }
    }
    sm.res_bits = 6 + best;   // method (2) + partition order (4) + partitions
    sm.res_porder = bp;
    sm.res_rice5 = bm;
  }
  __syncthreads();
  const int bp = sm.res_porder, bm = sm.res_rice5;
  const uint64_t bits = sm.res_bits;
  if (params) {
    for (int t = tid; t < (1 << bp); t += kThreads) {
      const int item = (1 << bp) - 1 + t;
      int k;
      partition_cost(cnt + item * 32, (bs >> bp) - (t == 0 ? order : 0), bm, &k);
      params[t] = (uint8_t)k;
    }
  }
  if (porder_out) *porder_out = bp;
  if (rice5_out) *rice5_out = bm;
  __syncthreads();   // the tree and the result are reused by the next call
  return bits;
}

// Tukey(0.5)-windowed autocorrelation of sm.sig and Levinson-Durbin: quantised coefficients of every order 1..12
__device__ __forceinline__ void lpc_analyse(AnalyseSmem& sm, int s, int bs) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int maxo = min(kMaxLpc, bs - 1);
  const double edge = 0.25 * (bs - 1);   // alpha (N - 1) / 2 with alpha = 0.5
  for (int j = tid; j < bs; j += kThreads) {
    double w = 1.0;
    const double d = j < edge ? j : (bs - 1 - j < edge ? bs - 1 - j : edge);
    if (d < edge) w = 0.5 * (1.0 - cospi(d / edge));
    sm.win[j] = w * sm.sig[j];
  }
  __syncthreads();
  double acc[kMaxLpc + 1];
#pragma unroll
  for (int l = 0; l <= kMaxLpc; ++l) acc[l] = 0.0;
  for (int j = tid; j < bs; j += kThreads) {
    const double v = sm.win[j];
#pragma unroll
    for (int l = 0; l <= kMaxLpc; ++l)
      if (j + l < bs) acc[l] = fma(v, sm.win[j + l], acc[l]);
  }
#pragma unroll
  for (int l = 0; l <= kMaxLpc; ++l) {
    double v = acc[l];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sm.acf[warp][l] = v;
  }
  __syncthreads();
  if (tid == 0) {
    double* r = sm.lev_r;
    double* a = sm.lev_a;
    double* tmp = sm.lev_t;
    for (int l = 0; l <= kMaxLpc; ++l) {
      double v = 0.0;
      for (int w = 0; w < kThreads / 32; ++w) v += sm.acf[w][l];
      r[l] = v;
    }
    a[0] = 1.0;
    for (int i = 1; i <= kMaxLpc; ++i) a[i] = 0.0;
    double err = r[0] * (1.0 + 1e-9);
    for (int o = 1; o <= kMaxLpc; ++o) {
      sm.shift[s][o - 1] = -1;
      if (o > maxo || !(err > 0.0)) continue;
      double acc2 = r[o];
      for (int i = 1; i < o; ++i) acc2 += a[i] * r[o - i];
      const double k = -acc2 / err;
      for (int i = 0; i <= o; ++i) tmp[i] = a[i];
      for (int i = 1; i < o; ++i) a[i] = tmp[i] + k * tmp[o - i];
      a[o] = k;
      err *= 1.0 - k * k;
      double amax = 0.0;   // predictor s[j] ~ sum_i c[i] s[j-1-i] with c = -a[1..o]
      for (int i = 1; i <= o; ++i) amax = fmax(amax, fabs(a[i]));
      if (!(amax > 0.0) || !isfinite(amax)) continue;
      const int e = ilogb(amax) + 1;   // amax < 2^e
      const int sh = min(kLpcPrecision - 1 - e, 15);
      if (sh < 0) continue;
      const double lim = (double)(1 << (kLpcPrecision - 1));
      for (int i = 0; i < o; ++i)
        sm.coef[s][o - 1][i] = (int32_t)fmin(fmax(rint(-a[i + 1] * ldexp(1.0, sh)), -lim), lim - 1.0);
      sm.shift[s][o - 1] = sh;
    }
  }
  __syncthreads();
}

__device__ __forceinline__ void load_signal(AnalyseSmem& sm, int s, int bs) {
  for (int j = threadIdx.x; j < bs; j += kThreads) sm.sig[j] = signal_at(s, sm.x[0], sm.x[1], j);
  __syncthreads();
}

// the bits of a FIXED / LPC subframe before its residual
__device__ __forceinline__ uint64_t predictor_bits(int kind, int order, int sb) {
  return 8 + (uint64_t)order * sb + (kind == kLpc ? 4 + 5 + (uint64_t)order * kLpcPrecision : 0);
}

// per-signal best coding (thread 0 writes sm.best[s])
__device__ __forceinline__ void choose_subframe(AnalyseSmem& sm, int s, int bs, int sb) {
  load_signal(sm, s, bs);
  const int32_t first = sm.sig[0];
  bool differs = false;
  for (int j = threadIdx.x; j < bs; j += kThreads) differs |= sm.sig[j] != first;
  if (!__syncthreads_or(differs)) {
    if (threadIdx.x == 0) sm.best[s] = Choice{kConstant, 0, 0, 0, 8 + (uint64_t)sb};
    __syncthreads();
    return;
  }
  Choice best{kVerbatim, 0, 0, 0, 8 + (uint64_t)bs * sb};
  for (int o = 0; o <= 4 && o < bs; ++o) {
    int po, r5;
    const uint64_t rb = price_residual(sm, bs, kFixed, o, nullptr, 0, &po, &r5, nullptr);
    if (rb >= kInf) continue;
    const uint64_t bits = predictor_bits(kFixed, o, sb) + rb;
    if (bits < best.bits) best = Choice{kFixed, o, po, r5, bits};
  }
  if (bs >= 32) {
    lpc_analyse(sm, s, bs);
    for (int o = 1; o <= kMaxLpc; ++o) {
      const int sh = sm.shift[s][o - 1];
      if (sh < 0) continue;
      int po, r5;
      const uint64_t rb = price_residual(sm, bs, kLpc, o, sm.coef[s][o - 1], sh, &po, &r5, nullptr);
      if (rb >= kInf) continue;
      const uint64_t bits = predictor_bits(kLpc, o, sb) + rb;
      if (bits < best.bits) best = Choice{kLpc, o, po, r5, bits};
    }
  }
  if (threadIdx.x == 0) sm.best[s] = best;
  __syncthreads();
}

}  // namespace

template <int BITS>
__global__ void __launch_bounds__(kThreads, 2) flac_analyse_kernel(const float* __restrict__ x, int C, int64_t n,
                                                               int rate_code,
                                                               typename Pcm<BITS>::type* __restrict__ pcm,
                                                               int32_t* __restrict__ plan) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AnalyseSmem& sm = *reinterpret_cast<AnalyseSmem*>(smem_raw);
  const int f = blockIdx.x;
  const int64_t start = (int64_t)f * kBlock;
  const int bs = (int)(n - start < kBlock ? n - start : kBlock);
  for (int c = 0; c < C; ++c)
    for (int j = threadIdx.x; j < bs; j += kThreads) {
      const typename Pcm<BITS>::type q = quantise<BITS>(x[(int64_t)c * n + start + j]);
      sm.x[c][j] = q;
      pcm[(start + j) * C + c] = q;
    }
  __syncthreads();
  const int nsig = C == 2 ? 4 : 1;
  for (int s = 0; s < nsig; ++s) choose_subframe(sm, s, bs, BITS + (s == 3));

  // channel assignment by exact size: independent, left/side, side/right, mid/side
  __shared__ int sig_of[2], ch_code;
  if (threadIdx.x == 0) {
    if (C == 1) {
      ch_code = 0; sig_of[0] = 0; sig_of[1] = 0;
    } else {
      const uint64_t L = sm.best[0].bits, R = sm.best[1].bits, M = sm.best[2].bits, S = sm.best[3].bits;
      uint64_t b = L + R;
      ch_code = 1; sig_of[0] = 0; sig_of[1] = 1;
      if (L + S < b) { b = L + S; ch_code = 8; sig_of[0] = 0; sig_of[1] = 3; }
      if (S + R < b) { b = S + R; ch_code = 9; sig_of[0] = 3; sig_of[1] = 1; }
      if (M + S < b) { b = M + S; ch_code = 10; sig_of[0] = 2; sig_of[1] = 3; }
    }
  }
  __syncthreads();
  int32_t* row = plan + (int64_t)f * kPlanInts;
  uint8_t* params = reinterpret_cast<uint8_t*>(row + kParamBase);
  uint64_t total = 0;
  for (int c = 0; c < C; ++c) {
    const int s = sig_of[c];
    const Choice ch = sm.best[s];
    int32_t* sub = row + kSubBase + c * kSubInts;
    if (ch.kind == kFixed || ch.kind == kLpc) {   // once more for the chosen predictor, to keep its parameters
      load_signal(sm, s, bs);
      const int32_t* coef = ch.kind == kLpc ? sm.coef[s][ch.order - 1] : nullptr;
      const int sh = ch.kind == kLpc ? sm.shift[s][ch.order - 1] : 0;
      price_residual(sm, bs, ch.kind, ch.order, coef, sh, nullptr, nullptr, params + c * 256);
      if (threadIdx.x < kMaxLpc) sub[8 + threadIdx.x] = coef && threadIdx.x < ch.order ? coef[threadIdx.x] : 0;
      if (threadIdx.x == 0) sub[4] = sh;
    } else if (threadIdx.x == 0) {
      sub[4] = 0;
    }
    if (threadIdx.x == 0) {
      sub[0] = ch.kind; sub[1] = ch.order; sub[2] = ch.porder; sub[3] = ch.rice5;
      sub[5] = BITS + (s == 3); sub[6] = (int32_t)ch.bits;
    }
    total += ch.bits;
  }
  if (threadIdx.x == 0) {
    const int hb = header_bytes(f, bs, rate_code);
    row[0] = (int32_t)(hb + (total + 7) / 8 + 2);
    row[1] = hb;
    row[2] = ch_code;
    row[3] = bs;
  }
}

namespace {

template <int BITS>
struct PackSmem {
  int32_t x[2][kBlock];
  int32_t sig[kBlock];
  uint32_t buf[kBufWords<BITS>];
  uint32_t warp_tot[kThreads / 32];
  uint16_t crc_tab[256];
  int32_t row[kPlanInts];
  uint8_t hdr[16];
};

// MSB-first: bits [pos, pos + len) of the buffer get the low len bits of v (1 <= len <= 32)
__device__ __forceinline__ void put_bits(uint32_t* buf, uint64_t pos, uint32_t v, int len) {
  const int off = (int)(pos & 31);
  const uint64_t w = ((uint64_t)(len == 32 ? v : v & ((1u << len) - 1))) << (64 - off - len);
  const uint32_t hi = (uint32_t)(w >> 32), lo = (uint32_t)w;
  if (hi) atomicOr(&buf[pos >> 5], hi);
  if (lo) atomicOr(&buf[(pos >> 5) + 1], lo);
}

// serial writer for the few scalar fields of a frame (one thread)
struct FieldWriter {
  uint32_t* buf;
  uint64_t pos;
  __device__ __forceinline__ void put(uint32_t v, int len) {
    if (len) put_bits(buf, pos, v, len);
    pos += len;
  }
};

}  // namespace

template <int BITS>
__global__ void __launch_bounds__(kThreads, 2) flac_pack_kernel(const typename Pcm<BITS>::type* __restrict__ pcm, int C,
                                                            int64_t n, const int32_t* __restrict__ plan,
                                                            const int64_t* __restrict__ offsets, int rate_code,
                                                            int rate_value, uint8_t* __restrict__ out,
                                                            int32_t* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PackSmem<BITS>& sm = *reinterpret_cast<PackSmem<BITS>*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int f = blockIdx.x;
  const int64_t start = (int64_t)f * kBlock;
  for (int i = tid; i < kPlanInts; i += kThreads) sm.row[i] = plan[(int64_t)f * kPlanInts + i];
  flac::crc16_table(sm.crc_tab);
  __syncthreads();
  const int bytes = sm.row[0], hb = sm.row[1], ch_code = sm.row[2], bs = sm.row[3];
  for (int c = 0; c < C; ++c)
    for (int j = tid; j < bs; j += kThreads) sm.x[c][j] = pcm[(start + j) * C + c];
  const int words = (bytes + 3) / 4 + 1;
  for (int i = tid; i < words; i += kThreads) sm.buf[i] = 0;
  __syncthreads();

  if (tid == 0) {   // frame header and its CRC-8
    uint8_t* h = sm.hdr;
    int k = 0;
    h[k++] = 0xFF;
    h[k++] = 0xF8;
    const int bs_code = bs == kBlock ? flac::kBlockCodeTable4096 : (bs <= 256 ? flac::kBlockCode8Bit : flac::kBlockCode16Bit);
    h[k++] = (uint8_t)((bs_code << 4) | rate_code);
    h[k++] = (uint8_t)((ch_code << 4) | ((BITS == 16 ? flac::kBpsCode16 : flac::kBpsCode24) << 1));
    const int nl = utf8_len(f);
    if (nl == 1) {
      h[k++] = (uint8_t)f;
    } else {
      h[k++] = (uint8_t)((0xFF00 >> nl) | (f >> (6 * (nl - 1))));
      for (int i = nl - 2; i >= 0; --i) h[k++] = (uint8_t)(0x80 | ((f >> (6 * i)) & 0x3F));
    }
    if (bs_code == flac::kBlockCode8Bit) h[k++] = (uint8_t)(bs - 1);
    if (bs_code == flac::kBlockCode16Bit) { h[k++] = (uint8_t)((bs - 1) >> 8); h[k++] = (uint8_t)(bs - 1); }
    const int rb = flac::rate_code_bytes(rate_code);
    for (int i = rb - 1; i >= 0; --i) h[k++] = (uint8_t)(rate_value >> (8 * i));
    uint32_t c8 = 0;
    for (int i = 0; i < k; ++i) c8 = flac::crc8_byte(c8, h[i]);
    h[k++] = (uint8_t)c8;
    FieldWriter fw{sm.buf, 0};
    for (int i = 0; i < k; ++i) fw.put(h[i], 8);
    if (k != hb) status[f] = 1;
  }

  uint64_t base = 8ull * hb;
  bool bad = false;
  for (int c = 0; c < C; ++c) {
    const int32_t* sub = sm.row + kSubBase + c * kSubInts;
    const int kind = sub[0], order = sub[1], porder = sub[2], rice5 = sub[3], shift = sub[4], sb = sub[5];
    const uint8_t* params = reinterpret_cast<const uint8_t*>(sm.row + kParamBase) + c * 256;
    const int s = ch_code == 0 || ch_code == 1 ? c : (ch_code == 8 ? (c ? 3 : 0) : (ch_code == 9 ? (c ? 1 : 3) : (c ? 3 : 2)));
    for (int j = tid; j < bs; j += kThreads) sm.sig[j] = signal_at(s, sm.x[0], sm.x[1], j);
    __syncthreads();
    const uint64_t msk = (1ull << sb) - 1;
    uint64_t res0 = 0;   // first residual bit
    if (tid == 0) {
      FieldWriter fw{sm.buf, base};
      const int type = kind == kConstant ? 0 : kind == kVerbatim ? 1 : kind == kFixed ? 8 + order : 31 + order;
      fw.put(0, 1);
      fw.put(type, 6);
      fw.put(0, 1);
      if (kind == kConstant) fw.put((uint32_t)(sm.sig[0] & msk), sb);
      if (kind == kFixed || kind == kLpc) {
        for (int j = 0; j < order; ++j) fw.put((uint32_t)(sm.sig[j] & msk), sb);
        if (kind == kLpc) {
          fw.put(kLpcPrecision - 1, 4);
          fw.put(shift, 5);
          for (int i = 0; i < order; ++i) fw.put((uint32_t)sub[8 + i] & ((1u << kLpcPrecision) - 1), kLpcPrecision);
        }
        fw.put(rice5, 2);
        fw.put(porder, 4);
      }
      sm.warp_tot[0] = (uint32_t)(fw.pos - base);
    }
    __syncthreads();
    res0 = base + sm.warp_tot[0];
    __syncthreads();
    uint64_t end = res0;
    if (kind == kVerbatim) {
      for (int j = tid; j < bs; j += kThreads) put_bits(sm.buf, base + 8 + (uint64_t)j * sb, (uint32_t)(sm.sig[j] & msk), sb);
      end = base + 8 + (uint64_t)bs * sb;
    } else if (kind == kFixed || kind == kLpc) {
      const int psize = bs >> porder, pbits = rice5 ? 5 : 4;
      const int chunk = (bs + kThreads - 1) / kThreads;
      const int j_lo = min(tid * chunk, bs), j_hi = min(j_lo + chunk, bs);
      const int32_t* coef = sub + 8;
      // code length of residual j (with its partition's parameter field in front of the partition's first residual)
      auto code = [&](int j, int32_t& r, int& k, int& hdr) -> uint32_t {
        bad |= !residual_at(sm.sig, j, kind, order, coef, shift, r);
        const int p = j / psize;
        k = params[p];
        hdr = j == max(order, p * psize) ? pbits + ((k & 0x80) ? 5 : 0) : 0;
        return hdr + ((k & 0x80) ? (k & 0x7F) : (zigzag(r) >> k) + 1 + k);
      };
      uint32_t mine = 0;
      for (int j = max(j_lo, order); j < j_hi; ++j) {
        int32_t r;
        int k, hdr;
        mine += code(j, r, k, hdr);
      }
      uint32_t incl = mine;   // block exclusive scan of the per-thread lengths
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      if (lane == 31) sm.warp_tot[warp] = incl;
      __syncthreads();
      uint64_t pos = res0 + incl - mine, all = 0;
      for (int w = 0; w < kThreads / 32; ++w) {
        if (w < warp) pos += sm.warp_tot[w];
        all += sm.warp_tot[w];
      }
      for (int j = max(j_lo, order); j < j_hi; ++j) {
        int32_t r;
        int k, hdr;
        const uint32_t len = code(j, r, k, hdr);
        if (hdr) {
          put_bits(sm.buf, pos, k & 0x80 ? (1u << pbits) - 1 : (uint32_t)k, pbits);
          if (k & 0x80) put_bits(sm.buf, pos + pbits, k & 0x7F, 5);
        }
        if (k & 0x80) {
          const int raw = k & 0x7F;
          if (raw) put_bits(sm.buf, pos + hdr, (uint32_t)r, raw);
        } else {
          const uint32_t u = zigzag(r);
          put_bits(sm.buf, pos + hdr + (u >> k), (1u << k) | (u & ((1u << k) - 1)), k + 1);
        }
        pos += len;
      }
      end = res0 + all;
      __syncthreads();
    } else {
      end = base + 8 + sb;
    }
    if (end - base != (uint64_t)(uint32_t)sub[6]) bad = true;   // every frame ends where the plan said it would
    base = end;
    __syncthreads();
  }
  if (__syncthreads_or(bad) && tid == 0) status[f] = 2;
  const int body = (int)((base + 7) / 8);
  if (tid == 0 && body + 2 != bytes) status[f] = 3;
  __syncthreads();

  uint8_t* dst = out + offsets[f];
  auto byte_at = [&](int64_t i) { return (sm.buf[i >> 2] >> (24 - 8 * (i & 3))) & 0xFFu; };
  for (int i = tid; i < body; i += kThreads) dst[i] = (uint8_t)byte_at(i);
  if (warp == 0) {
    const uint32_t crc = flac::warp_crc16(body, sm.crc_tab, byte_at);
    if (lane == 0) {
      dst[body] = (uint8_t)(crc >> 8);
      dst[body + 1] = (uint8_t)crc;
    }
  }
}

namespace {

// x [C][n] -> interleaved little-endian PCM of BITS / 8 bytes per sample.  A thread takes 16 consecutive interleaved
// samples, which are BITS / 8 aligned 16-byte words of the output.
template <int BITS>
__global__ void __launch_bounds__(kThreads) pcm_pack_kernel(const float* __restrict__ x, int C, int64_t n,
                                                            uint8_t* __restrict__ out) {
  constexpr int kBytes = BITS / 8;
  const int64_t total = n * C;
  const int64_t i0 = 16 * ((int64_t)blockIdx.x * kThreads + threadIdx.x);
  if (i0 >= total) return;
  auto sample = [&](int64_t t) {   // interleaved index -> quantised sample
    return (uint32_t)(int32_t)quantise<BITS>(C == 1 ? x[t] : x[(t & 1) * n + (t >> 1)]);
  };
  uint8_t* dst = out + i0 * kBytes;
  if (total - i0 < 16) {   // the last, partial group: byte stores
    for (int i = 0; i < (int)(total - i0); ++i) {
      const uint32_t q = sample(i0 + i);
      for (int b = 0; b < kBytes; ++b) dst[kBytes * i + b] = (uint8_t)(q >> (8 * b));
    }
    return;
  }
  uint32_t w[4 * kBytes];
#pragma unroll
  for (int k = 0; k < 4 * kBytes; ++k) w[k] = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const uint32_t q = sample(i0 + i);
#pragma unroll
    for (int b = 0; b < kBytes; ++b) w[(kBytes * i + b) >> 2] |= ((q >> (8 * b)) & 0xFFu) << (8 * ((kBytes * i + b) & 3));
  }
#pragma unroll
  for (int k = 0; k < kBytes; ++k)
    reinterpret_cast<uint4*>(dst)[k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
}

template <int BITS>
cudaError_t analyse(const float* x, int channels, int64_t n, int rate_code, void* pcm, int32_t* plan, int64_t frames,
                    cudaStream_t stream) {
  const int smem = (int)sizeof(AnalyseSmem);
  cudaError_t e = cudaFuncSetAttribute(flac_analyse_kernel<BITS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  flac_analyse_kernel<BITS><<<(unsigned)frames, kThreads, smem, stream>>>(
      x, channels, n, rate_code, static_cast<typename Pcm<BITS>::type*>(pcm), plan);
  return cudaGetLastError();
}

template <int BITS>
cudaError_t pack(const void* pcm, int channels, int64_t n, const int32_t* plan, const int64_t* offsets, int rate_code,
                 int rate_value, uint8_t* out, int32_t* status, int64_t frames, cudaStream_t stream) {
  const int smem = (int)sizeof(PackSmem<BITS>);
  cudaError_t e = cudaFuncSetAttribute(flac_pack_kernel<BITS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  flac_pack_kernel<BITS><<<(unsigned)frames, kThreads, smem, stream>>>(
      static_cast<const typename Pcm<BITS>::type*>(pcm), channels, n, plan, offsets, rate_code, rate_value, out, status);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_flac_encode_analyse(const float* x, int channels, int64_t n, int rate_code, int bits, void* pcm,
                                       int32_t* plan, cudaStream_t stream) {
  if (!x || !pcm || !plan || channels < 1 || channels > 2 || n < 1 || rate_code < 1 || rate_code > 14 ||
      (bits != 16 && bits != 24))
    return cudaErrorInvalidValue;
  const int64_t frames = (n + kBlock - 1) / kBlock;
  if (frames > (1ll << 30)) return cudaErrorInvalidValue;
  return bits == 16 ? analyse<16>(x, channels, n, rate_code, pcm, plan, frames, stream)
                    : analyse<24>(x, channels, n, rate_code, pcm, plan, frames, stream);
}

cudaError_t launch_flac_encode_pack(const void* pcm, int channels, int64_t n, int bits, const int32_t* plan,
                                    const int64_t* offsets, int rate_code, int rate_value, uint8_t* out,
                                    int32_t* status, cudaStream_t stream) {
  if (!pcm || !plan || !offsets || !out || !status || channels < 1 || channels > 2 || n < 1 || rate_code < 1 ||
      rate_code > 14 || (bits != 16 && bits != 24))
    return cudaErrorInvalidValue;
  const int64_t frames = (n + kBlock - 1) / kBlock;
  if (frames > (1ll << 30)) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(status, 0, sizeof(int32_t) * frames, stream);
  if (e != cudaSuccess) return e;
  return bits == 16 ? pack<16>(pcm, channels, n, plan, offsets, rate_code, rate_value, out, status, frames, stream)
                    : pack<24>(pcm, channels, n, plan, offsets, rate_code, rate_value, out, status, frames, stream);
}

cudaError_t launch_pcm_pack(const float* x, int channels, int64_t n, int bits, uint8_t* out, cudaStream_t stream) {
  if (!x || !out || channels < 1 || channels > 2 || n < 1 || (bits != 16 && bits != 24) ||
      (reinterpret_cast<uintptr_t>(out) & 15))
    return cudaErrorInvalidValue;
  const int64_t groups = (n * channels + 15) / 16;
  const int64_t blocks = (groups + kThreads - 1) / kThreads;
  if (blocks > 0x7fffffffll) return cudaErrorInvalidValue;
  if (bits == 16)
    pcm_pack_kernel<16><<<(unsigned)blocks, kThreads, 0, stream>>>(x, channels, n, out);
  else
    pcm_pack_kernel<24><<<(unsigned)blocks, kThreads, 0, stream>>>(x, channels, n, out);
  return cudaGetLastError();
}

}  // namespace vr
