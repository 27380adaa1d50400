// FLAC frame decoding (RFC 9639) on the device: the decode in front of the hot path for .flac input
// (lib/flac.py drives it; oracle/flac_oracle.py restates the format independently).
//
// A frame header does not store the frame's length, so decoding takes two kernels and a host step between them:
//   flac_scan_kernel   one thread per byte offset: sync 0xFFF8 / 0xFFF9, header parse, CRC-8; every candidate is
//                      appended (warp-aggregated atomics, unordered) as 4 int64: offset, coded number,
//                      block size | header length << 17 | strategy << 22, byte 2 | byte 3 << 8 | coded rate << 16.
//                      Reserved codes are recorded, not judged: the host rejects them on the frames it chains.
//   (host)             chains the candidates by coded number from the end of the metadata: each frame's byte span
//                      [start, next start) and first sample.
//   flac_decode_kernel one warp per frame.  Lane 0 walks the subframes in order (a subframe starts where the previous
//                      one ends) and stages warm-up samples and residuals as int32 in the frame's slice of the float
//                      output; the 32 lanes check the CRC-16 over the frame's bytes; lane c restores channel c
//                      (FIXED / LPC recurrences, int64 sums, wasted bits); the 32 lanes undo stereo decorrelation and
//                      write float32(x) / 2^(bps-1) over the staged integers.
// Malformed input is data: every read is bounded by the frame's span (bits past it read as zero and fail the frame),
// every write stays in the frame's own samples, and each frame leaves a status word (0, or code << 40 | bit offset in
// the frame) for the host to turn into an error.
#include "bitstream.cuh"
#include "common.cuh"
#include "flac_common.cuh"
#include "kernels.h"

namespace vr {

namespace {

using flac::crc8_byte;

constexpr int kWarpsPerBlock = 4;
constexpr int kMaxChannels = 8;
constexpr int kMaxLpcOrder = 32;

// status codes; lib/flac.py has the message of each
enum FlacError : int64_t {
  kOverrun = 1,         // a read ran past the frame's byte span
  kPadBit = 2,          // subframe padding bit or byte-alignment bits not zero
  kReservedType = 3,    // reserved subframe type
  kOrderTooLarge = 4,   // predictor order larger than the block
  kLpcPrecision = 5,    // LPC precision code 1111
  kLpcShift = 6,        // negative LPC shift
  kResidualMethod = 7,  // reserved residual coding method
  kPartitionOrder = 8,  // partition order does not divide the block or leaves the first partition short
  kRiceOverflow = 9,    // Rice-coded value does not fit 32 bits
  kSampleRange = 10,    // restored sample outside the subframe's bit depth
  kFrameEnd = 11,       // the subframes do not end 2 bytes before the next frame (or the end of the data)
  kCrc16 = 12,          // CRC-16 mismatch
  kFrameShape = 13,     // channel assignment, bit depth or sample span the stream does not have
  kWastedBits = 14,     // wasted bits leave no sample bits
};

// the frame header at byte i (d[i] == 0xFF and d[i+1] is 0xF8 / 0xF9 already); false if it is not one
__device__ bool parse_frame_header(const uint8_t* __restrict__ d, int64_t n, int64_t i, int64_t rec[4]) {
  if (i + 5 > n) return false;
  const uint32_t b2 = d[i + 2], b3 = d[i + 3];
  int64_t p = i + 4;
  uint32_t lead = d[p++];
  int cont;
  uint64_t v;
  if (lead < 0x80) { cont = 0; v = lead; }
  else if ((lead & 0xE0) == 0xC0) { cont = 1; v = lead & 0x1F; }
  else if ((lead & 0xF0) == 0xE0) { cont = 2; v = lead & 0x0F; }
  else if ((lead & 0xF8) == 0xF0) { cont = 3; v = lead & 0x07; }
  else if ((lead & 0xFC) == 0xF8) { cont = 4; v = lead & 0x03; }
  else if ((lead & 0xFE) == 0xFC) { cont = 5; v = lead & 0x01; }
  else if (lead == 0xFE) { cont = 6; v = 0; }
  else return false;
  for (int k = 0; k < cont; ++k) {
    if (p >= n) return false;
    const uint32_t b = d[p++];
    if ((b & 0xC0) != 0x80) return false;
    v = (v << 6) | (b & 0x3F);
  }
  const uint32_t bs_code = b2 >> 4, rate_code = b2 & 15;
  int64_t bs = 0;
  if (bs_code == 1) bs = 192;
  else if (bs_code >= 2 && bs_code <= 5) bs = 576 << (bs_code - 2);
  else if (bs_code == 6 || bs_code == 7) {
    const int k = (int)bs_code - 5;
    if (p + k > n) return false;
    int64_t x = 0;
    for (int j = 0; j < k; ++j) x = (x << 8) | d[p++];
    bs = x + 1;
  } else if (bs_code >= 8) bs = 256 << (bs_code - 8);
  int64_t rate_val = 0;
  if (rate_code >= 12 && rate_code <= 14) {
    const int k = rate_code == 12 ? 1 : 2;
    if (p + k > n) return false;
    for (int j = 0; j < k; ++j) rate_val = (rate_val << 8) | d[p++];
  }
  if (p >= n) return false;
  uint32_t c = 0;
  for (int64_t j = i; j < p; ++j) c = crc8_byte(c, d[j]);
  if (c != d[p]) return false;
  rec[0] = i;
  rec[1] = (int64_t)v;
  rec[2] = bs | ((p + 1 - i) << 17) | ((int64_t)(d[i + 1] & 1) << 22);
  rec[3] = (int64_t)(b2 | (b3 << 8)) | (rate_val << 16);
  return true;
}

// MSB-first bit reader over [.., end): a 64-bit window refilled with whole bytes; bytes at or past `end` read as zero,
// and pos() > 8 * end afterwards tells that the frame ran out
struct BitReader {
  const uint8_t* __restrict__ d;
  int64_t next, end;
  uint64_t cache;
  int nbits;

  __device__ BitReader(const uint8_t* data, int64_t start, int64_t stop) : d(data), next(start), end(stop), cache(0), nbits(0) {}
  __device__ __forceinline__ int64_t pos() const { return next * 8 - nbits; }
  __device__ __forceinline__ void refill() {
    if (next + 8 <= end) {   // whole bytes up to 64 bits from 8 independent loads
      uint64_t w = 0;
#pragma unroll
      for (int b = 0; b < 8; ++b) w = (w << 8) | (uint64_t)__ldg(d + next + b);
      const int nb = (64 - nbits) >> 3;   // >= 1: refill runs with fewer than 57 bits
      cache |= (nb == 8 ? w : w >> (64 - 8 * nb)) << (64 - nbits - 8 * nb);
      next += nb;
      nbits += 8 * nb;
      return;
    }
    while (nbits <= 56) {
      const uint64_t b = next < end ? (uint64_t)__ldg(d + next) : 0ull;
      cache |= b << (56 - nbits);
      ++next;
      nbits += 8;
    }
  }
  __device__ __forceinline__ uint32_t read(int k) {   // 0 <= k <= 32
    if (k == 0) return 0;
    if (nbits < k) refill();
    const uint32_t v = (uint32_t)(cache >> (64 - k));
    cache <<= k;
    nbits -= k;
    return v;
  }
  __device__ __forceinline__ int32_t read_signed(int k) {   // 1 <= k <= 32
    const uint32_t v = read(k);
    return (int32_t)(v << (32 - k)) >> (32 - k);
  }
  // zeros before the next one; the run is taken with __clzll on the window
  __device__ __forceinline__ uint64_t unary() {
    uint64_t q = 0;
    while (true) {
      if (nbits == 0 || cache == 0) {
        q += nbits;
        cache = 0;
        nbits = 0;
        if (next >= end) {   // no one left in the span: consume one bit past it so that pos() reports the overrun
          next = end + 1;
          return q;
        }
        refill();
        continue;
      }
      const int z = __clzll((long long)cache);   // < nbits: the bits below the window are zero
      q += z;
      cache = z + 1 >= 64 ? 0ull : cache << (z + 1);
      nbits -= z + 1;
      return q;
    }
  }
};

struct SubMeta {
  int kind;     // 0 constant, 1 verbatim, 2 fixed, 3 lpc
  int order;
  int shift;
  int wasted;
  int bits;     // sample bits after the wasted bits are removed
  int value;    // CONSTANT value
};

__device__ __forceinline__ bool is_side(int ch_code, int c) {
  return (ch_code == 8 && c == 1) || (ch_code == 9 && c == 0) || (ch_code == 10 && c == 1);
}

// residual of one subframe into dst[order, bs); returns 0 or a status
__device__ int64_t read_residual(BitReader& br, int64_t frame_bit0, int32_t* __restrict__ dst, int bs, int order) {
  const uint32_t method = br.read(2);
  if (method > 1) return frame_status(kResidualMethod, br.pos() - frame_bit0);
  const int pbits = method ? 5 : 4;
  const uint32_t escape = method ? 31u : 15u;
  const int porder = (int)br.read(4);
  const int psize = bs >> porder;
  if ((psize << porder) != bs || psize < order) return frame_status(kPartitionOrder, br.pos() - frame_bit0);
  int j = order;
  for (int p = 0; p < (1 << porder); ++p) {
    const int stop = (p + 1) * psize;
    const uint32_t k = br.read(pbits);
    if (k == escape) {
      const int raw = (int)br.read(5);
      for (; j < stop; ++j) dst[j] = raw ? br.read_signed(raw) : 0;
    } else {
      for (; j < stop; ++j) {
        const uint64_t q = br.unary();
        if (q >> (32 - k)) return frame_status(kRiceOverflow, br.pos() - frame_bit0);
        const uint32_t u = ((uint32_t)q << k) | br.read((int)k);
        dst[j] = (int32_t)(u >> 1) ^ -(int32_t)(u & 1);
      }
    }
    if (br.pos() > 8 * br.end) return frame_status(kOverrun, br.pos() - frame_bit0);
  }
  return 0;
}

// lane 0: every subframe header, warm-up sample and residual of the frame; dst(c) is channel c's staged int32 slice
__device__ int64_t parse_subframes(BitReader& br, int64_t frame_bit0, int32_t* __restrict__ stage, int64_t n, int C,
                                   int ch_code, int bs, int bps, SubMeta* __restrict__ meta,
                                   int32_t (*__restrict__ coef)[kMaxLpcOrder]) {
  for (int c = 0; c < C; ++c) {
    int32_t* dst = stage + (int64_t)c * n;
    const int sub_bps = bps + (is_side(ch_code, c) ? 1 : 0);
    if (br.read(1)) return frame_status(kPadBit, br.pos() - 1 - frame_bit0);
    const int type = (int)br.read(6);
    int wasted = 0;
    if (br.read(1)) {
      const uint64_t w = br.unary() + 1;
      if (w >= (uint64_t)sub_bps) return frame_status(kWastedBits, br.pos() - frame_bit0);
      wasted = (int)w;
    }
    const int eb = sub_bps - wasted;
    SubMeta m{0, 0, 0, wasted, eb, 0};
    if (type == 0) {
      m.kind = 0;
      m.value = br.read_signed(eb);
    } else if (type == 1) {
      m.kind = 1;
      for (int j = 0; j < bs; ++j) dst[j] = br.read_signed(eb);
    } else if ((type >= 8 && type <= 12) || type >= 32) {
      m.kind = type >= 32 ? 3 : 2;
      m.order = type >= 32 ? type - 31 : type - 8;
      if (m.order > bs) return frame_status(kOrderTooLarge, br.pos() - frame_bit0);
      for (int j = 0; j < m.order; ++j) dst[j] = br.read_signed(eb);
      if (m.kind == 3) {
        const int prec = (int)br.read(4) + 1;
        if (prec == 16) return frame_status(kLpcPrecision, br.pos() - 4 - frame_bit0);
        m.shift = br.read_signed(5);
        if (m.shift < 0) return frame_status(kLpcShift, br.pos() - 5 - frame_bit0);
        for (int j = 0; j < m.order; ++j) coef[c][j] = br.read_signed(prec);
      }
      const int64_t e = read_residual(br, frame_bit0, dst, bs, m.order);
      if (e) return e;
    } else {
      return frame_status(kReservedType, br.pos() - 6 - frame_bit0);
    }
    if (br.pos() > 8 * br.end) return frame_status(kOverrun, br.pos() - frame_bit0);
    meta[c] = m;
  }
  return 0;
}

// lane c: turns channel c's staged warm-up + residual into samples in place, then shifts the wasted bits back in.
// Warm-up and VERBATIM samples were read with the subframe's bit depth, so only predicted samples need a range check.
__device__ int64_t restore_channel(int32_t* __restrict__ dst, int bs, const SubMeta& m, const int32_t* __restrict__ coef,
                                   int32_t* __restrict__ hist) {
  const int64_t lo = -(1ll << (m.bits - 1)), hi = (1ll << (m.bits - 1)) - 1;
  if (m.kind == 0) {
    for (int j = 0; j < bs; ++j) dst[j] = (int32_t)((uint32_t)m.value << m.wasted);
    return 0;
  }
  if (m.kind == 2) {
    int64_t s1 = 0, s2 = 0, s3 = 0, s4 = 0;   // s[j-1] .. s[j-4]
    for (int j = 0; j < bs; ++j) {
      int64_t s = dst[j];
      if (j >= m.order) {
        switch (m.order) {
          case 1: s += s1; break;
          case 2: s += 2 * s1 - s2; break;
          case 3: s += 3 * s1 - 3 * s2 + s3; break;
          case 4: s += 4 * s1 - 6 * s2 + 4 * s3 - s4; break;
          default: break;
        }
        if (s < lo || s > hi) return frame_status(kSampleRange, j);
      }
      s4 = s3; s3 = s2; s2 = s1; s1 = s;
      dst[j] = (int32_t)s;
    }
  } else if (m.kind == 3) {   // the last 32 samples live in a shared-memory ring
    for (int j = 0; j < m.order; ++j) hist[j] = dst[j];
    for (int j = m.order; j < bs; ++j) {
      int64_t sum = 0;
      for (int k = 0; k < m.order; ++k) sum += (int64_t)coef[k] * hist[(j - 1 - k) & (kMaxLpcOrder - 1)];
      const int64_t s = (int64_t)dst[j] + (sum >> m.shift);
      if (s < lo || s > hi) return frame_status(kSampleRange, j);
      hist[j & (kMaxLpcOrder - 1)] = (int32_t)s;
      dst[j] = (int32_t)s;
    }
  }
  if (m.wasted)
    for (int j = 0; j < bs; ++j) dst[j] = (int32_t)((uint32_t)dst[j] << m.wasted);
  return 0;
}

}  // namespace

__global__ void __launch_bounds__(256) flac_scan_kernel(const uint8_t* __restrict__ d, int64_t n, int64_t begin,
                                                        int64_t* __restrict__ cands, int max_cands, int* __restrict__ count) {
  const int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t rec[4];
  bool found = false;
  if (i + 1 < n && d[i] == 0xFF && (d[i + 1] & 0xFE) == 0xF8) found = parse_frame_header(d, n, i, rec);
  const int slot = warp_append(found, count, max_cands);
  if (slot < 0) return;
#pragma unroll
  for (int k = 0; k < 4; ++k) cands[(int64_t)slot * 4 + k] = rec[k];
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) flac_decode_kernel(
    const uint8_t* __restrict__ d, int64_t n_bytes, const int64_t* __restrict__ frames, int n_frames, int C, int64_t n,
    float* __restrict__ out, int64_t* __restrict__ status) {
  __shared__ uint16_t crc_tab[256];
  __shared__ SubMeta meta_s[kWarpsPerBlock][kMaxChannels];
  __shared__ int32_t coef_s[kWarpsPerBlock][kMaxChannels][kMaxLpcOrder];
  __shared__ int32_t hist_s[kWarpsPerBlock][kMaxChannels][kMaxLpcOrder];
  flac::crc16_table(crc_tab);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * kWarpsPerBlock + warp;
  if (f >= n_frames) return;
  const int64_t start = frames[4 * f + 0];
  const int64_t end = min(frames[4 * f + 1], n_bytes);
  const int64_t off = frames[4 * f + 2];
  const int64_t info = frames[4 * f + 3];
  const int bs = (int)(info & 0x1FFFF), hlen = (int)((info >> 17) & 0x1F), ch_code = (int)((info >> 24) & 0xF);
  const int bps = (int)((info >> 28) & 0x1F);
  const int nch = ch_code < 8 ? ch_code + 1 : (ch_code <= 10 ? 2 : 0);
  int32_t* stage = reinterpret_cast<int32_t*>(out) + off;

  int64_t err = 0;
  if (nch != C || C > kMaxChannels || bs < 1 || off < 0 || off + bs > n || bps < 4 || bps > 24 || start < 0 ||
      start + hlen >= end)
    err = frame_status(kFrameShape, 0);
  int64_t e = 0;   // the byte after the subframes (where the CRC-16 sits)
  if (!err && lane == 0) {
    BitReader br(d, start + hlen, end);
    const int64_t bit0 = 8 * start;
    err = parse_subframes(br, bit0, stage, n, C, ch_code, bs, bps, meta_s[warp], coef_s[warp]);
    if (!err) {
      const int pad = (int)((8 - (br.pos() & 7)) & 7);
      if (br.read(pad)) err = frame_status(kPadBit, br.pos() - bit0);
      e = br.pos() >> 3;
      if (!err && e + 2 != end) err = frame_status(kFrameEnd, 8 * e - bit0);
    }
  }
  err = __shfl_sync(0xffffffffu, err, 0);
  e = __shfl_sync(0xffffffffu, e, 0);
  __syncwarp();   // lane 0's staged samples are visible to the other lanes

  if (!err) {   // CRC-16 of [start, e)
    const uint8_t* fr = d + start;
    const uint32_t r = flac::warp_crc16(e - start, crc_tab, [&](int64_t v) { return (uint32_t)__ldg(fr + v); });
    const uint32_t want = ((uint32_t)__ldg(d + e) << 8) | __ldg(d + e + 1);
    if (r != want) err = frame_status(kCrc16, 8 * (e - start));
  }

  if (!err) {
    int64_t lerr = 0;
    if (lane < C) lerr = restore_channel(stage + (int64_t)lane * n, bs, meta_s[warp][lane], coef_s[warp][lane],
                                         hist_s[warp][lane]);
    const unsigned bad = __ballot_sync(0xffffffffu, lerr != 0);
    if (bad) err = __shfl_sync(0xffffffffu, lerr, __ffs(bad) - 1);
    __syncwarp();
  }

  if (!err) {
    const float scale = __int_as_float((127 - (bps - 1)) << 23);   // 2^-(bps-1)
    if (C == 2 && ch_code >= 8) {
      int32_t* s0 = stage;
      int32_t* s1 = stage + n;
      for (int j = lane; j < bs; j += 32) {
        const int32_t a = s0[j], b = s1[j];
        int32_t l, r;
        if (ch_code == 8) { l = a; r = a - b; }
        else if (ch_code == 9) { l = a + b; r = b; }
        else {
          const int32_t m = (int32_t)(((uint32_t)a << 1) | (uint32_t)(b & 1));
          l = (m + b) >> 1;
          r = (m - b) >> 1;
        }
        reinterpret_cast<float*>(s0)[j] = (float)l * scale;
        reinterpret_cast<float*>(s1)[j] = (float)r * scale;
      }
    } else {
      for (int c = 0; c < C; ++c) {
        int32_t* s = stage + (int64_t)c * n;
        for (int j = lane; j < bs; j += 32) reinterpret_cast<float*>(s)[j] = (float)s[j] * scale;
      }
    }
  }
  if (lane == 0) status[f] = err;
}

cudaError_t launch_flac_scan(const uint8_t* data, int64_t n_bytes, int64_t begin, int64_t* cands, int max_cands,
                             int* count, cudaStream_t stream) {
  if (!data || !cands || !count || n_bytes < 0 || begin < 0 || max_cands < 0) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(count, 0, sizeof(int), stream);
  if (e != cudaSuccess) return e;
  if (begin >= n_bytes) return cudaSuccess;
  const int64_t threads = n_bytes - begin;
  flac_scan_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(data, n_bytes, begin, cands, max_cands, count);
  return cudaGetLastError();
}

cudaError_t launch_flac_decode(const uint8_t* data, int64_t n_bytes, const int64_t* frames, int n_frames, int channels,
                               int64_t n_samples, float* out, int64_t* status, cudaStream_t stream) {
  if (!data || !frames || !out || !status || n_frames < 0 || channels < 1 || channels > kMaxChannels || n_samples < 0)
    return cudaErrorInvalidValue;
  if (n_frames == 0) return cudaSuccess;
  flac_decode_kernel<<<(n_frames + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, 0, stream>>>(
      data, n_bytes, frames, n_frames, channels, n_samples, out, status);
  return cudaGetLastError();
}

}  // namespace vr
