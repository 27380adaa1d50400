// FLAC (RFC 9639) pieces shared by the device decoder (flac.cu) and encoder (flac_encode.cu): the header CRC-8, the
// frame CRC-16 table and its 32-lane combine, and the header codes both sides read or write.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vr {
namespace flac {

constexpr int kBpsCode16 = 4;   // sample-size code of 16 bits per sample
constexpr int kBlockCodeTable4096 = 12;   // block-size code 256 << (12 - 8) = 4096
constexpr int kBlockCode8Bit = 6;         // block size - 1 in one byte after the coded number
constexpr int kBlockCode16Bit = 7;        // block size - 1 in two bytes
// sample-rate codes 12 / 13 / 14: the rate in kHz (1 byte), in Hz (2 bytes), in tens of Hz (2 bytes) after the header
__host__ __device__ __forceinline__ int rate_code_bytes(int rate_code) {
  return rate_code == 12 ? 1 : (rate_code == 13 || rate_code == 14 ? 2 : 0);
}

// CRC-8 of the frame header: poly x^8 + x^2 + x + 1, init 0, not reflected
__device__ __forceinline__ uint32_t crc8_byte(uint32_t c, uint32_t b) {
  c ^= b;
#pragma unroll
  for (int i = 0; i < 8; ++i) c = (c & 0x80) ? ((c << 1) ^ 0x07) & 0xFF : (c << 1) & 0xFF;
  return c;
}

// CRC-16 of the frame (poly 0x8005, init 0, not reflected): the byte table, filled by the whole block
__device__ __forceinline__ void crc16_table(uint16_t* tab) {
  for (int b = threadIdx.x; b < 256; b += blockDim.x) {
    uint32_t c = (uint32_t)b << 8;
    for (int k = 0; k < 8; ++k) c = (c & 0x8000) ? ((c << 1) ^ 0x8005) : (c << 1);
    tab[b] = (uint16_t)c;
  }
}

// CRC-16 of the L bytes byte(0) .. byte(L-1), one full warp: lane t takes one chunk of the message left-padded with
// zeros to 32 chunks (leading zeros leave a CRC with init 0 unchanged); the chunk CRCs are combined in lane order by the
// 16x16 matrix that advances a CRC over one chunk of zero bytes.  Every lane returns the CRC.
template <typename ByteAt>
__device__ __forceinline__ uint32_t warp_crc16(int64_t L, const uint16_t* __restrict__ tab, ByteAt byte) {
  const int lane = threadIdx.x & 31;
  const int64_t chunk = (L + 31) / 32, pad = 32 * chunk - L;
  uint32_t c = 0, col = lane < 16 ? 1u << lane : 0u;   // col: bit `lane` advanced over `chunk` zero bytes
  for (int64_t v = lane * chunk; v < (lane + 1) * chunk; ++v) {
    if (v >= pad) c = ((c << 8) & 0xFFFF) ^ tab[(c >> 8) ^ byte(v - pad)];
    col = ((col << 8) & 0xFFFF) ^ tab[col >> 8];
  }
  uint32_t cols[16];
#pragma unroll
  for (int b = 0; b < 16; ++b) cols[b] = __shfl_sync(0xffffffffu, col, b);
  uint32_t r = 0;
  for (int t = 0; t < 32; ++t) {
    uint32_t a = 0;
#pragma unroll
    for (int b = 0; b < 16; ++b) a ^= ((r >> b) & 1u) ? cols[b] : 0u;
    r = a ^ __shfl_sync(0xffffffffu, c, t);
  }
  return r;
}

}  // namespace flac
}  // namespace vr
