// Bitstream pieces the input decoders (flac.cu, mp3.cu, aac.cu, vorbis.cu) share: the per-frame status word, MSB-first
// and LSB-first readers at absolute bit offsets, 2^(q/4), canonical Huffman books in shared memory, the warp-aggregated
// append of sync candidates and the carving of one device workspace.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace vr {

// Each frame (or packet) leaves one int64 status word: 0 when it decoded, else code << 40 | bit, with the format's
// error code (lib/flac.py, lib/mp3.py and lib/aac.py have the message of each) and the bit offset, within the frame
// or from its first byte, where it was found.  lib/codec.py splits the word again.
__device__ __forceinline__ int64_t frame_status(int64_t code, int64_t bit) { return (code << 40) | (bit & 0xFFFFFFFFFFLL); }

// MSB-first reads at any bit offset of [0, 8 * n) of d; bytes past n read as zero, and a read past ``end`` (the last
// bit the caller's unit may take) is caught by over()
struct PeekBits {
  const uint8_t* __restrict__ d;
  int64_t n, pos, end;
  __device__ __forceinline__ uint32_t peek32() const {
    const int64_t b = pos >> 3;
    uint64_t w = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) w = (w << 8) | (b + k < n ? (uint64_t)__ldg(d + b + k) : 0ull);
    return (uint32_t)(w >> (8 - (pos & 7)));
  }
  __device__ __forceinline__ uint32_t read(int k) {   // 0 <= k <= 24
    if (k == 0) return 0;
    const uint32_t v = peek32() >> (32 - k);
    pos += k;
    return v;
  }
  __device__ __forceinline__ bool over() const { return pos > end; }
};

// LSB-first reads (Vorbis packs bits from the least significant end of each byte) at any bit offset of [0, 8 * n) of
// d; bytes past n read as zero, and a read past ``end`` (the packet's last bit + 1) is caught by over()
struct LsbBits {
  const uint8_t* __restrict__ d;
  int64_t n, pos, end;
  __device__ __forceinline__ uint32_t peek32() const {
    const int64_t b = pos >> 3;
    uint64_t w = 0;
#pragma unroll
    for (int k = 4; k >= 0; --k) w = (w << 8) | (b + k < n ? (uint64_t)__ldg(d + b + k) : 0ull);
    return (uint32_t)(w >> (pos & 7));
  }
  __device__ __forceinline__ uint32_t read(int k) {   // 0 <= k <= 32
    if (k == 0) return 0;
    const uint32_t v = peek32();
    pos += k;
    return k == 32 ? v : v & ((1u << k) - 1u);
  }
  __device__ __forceinline__ bool over() const { return pos > end; }
};

__device__ __forceinline__ float exp2_quarter(int q4) {   // 2^(q4 / 4), exactly rounded for the four fractions
  const int r = q4 & 3;
  const float frac = r == 0 ? 1.0f : r == 1 ? 1.18920711500272f : r == 2 ? 1.41421356237310f : 1.68179283050743f;
  return ldexpf(frac, q4 >> 2);
}

// Canonical Huffman books back to back, book b being entries [start[b], start[b + 1]) in increasing code order: each
// code is the previous one plus one at its own length.  Kept in shared memory with every code left-aligned to 32 bits,
// so that the entry of the next codeword is the last one whose code is at or below the next 32 bits of the stream.
template <typename Sym, int kEntries>
struct HuffBooks {
  uint32_t code[kEntries];
  Sym sym[kEntries];
  uint8_t len[kEntries];

  // the whole block calls it: the symbols and lengths copied, one thread per book assigning its codes
  __device__ __forceinline__ void build(const Sym* syms, const uint8_t* lens, const uint16_t* start, int books) {
    for (int i = threadIdx.x; i < kEntries; i += blockDim.x) {
      sym[i] = syms[i];
      len[i] = lens[i];
    }
    if (threadIdx.x < books) {
      uint32_t c = 0;
      for (int i = start[threadIdx.x]; i < start[threadIdx.x + 1]; ++i) {
        code[i] = c;
        c += 1u << (32 - lens[i]);
      }
    }
    __syncthreads();
  }

  // the entry of [first, last) that the stream codes at br.pos (a binary search whose trip count depends on the book
  // size only); br.pos moves past its codeword
  __device__ __forceinline__ int decode(PeekBits& br, int first, int last) const {
    const uint32_t w = br.peek32();
    int a = first, span = last - first;
    while (span > 1) {
      const int half = span >> 1;
      if (code[a + half] <= w) a += half;
      span -= half;
    }
    br.pos += len[a];
    return a;
  }
};

// One append per warp to a list of ``cap`` slots: one atomicAdd on ``count`` for all the warp's lanes that found
// something.  Every lane of the warp calls it; a lane gets its slot, or -1 when it found nothing or its slot is past
// ``cap`` (the count still includes it, so that the host can retry with room for all).
__device__ __forceinline__ int warp_append(bool found, int* count, int cap) {
  const unsigned mask = __ballot_sync(0xffffffffu, found);
  if (!mask) return -1;
  const int lane = threadIdx.x & 31, leader = __ffs(mask) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(count, __popc(mask));
  base = __shfl_sync(0xffffffffu, base, leader);
  const int slot = base + __popc(mask & ((1u << lane) - 1));
  return found && slot < cap ? slot : -1;
}

// One device workspace cut into 256-byte-aligned slices in the order they are taken; with a null base it only adds up
// ``bytes``, which is how the workspace is sized.
struct Carver {
  uint8_t* base;
  int64_t bytes = 0;
  template <typename T = uint8_t>
  T* take(int64_t n) {
    const int64_t at = bytes;
    bytes += (n + 255) & ~(int64_t)255;
    return base ? reinterpret_cast<T*>(base + at) : nullptr;
  }
};

}  // namespace vr
