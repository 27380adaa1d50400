// Raw-PTX device helpers shared by the wgmma convolution kernels (mbarrier rings, TMA, GMMA descriptors, wgmma) and
// their epilogue.
#pragma once
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

#include "common.cuh"

namespace vr {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// one lane of a converged warp (the CUTLASS elect_one_sync idiom): keeps the surrounding code warp-uniform
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "elect.sync _|P1, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Spin on an mbarrier phase: the bare try_wait loop (a poll counter + trap on the hot path costs throughput).
// -DVR_WAIT_TIMEOUT builds the trapping variant for bring-up of new pipelines (a barrier bug then aborts the kernel
// after ~2^28 polls instead of hanging the GPU).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
#ifdef VR_WAIT_TIMEOUT
  asm volatile(
      "{\n\t"
      ".reg .pred p, q;\n\t"
      ".reg .u32 n;\n\t"
      "mov.u32 n, 0;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.lt.u32 q, n, 0x10000000;\n\t"
      "@q bra WAIT_LOOP;\n\t"
      "trap;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(bar),
      "r"(parity)
      : "memory");
#else
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(bar),
      "r"(parity)
      : "memory");
#endif
}
// __syncwarp, then one arrive for the warp (an empty barrier counts one arrive per consumer warp)
__device__ __forceinline__ void warp_arrive(uint32_t bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}

// A ring of shared-memory slots [lo, hi) guarded by two mbarrier arrays: full[s] completes once slot s has been filled
// (the TMA transaction bytes, or one arrive per producer warp), empty[s] once every consumer warp has released it (one
// arrive each).  Every role keeps
// its own copy and walks the slots in the same order: the producer waits for a slot's empty phase, fills it and moves
// on; a consumer waits for its full phase, reads it, releases it and moves on.  `phase` is the parity of the slot's
// current use.  It flips each time the ring wraps, and the producer's first pass waits on the parity before the
// initial one, which a fresh barrier reports complete.
struct MbarRing {
  uint32_t full0, empty0;   // shared addresses of full[0] and empty[0]
  int lo, hi, slot;
  uint32_t phase;

  __device__ __forceinline__ MbarRing(uint32_t full0_, uint32_t empty0_, int lo_, int hi_)
      : full0(full0_), empty0(empty0_), lo(lo_), hi(hi_), slot(lo_), phase(0) {}
  __device__ __forceinline__ uint32_t full(int s) const { return full0 + (uint32_t)s * 8u; }
  __device__ __forceinline__ uint32_t empty(int s) const { return empty0 + (uint32_t)s * 8u; }
  __device__ __forceinline__ uint32_t full() const { return full(slot); }
  __device__ __forceinline__ uint32_t empty() const { return empty(slot); }
  __device__ __forceinline__ void wait_full() const { mbar_wait(full(), phase); }
  __device__ __forceinline__ void wait_empty() const { mbar_wait(empty(), phase ^ 1u); }
  __device__ __forceinline__ void advance() {
    if (++slot == hi) {
      slot = lo;
      phase ^= 1u;
    }
  }
  // one thread, before the block's first barrier: the barriers of every slot of the ring
  __device__ __forceinline__ void init(uint32_t full_count, uint32_t empty_count) const {
    for (int s = lo; s < hi; ++s) {
      mbar_init(full(s), full_count);
      mbar_init(empty(s), empty_count);
    }
  }
};

// The slot of a ring whose last wgmma group may still be in flight.  A consumer holds it once it has committed that
// group.  release() after the wg_wait<1> that follows the next commit hands it back; release_last() after the
// wg_wait<0> at the end of a tile hands back the last one.  Every tile commits at least one group, so a slot is always
// held there.  A slot that no wgmma reads (an A slot read with ldmatrix) is released right after its last ldmatrix
// instead, with warp_arrive.
struct HeldSlot {
  int slot = -1;
  __device__ __forceinline__ void hold(const MbarRing& r) { slot = r.slot; }
  __device__ __forceinline__ void release(const MbarRing& r, int lane) {
    if (slot >= 0) {
      warp_arrive(r.empty(slot), lane);
      slot = -1;
    }
  }
  __device__ __forceinline__ void release_last(const MbarRing& r, int lane) {
    warp_arrive(r.empty(slot), lane);
    slot = -1;
  }
};

__device__ __forceinline__ void tma_prefetch(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            int c4, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, "
      "%6}], [%7];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2,
                                            uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], "
      "[%5];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}

// sm_90 GMMA shared-memory matrix descriptor of a K-major, swizzled operand, split into its two 32-bit words:
//   low word:  start address >> 4 [0,14), leading-byte offset >> 4 [16,30) (unused for swizzled K-major: 1)
//   high word: stride-byte offset >> 4 [0,14) (= 8 rows of the tile), layout [30,32): 1 = 128B, 2 = 64B, 3 = 32B swizzle
// Advancing a tile by `bytes` is one 32-bit add of bytes>>4 on the low word (shared memory addresses are < 2^18).
__device__ __forceinline__ uint32_t desc_lo(uint32_t addr) { return ((addr & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ uint32_t desc_hi(uint32_t sbo_bytes, uint32_t layout_type) {
  return (sbo_bytes >> 4) | (layout_type << 30);
}
__device__ __forceinline__ uint64_t desc64(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory");
}

// D[64][N] += A[64][16] * B[N][16]^T: bf16 operands from shared memory (both K-major), fp32 accumulator fragment d[N/2]
// in registers.  Thread t of the warpgroup holds rows m = 16*(t/32) + (t%32)/4 and m + 8, columns 8j + 2*(t%4) + {0,1}:
// d[4j + {0,1}] for row m, d[4j + {2,3}] for row m + 8.
template <int N>
struct Wgmma;
template <>
struct Wgmma<16> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 1, 1, 1, 0, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b)
        : "memory");
  }
};
template <>
struct Wgmma<32> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1, 1, 1, 0, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b)
        : "memory");
  }
};
template <>
struct Wgmma<48> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, 1, 1, 1, 0, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(a), "l"(b)
        : "memory");
  }
};
template <>
struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, 0, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b)
        : "memory");
  }
};
template <>
struct Wgmma<80> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, 1, 1, 1, 0, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
        : "l"(a), "l"(b)
        : "memory");
  }
};
template <>
struct Wgmma<96> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, 1, 1, 1, 0, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(a), "l"(b)
        : "memory");
  }
};
template <>
struct Wgmma<112> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, 1, 1, 1, 0, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
        : "l"(a), "l"(b)
        : "memory");
  }
};
template <>
struct Wgmma<128> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, 0, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b)
        : "memory");
  }
};
// The three split-precision products of one 16-channel k-step, hi*hi + lo*hi + hi*lo, into one accumulator
template <int N>
__device__ __forceinline__ void wgmma_split3(float* d, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                             uint32_t dhi) {
  Wgmma<N>::mma(d, desc64(a_hi, dhi), desc64(b_hi, dhi));
  Wgmma<N>::mma(d, desc64(a_lo, dhi), desc64(b_hi, dhi));
  Wgmma<N>::mma(d, desc64(a_hi, dhi), desc64(b_lo, dhi));
}

// D[64][N] += A[64][16] * B[N][16]^T with A from registers: a[4] is the m16n8k16-style fragment of the warp's 16 rows
// (rows m, m + 8 at channels 2*(t%4) + {0,1} and + 8), as ldmatrix.x4 of the 16 x 16 tile returns it; B as above.
template <int N>
struct WgmmaRS;
template <>
struct WgmmaRS<16> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
        : "memory");
  }
};
template <>
struct WgmmaRS<32> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
        : "memory");
  }
};
template <>
struct WgmmaRS<48> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
        : "memory");
  }
};
template <>
struct WgmmaRS<64> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
        : "memory");
  }
};
template <>
struct WgmmaRS<96> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, {%48, %49, %50, %51}, %52, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
        : "memory");
  }
};
template <>
struct WgmmaRS<128> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
        : "memory");
  }
};
// The same three products with the A operands held in registers (a_hi[4], a_lo[4])
template <int N>
__device__ __forceinline__ void wgmma_split3_rs(float* d, const uint32_t* a_hi, const uint32_t* a_lo, uint32_t b_hi,
                                                uint32_t b_lo, uint32_t dhi) {
  WgmmaRS<N>::mma(d, a_hi, desc64(b_hi, dhi));
  WgmmaRS<N>::mma(d, a_lo, desc64(b_hi, dhi));
  WgmmaRS<N>::mma(d, a_hi, desc64(b_lo, dhi));
}

// four 8x8 bf16 matrices from shared memory: lane l supplies the address of row l % 8 of matrix l / 8
__device__ __forceinline__ void ldsm_x4(uint32_t* r, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}

// per-thread register budget of the executing warpgroup (every thread of the warpgroup executes it)
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// The epilogue applies the activation as y = max(v,0) + slope*min(v,0), branch-free: slope 0 = ReLU, 0.01 = LeakyReLU,
// 1 = identity.
__device__ __forceinline__ float act_slope(int act) { return act == ACT_RELU ? 0.f : act == ACT_LEAKY ? 0.01f : 1.f; }

// bias + activation + split-bf16 store of the two adjacent channels (c, c + 1) a thread holds of one pixel
__device__ __forceinline__ void epilogue_pair(float v0, float v1, const float* bias_s, int c, int Cout, float slope,
                                              bf16* out_hi, bf16* out_lo) {
  if (c >= Cout) return;
  const float t0 = v0 + bias_s[c], t1 = v1 + bias_s[c + 1];
  const float y0 = fmaxf(t0, 0.f) + slope * fminf(t0, 0.f);
  const float y1 = fmaxf(t1, 0.f) + slope * fminf(t1, 0.f);
  bf16* h = out_hi + c;
  bf16* l = out_lo + c;
  if (c + 1 < Cout && ((reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(l)) & 3) == 0) {
    const uint32_t uh = f2_to_bf2(y0, y1);
    const float2 hf = bf2_to_f2(uh);
    *reinterpret_cast<uint32_t*>(h) = uh;
    *reinterpret_cast<uint32_t*>(l) = f2_to_bf2(y0 - hf.x, y1 - hf.y);
  } else {
    split_bf16(y0, h[0], l[0]);
    if (c + 1 < Cout) split_bf16(y1, h[1], l[1]);
  }
}

// bias + activation + split into bf16 hi / lo of the channel pair (c, c + 1) a thread holds: epilogue_pair's arithmetic
__device__ __forceinline__ void act_split2(float v0, float v1, const float* bias_s, int c, float slope, uint32_t& hi,
                                           uint32_t& lo) {
  const float t0 = v0 + bias_s[c], t1 = v1 + bias_s[c + 1];
  const float y0 = fmaxf(t0, 0.f) + slope * fminf(t0, 0.f);
  const float y1 = fmaxf(t1, 0.f) + slope * fminf(t1, 0.f);
  hi = f2_to_bf2(y0, y1);
  const float2 hf = bf2_to_f2(hi);
  lo = f2_to_bf2(y0 - hf.x, y1 - hf.y);
}

// The destination of one thread's two pixels of a 64-pixel accumulator block: the fragment rows m and m + 8 (pixel
// halves hr = 0 / 1) at element offsets obase[hr] of the output planes, stored where keep[hr]; channel c0 + c of the
// block is channel c of the pixel's slice, and those at or past Cout do not exist.  vec16: the planes are 16-byte
// aligned and the strides multiples of 8 channels.
struct EpiDest {
  bf16* out_hi;
  bf16* out_lo;
  int64_t obase[2];
  bool keep[2];
  int c0, Cout;
  bool vec16;
};

// One set of four (pixel half, 8-channel group) slots of the block: SPLIT = false, groups j0 .. j0 + 3 of pixel half hr;
// SPLIT = true, groups j0 and j0 + 1 of both halves.  With 16-byte stores every lane of the quad that shares the pixels
// computes its channel pair of each slot, the quad transposes them with four shuffles (every lane takes part) so that
// lane q holds the 8 consecutive channels of slot q, and lane q stores them with one 16-byte store per plane if its
// group lies below Cout.  A set with a group that straddles Cout, or a launch without vec16, takes epilogue_pair.
template <bool SPLIT>
__device__ __forceinline__ void epilogue_set(const float* v, const float* bias_s, float slope, int lane,
                                             const EpiDest& d, int hr, int j0) {
  const int q = lane & 3;
  bool straddle = false;   // warp-uniform, as the shuffles need
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    const int c = d.c0 + 8 * (SPLIT ? j0 + (s & 1) : j0 + s);
    straddle |= c < d.Cout && c + 8 > d.Cout;
  }
  if (d.vec16 && !straddle) {
    uint32_t hi[4], lo[4], oh[4], ol[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int j = SPLIT ? j0 + (s & 1) : j0 + s, h = SPLIT ? s >> 1 : hr;
      act_split2(v[4 * j + 2 * h], v[4 * j + 2 * h + 1], bias_s, d.c0 + 8 * j + 2 * q, slope, hi[s], lo[s]);
    }
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int gs = (q + s) & 3, src = (q - s) & 3;   // send slot gs, receive slot q from lane src
      const uint32_t sh = gs == 0 ? hi[0] : gs == 1 ? hi[1] : gs == 2 ? hi[2] : hi[3];
      const uint32_t sl = gs == 0 ? lo[0] : gs == 1 ? lo[1] : gs == 2 ? lo[2] : lo[3];
      const uint32_t rh = __shfl_sync(0xffffffffu, sh, (lane & ~3) | src);
      const uint32_t rl = __shfl_sync(0xffffffffu, sl, (lane & ~3) | src);
#pragma unroll
      for (int g = 0; g < 4; ++g)
        if (src == g) {
          oh[g] = rh;
          ol[g] = rl;
        }
    }
    const int h = SPLIT ? q >> 1 : hr;
    const int c = d.c0 + 8 * (SPLIT ? j0 + (q & 1) : j0 + q);
    if ((h ? d.keep[1] : d.keep[0]) && c + 8 <= d.Cout) {
      const int64_t o = (h ? d.obase[1] : d.obase[0]) + c;
      *reinterpret_cast<uint4*>(d.out_hi + o) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
      *reinterpret_cast<uint4*>(d.out_lo + o) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
    }
  } else {
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int j = SPLIT ? j0 + (s & 1) : j0 + s, h = SPLIT ? s >> 1 : hr;
      if (h ? d.keep[1] : d.keep[0]) {
        const int64_t o = h ? d.obase[1] : d.obase[0];
        epilogue_pair(v[4 * j + 2 * h], v[4 * j + 2 * h + 1], bias_s, d.c0 + 8 * j + 2 * (lane & 3), d.Cout, slope,
                      d.out_hi + o, d.out_lo + o);
      }
    }
  }
}

// The store of one pixel with 8-byte stores, for the variants that have no registers to spare for epilogue_store's
// transposes.  v: this lane's accumulators of the pixel (channels c0 + 8 j + 2 (lane % 4) + {0, 1} in v[4 j], v[4 j + 1]),
// out_hi / out_lo: the pixel's channel 0.  For each pair of groups j, j + 1 the lanes q and q ^ 1 swap one channel pair
// (one shuffle per plane): an even lane then holds channels 2 q .. 2 q + 3 of group j, an odd lane channels
// 2 (q - 1) .. 2 q + 1 of group j + 1, and each writes its four with one 8-byte store per plane.  The quad so writes the
// 16 channels of both groups, 32 bytes per plane, in one instruction instead of four half-sector ones.  The store rules
// and the values are those of epilogue_store: a lane stores only where its group lies below Cout, and a pair with a
// group straddling Cout, or a launch without vec16, takes epilogue_pair.
template <int BN>
__device__ __forceinline__ void epilogue_pixel8(const float* v, const float* bias_s, int c0, int Cout, float slope,
                                                int lane, bf16* out_hi, bf16* out_lo, bool vec16) {
  const int q = lane & 3;
  const bool odd = q & 1;
#pragma unroll
  for (int j = 0; j < BN / 8; j += 2) {
    const int cj = c0 + 8 * j;
    const bool straddle = (cj < Cout && cj + 8 > Cout) || (cj + 8 < Cout && cj + 16 > Cout);   // warp-uniform
    if (vec16 && !straddle) {
      uint32_t h0, l0, h1, l1;
      act_split2(v[4 * j], v[4 * j + 1], bias_s, cj + 2 * q, slope, h0, l0);
      act_split2(v[4 * j + 4], v[4 * j + 5], bias_s, cj + 8 + 2 * q, slope, h1, l1);
      // an even lane keeps group j and sends group j + 1, an odd lane the reverse
      const uint32_t rh = __shfl_xor_sync(0xffffffffu, odd ? h0 : h1, 1);
      const uint32_t rl = __shfl_xor_sync(0xffffffffu, odd ? l0 : l1, 1);
      const int g = odd ? cj + 8 : cj;   // first channel of the lane's group
      if (g + 8 <= Cout) {
        const int c = odd ? g + 2 * (q - 1) : g + 2 * q;
        *reinterpret_cast<uint2*>(out_hi + c) = odd ? make_uint2(rh, h1) : make_uint2(h0, rh);
        *reinterpret_cast<uint2*>(out_lo + c) = odd ? make_uint2(rl, l1) : make_uint2(l0, rl);
      }
    } else {
      epilogue_pair(v[4 * j], v[4 * j + 1], bias_s, cj + 2 * q, Cout, slope, out_hi, out_lo);
      epilogue_pair(v[4 * j + 4], v[4 * j + 5], bias_s, cj + 8 + 2 * q, Cout, slope, out_hi, out_lo);
    }
  }
}

// The epilogue of one thread's share of a 64 x BN accumulator block v[BN / 2] (the Wgmma fragment): bias, activation
// and split-bf16 store of both its pixels.  The slot sets are four groups of one pixel half where BN % 32 == 0; where
// BN % 32 == 16 the last two groups of both halves form one more set.  The three wgmma kernels store through it.
template <int BN>
__device__ __forceinline__ void epilogue_store(const float* v, const float* bias_s, float slope, int lane,
                                               const EpiDest& d) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr)
#pragma unroll
    for (int j0 = 0; j0 + 4 <= BN / 8; j0 += 4) epilogue_set<false>(v, bias_s, slope, lane, d, hr, j0);
  if constexpr (BN % 32 == 16) epilogue_set<true>(v, bias_s, slope, lane, d, 0, BN / 8 - 2);
}

// 8-channel groups of chunk cc that carry any non-zero weight (4 bits per 32-channel chunk)
__device__ __forceinline__ uint32_t chunk_groups(unsigned long long kmask, int cc) {
  const int sh = cc * 4;
  return sh + 4 <= 64 ? (uint32_t)(kmask >> sh) & 0xFu : 0xFu;
}

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], "
      "[%6];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
      : "memory");
}

}  // namespace vr
