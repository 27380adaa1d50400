// Shared device/host definitions for the vocal-remover H100 hot path (sm_90a only).
//
// Activation storage ("split-bf16"): every activation tensor of the CascadedNet forward
// (reference lib/nets.py:82-117) lives in HBM as TWO NHWC bf16 planes, hi = bf16(x) and
// lo = bf16(x - hi).  hi+lo carries a 16-bit significand, which is what lets the wgmma
// bf16 tensor-core convolution (conv_tc.cu) reach the 1e-3 mask parity gate with three
// bf16 passes (hi*hi + lo*hi + hi*lo, fp32 accumulate in registers); a single bf16/fp16 pass fails it
// (DESIGN.md "Precision").  The planes cost the same 4 B/element as fp32 and are directly
// TMA-loadable as tensor-core operands.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vr {

typedef __nv_bfloat16 bf16;

enum ActKind { ACT_NONE = 0, ACT_RELU = 1, ACT_LEAKY = 2 };

// View of an NHWC split-bf16 tensor (possibly a channel slice / band of a larger buffer).
struct ActView {
  bf16* hi;
  bf16* lo;
  int N, H, W, C;   // logical extent of the view (C = channels visible through it)
  int64_t sn;       // element stride between images
  int64_t sh;       // element stride between rows (H)
  int sw;           // element stride between pixels (= channel count of the underlying buffer)
};

// Parameters of one fused Conv2d(bias=False)+BatchNorm2d(eval)+activation layer
// (reference lib/layers.py:8-26) in implicit-GEMM form.
struct ConvParams {
  ActView in;        // in.C == CinPad (multiple of 8; zero weights on pad channels)
  ActView out;       // out.C == number of output channels stored (Cout)
  const float* w;    // fp32 [taps][CinPad][CoutPad], BN scale folded in
  const float* bias; // fp32 [CoutPad], folded BN shift
  int CinPad, Cout, CoutPad;
  int KH, KW, stride, pad_h, pad_w, dil_h, dil_w;
  int act;
};

__device__ __forceinline__ float act_apply(float v, int act) {
  if (act == ACT_RELU) return fmaxf(v, 0.f);
  if (act == ACT_LEAKY) return v > 0.f ? v : 0.01f * v;   // nn.LeakyReLU default slope (lib/layers.py:31)
  return v;
}

__device__ __forceinline__ void split_bf16(float v, bf16& hi, bf16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

__device__ __forceinline__ float join_bf16(bf16 hi, bf16 lo) {
  return __bfloat162float(hi) + __bfloat162float(lo);
}

// 8 consecutive bf16 (16 bytes) <-> 8 floats.  All 16-byte accesses go through uint4 so that they compile to
// LDG.E.128 / STG.E.128 (a struct of __nv_bfloat162 members is copied member-wise as 4-byte accesses).
typedef uint4 bf16x8;

__device__ __forceinline__ float2 bf2_to_f2(uint32_t u) {
  // bf16 -> fp32 is a 16-bit shift
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ bf16x8 ld128(const bf16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void st128(bf16* p, const bf16x8& v) { *reinterpret_cast<uint4*>(p) = v; }

__device__ __forceinline__ void unpack8(const bf16x8& a, const bf16x8& b, float* x) {
  const uint32_t ua[4] = {a.x, a.y, a.z, a.w};
  const uint32_t ub[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 fa = bf2_to_f2(ua[i]);
    float2 fb = bf2_to_f2(ub[i]);
    x[2 * i] = fa.x + fb.x;
    x[2 * i + 1] = fa.y + fb.y;
  }
}

__device__ __forceinline__ void load8(const bf16* hi, const bf16* lo, float* x) {
  unpack8(ld128(hi), ld128(lo), x);
}

__device__ __forceinline__ void split8(const float* x, bf16x8& h, bf16x8& l) {
  uint32_t uh[4], ul[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uh[i] = f2_to_bf2(x[2 * i], x[2 * i + 1]);
    float2 hf = bf2_to_f2(uh[i]);
    ul[i] = f2_to_bf2(x[2 * i] - hf.x, x[2 * i + 1] - hf.y);
  }
  h = make_uint4(uh[0], uh[1], uh[2], uh[3]);
  l = make_uint4(ul[0], ul[1], ul[2], ul[3]);
}

// 32-byte (16-channel) store: one full sector per lane, as two 16-byte stores (sm_90 has no 256-bit store)
__device__ __forceinline__ void st256(bf16* p, const bf16x8& a, const bf16x8& b) {
  st128(p, a);
  st128(p + 8, b);
}

// Store `cnt` consecutive channels (fp32 values) of one pixel as split-bf16.
__device__ __forceinline__ void store_split(bf16* hi, bf16* lo, const float* x, int cnt) {
  if (cnt == 8 && ((reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 15) == 0) {
    bf16x8 h, l;
    split8(x, h, l);
    st128(hi, h);
    st128(lo, l);
  } else {
    for (int i = 0; i < cnt; ++i) split_bf16(x[i], hi[i], lo[i]);
  }
}

// 16 consecutive channels; uses full-sector 32-byte stores when the destination allows it
__device__ __forceinline__ void store_split16(bf16* hi, bf16* lo, const float* x, int cnt) {
  if (cnt == 16 && ((reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 31) == 0) {
    bf16x8 h0, l0, h1, l1;
    split8(x, h0, l0);
    split8(x + 8, h1, l1);
    st256(hi, h0, h1);
    st256(lo, l0, l1);
  } else {
    store_split(hi, lo, x, cnt < 8 ? cnt : 8);
    if (cnt > 8) store_split(hi + 8, lo + 8, x + 8, cnt - 8);
  }
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

}  // namespace vr
