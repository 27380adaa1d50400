// Vorbis I decoding on the device: the decode in front of the hot path for .ogg input (lib/vorbis.py reads the Ogg
// pages and the three headers, flattens the setup and drives it; oracle/vorbis_oracle.py restates the specification
// in float64 and is pinned against FFmpeg).
//
// The host hands over the audio packets back to back, one row per packet (byte offset, size, end of the packet's
// output range, offset of its spectrum slot, block flag), and the setup as one int32 array (layout below, written by
// lib/vorbis.flatten).  Each packet's block size is known on the host, so every packet writes at a known place.
//   vorbis_parse_kernel      one thread per packet: the floor 1 values of each channel, unwrapped into the points the
//                            curve passes through, and the residue vectors (every class, cascade pass and VQ
//                            codeword) into the packet's spectrum slot.  Codewords are found by a binary search over
//                            the book's left-aligned, sorted codes, in shared memory when all books fit and in global
//                            memory otherwise.  Every read is bounded by the packet; an end of packet in a floor leaves
//                            the channel unused and in a residue ends the residue decode, as the specification says; a
//                            malformed packet leaves code << 40 | bit in its status.
//   vorbis_synth_kernel      one CTA per packet: inverse coupling, floor curve x residue, the IMDCT of the block as an
//                            n/4-point complex FFT in shared memory between a pre- and a post-twiddle, the window with
//                            its slopes for the packet's flags; the left half to the output, the right half (the tail)
//                            over the spectrum slot.
//   vorbis_overlap_kernel    one CTA per packet: adds the previous packet's tail to the packet's output range.
#include <math.h>

#include "bitstream.cuh"
#include "common.cuh"
#include "kernels.h"

namespace vr {

namespace {

// Generated from oracle/vorbis_oracle.py's INVERSE_DB (tests/test_vorbis.py checks that the two agree).
__constant__ float kVorbisInverseDb[256] = {
    1.0649863e-07f, 1.1341951e-07f, 1.2079015e-07f, 1.2863978e-07f, 1.369995e-07f, 1.459025e-07f,
    1.5538409e-07f, 1.6548181e-07f, 1.7623574e-07f, 1.8768856e-07f, 1.998856e-07f, 2.1287531e-07f,
    2.2670913e-07f, 2.4144197e-07f, 2.5713223e-07f, 2.7384212e-07f, 2.9163792e-07f, 3.1059022e-07f,
    3.307741e-07f, 3.5226967e-07f, 3.7516213e-07f, 3.995423e-07f, 4.2550681e-07f, 4.5315863e-07f,
    4.8260745e-07f, 5.1397001e-07f, 5.4737063e-07f, 5.8294188e-07f, 6.2082472e-07f, 6.6116939e-07f,
    7.0413591e-07f, 7.4989464e-07f, 7.9862701e-07f, 8.5052631e-07f, 9.0579829e-07f, 9.6466215e-07f,
    1.0273513e-06f, 1.0941144e-06f, 1.1652161e-06f, 1.2409384e-06f, 1.3215816e-06f, 1.4074654e-06f,
    1.4989305e-06f, 1.5963394e-06f, 1.7000785e-06f, 1.8105592e-06f, 1.9282195e-06f, 2.053526e-06f,
    2.1869757e-06f, 2.3290977e-06f, 2.4804558e-06f, 2.6416496e-06f, 2.813319e-06f, 2.9961443e-06f,
    3.1908505e-06f, 3.3982101e-06f, 3.6190449e-06f, 3.8542307e-06f, 4.1047006e-06f, 4.3714472e-06f,
    4.6555283e-06f, 4.9580708e-06f, 5.2802739e-06f, 5.6234162e-06f, 5.9888571e-06f, 6.3780467e-06f,
    6.7925284e-06f, 7.2339453e-06f, 7.7040477e-06f, 8.2047e-06f, 8.7378876e-06f, 9.3057251e-06f, 9.9104636e-06f,
    1.0554501e-05f, 1.1240392e-05f, 1.1970856e-05f, 1.2748789e-05f, 1.3577278e-05f, 1.4459606e-05f,
    1.5399271e-05f, 1.6400005e-05f, 1.7465769e-05f, 1.8600793e-05f, 1.9809577e-05f, 2.1096914e-05f,
    2.2467912e-05f, 2.3928002e-05f, 2.5482977e-05f, 2.7139005e-05f, 2.890265e-05f, 3.078091e-05f,
    3.2781227e-05f, 3.4911533e-05f, 3.7180282e-05f, 3.9596467e-05f, 4.2169668e-05f, 4.4910092e-05f,
    4.7828602e-05f, 5.0936775e-05f, 5.4246932e-05f, 5.7772202e-05f, 6.1526567e-05f, 6.552491e-05f,
    6.9783084e-05f, 7.4317984e-05f, 7.9147583e-05f, 8.4291038e-05f, 8.976875e-05f, 9.5602423e-05f,
    0.00010181521f, 0.00010843174f, 0.00011547824f, 0.00012298267f, 0.00013097477f, 0.00013948625f,
    0.00014855085f, 0.00015820454f, 0.00016848555f, 0.00017943469f, 0.00019109536f, 0.00020351382f,
    0.0002167393f, 0.00023082423f, 0.00024582449f, 0.00026179955f, 0.00027881275f, 0.00029693157f,
    0.00031622787f, 0.00033677815f, 0.00035866388f, 0.00038197188f, 0.00040679457f, 0.00043323037f,
    0.0004613841f, 0.00049136748f, 0.00052329927f, 0.00055730622f, 0.00059352309f, 0.00063209358f,
    0.00067317061f, 0.00071691698f, 0.00076350628f, 0.00081312325f, 0.00086596457f, 0.00092223985f,
    0.00098217221f, 0.0010459992f, 0.0011139743f, 0.0011863665f, 0.0012634633f, 0.0013455702f, 0.0014330129f,
    0.0015261382f, 0.0016253153f, 0.0017309374f, 0.0018434235f, 0.0019632196f, 0.0020908006f, 0.0022266726f,
    0.0023713743f, 0.0025254795f, 0.0026895993f, 0.0028643848f, 0.0030505287f, 0.0032487691f, 0.0034598925f,
    0.0036847359f, 0.0039241905f, 0.0041792067f, 0.0044507948f, 0.0047400328f, 0.0050480668f, 0.0053761187f,
    0.005725489f, 0.0060975635f, 0.0064938175f, 0.0069158226f, 0.0073652514f, 0.0078438874f, 0.0083536273f,
    0.0088964924f, 0.009474637f, 0.010090352f, 0.01074608f, 0.011444421f, 0.012188144f, 0.012980198f,
    0.013823725f, 0.014722068f, 0.015678791f, 0.016697686f, 0.017782796f, 0.018938422f, 0.020169148f,
    0.021479854f, 0.022875736f, 0.024362329f, 0.025945531f, 0.027631618f, 0.029427277f, 0.031339627f,
    0.03337625f, 0.035545226f, 0.037855156f, 0.0403152f, 0.042935107f, 0.045725275f, 0.048696756f, 0.051861349f,
    0.05523159f, 0.058820851f, 0.062643364f, 0.066714279f, 0.07104975f, 0.075666964f, 0.080584228f,
    0.085821047f, 0.09139818f, 0.097337745f, 0.1036633f, 0.11039993f, 0.11757434f, 0.12521498f, 0.13335215f,
    0.14201812f, 0.15124726f, 0.16107617f, 0.17154381f, 0.18269168f, 0.19456401f, 0.20720787f, 0.22067343f,
    0.23501402f, 0.25028655f, 0.26655158f, 0.28387362f, 0.30232131f, 0.32196787f, 0.34289113f, 0.36517414f,
    0.3889052f, 0.41417846f, 0.44109413f, 0.4697589f, 0.50028646f, 0.53279793f, 0.56742209f, 0.60429639f,
    0.64356697f, 0.68538958f, 0.72993004f, 0.77736503f, 0.82788259f, 0.88168305f, 0.9389798f, 1.0f
};

// The setup array (int32 words).  Header, then the book rows, the codes (uint32, left-aligned, sorted per book), their
// info (entry << 6 | length), the VQ vectors (float32), the floors, residues, mappings and modes.
constexpr int kHdrChannels = 0, kHdrBs0 = 1, kHdrBs1 = 2, kHdrOffBooks = 4, kHdrOffCodes = 5,
              kHdrOffInfo = 6, kHdrOffVec = 7, kHdrOffFloors = 9, kHdrOffRes = 10, kHdrOffMaps = 11, kHdrModes = 12,
              kHdrOffModes = 13, kHdrCodes = 14, kHdrModeBits = 15, kHdrWords = 16;
constexpr int kBookWords = 8;   // dims, entries, first code, code count, vector offset (-1: none), single entry (-1)
constexpr int kFloorWords = 472, kFlParts = 0, kFlMult = 1, kFlValues = 2, kFlRange = 3, kFlPartClass = 4,
              kFlClassDim = 36, kFlClassSub = 52, kFlClassMaster = 68, kFlSubBooks = 84, kFlX = 212, kFlOrder = 277;
constexpr int kResWords = 518, kRsType = 0, kRsBegin = 1, kRsEnd = 2, kRsPsize = 3, kRsClasses = 4, kRsClassbook = 5,
              kRsBooks = 6;
constexpr int kMapWords = 548, kMpSubmaps = 0, kMpSteps = 1, kMpMux = 2, kMpFloor = 4, kMpResidue = 20,
              kMpCoupling = 36;
constexpr int kMaxValues = 65;
// per packet-channel: count, then (x << 16 | y) of the points the curve passes through, packed unsigned (x reaches
// 2^15 with rangebits 15)
constexpr int kListWords = 68;
constexpr int kParseThreads = 64;
constexpr int kSharedCodeBytes = 96 * 1024;

// status codes (lib/vorbis.py ERRORS)
constexpr int kErrType = 1, kErrMode = 2, kErrCodeword = 3, kErrFloorRange = 4, kErrHeader = 5;

__device__ __forceinline__ int ilog(uint32_t v) { return v ? 32 - __clz(v) : 0; }

struct Setup {
  const int* s;
  const uint32_t* codes;   // shared or global (generic pointers)
  const uint32_t* info;
  const float* vec;
  __device__ __forceinline__ const int* book(int b) const { return s + s[kHdrOffBooks] + b * kBookWords; }
  __device__ __forceinline__ const int* floor(int f) const { return s + s[kHdrOffFloors] + f * kFloorWords; }
  __device__ __forceinline__ const int* residue(int r) const { return s + s[kHdrOffRes] + r * kResWords; }
  __device__ __forceinline__ const int* mapping(int m) const { return s + s[kHdrOffMaps] + m * kMapWords; }
};

// The entry of book ``b`` that the stream codes at br.pos: >= 0 (br.pos moves past the codeword), -1 for an end of
// packet inside the codeword, -2 for a codeword the book does not hold (every codeword, when the book has no used
// entry: its first bit already leaves the tree, as in the oracle).  The next 32 stream bits, bit-reversed, are the
// codeword MSB-first; bits past the packet end are set to one for the search, so that the entry found is the last one
// that the packet's own bits can still begin.  Only the book's own codes [bk[2], bk[2] + bk[3]) are read.
__device__ __forceinline__ int read_entry(LsbBits& br, const Setup& st, int b) {
  const int* bk = st.book(b);
  if (bk[5] >= 0) return bk[5];
  const int64_t left = br.end - br.pos;
  if (left <= 0) {
    br.pos = br.end + 1;
    return -1;
  }
  const uint32_t w = __brev(br.peek32());
  const uint32_t pad = left >= 32 ? 0u : (0xFFFFFFFFu >> left);
  const uint32_t w1 = w | pad;
  int a = bk[2], span = bk[3];
  if (span <= 0) return -2;
  while (span > 1) {
    const int half = span >> 1;
    if (st.codes[a + half] <= w1) a += half;
    span -= half;
  }
  const uint32_t c = st.codes[a], inf = st.info[a];
  const int len = (int)(inf & 63u);
  const uint32_t mask = len >= 32 ? 0xFFFFFFFFu : ~(0xFFFFFFFFu >> len);
  if (c <= w1 && ((c ^ w) & mask) == 0 && len <= left) {
    br.pos += len;
    return (int)(inf >> 6);
  }
  // a code that starts with the packet's remaining bits: the packet ends inside it
  const uint32_t keep = ~pad;
  if (c <= w1 && (c & keep) == (w & keep)) {
    br.pos = br.end + 1;
    return -1;
  }
  return -2;
}

__device__ __forceinline__ int render_point(int x0, int y0, int x1, int y1, int x) {
  const int dy = y1 - y0, adx = x1 - x0;
  const int off = (abs(dy) * (x - x0)) / adx;
  return dy < 0 ? y0 - off : y0 + off;
}

// floor 1 of one channel -> 1 (used; the curve's points in list), 0 (unused, or end of packet), or -code
__device__ __forceinline__ int floor1_decode(LsbBits& br, const Setup& st, const int* fl, int16_t* y, int* list) {
  const int mult = fl[kFlMult], range = fl[kFlRange], values = fl[kFlValues];
  if (br.end - br.pos < 1) return 0;
  if (!br.read(1)) return 0;
  const int bits = ilog((uint32_t)(range - 1));
  y[0] = (int16_t)br.read(bits);
  y[1] = (int16_t)br.read(bits);
  if (br.over()) return 0;
  const bool y01_bad = y[0] >= range || y[1] >= range;
  int off = 2;
  for (int p = 0; p < fl[kFlParts]; ++p) {
    const int cls = fl[kFlPartClass + p];
    const int cdim = fl[kFlClassDim + cls], cbits = fl[kFlClassSub + cls], csub = (1 << cbits) - 1;
    int cval = 0;
    if (cbits) {
      cval = read_entry(br, st, fl[kFlClassMaster + cls]);
      if (cval == -1) return 0;
      if (cval < 0) return -kErrCodeword;
    }
    for (int j = 0; j < cdim; ++j) {
      const int book = fl[kFlSubBooks + cls * 8 + (cval & csub)];
      cval >>= cbits;
      int v = 0;
      if (book >= 0) {
        v = read_entry(br, st, book);
        if (v == -1) return 0;
        if (v < 0) return -kErrCodeword;
      }
      y[off++] = (int16_t)min(v, 0x7FFF);
    }
  }
  if (y01_bad) return -kErrFloorRange;
  // amplitude unwrap (step 2): final Y in y, the step2 flag in bit 14
  const int* X = fl + kFlX;
  const int* low = fl + kFlOrder + kMaxValues;   // the host's low_neighbor / high_neighbor of each value
  const int* high = fl + kFlOrder + 2 * kMaxValues;
  y[0] |= 0x4000;
  y[1] |= 0x4000;
  for (int i = 2; i < values; ++i) {
    const int lo = low[i], hi = high[i];
    const int pred = render_point(X[lo], y[lo] & 0x3FFF, X[hi], y[hi] & 0x3FFF, X[i]);
    const int val = y[i], hr = range - pred, lr = pred, room = 2 * min(hr, lr);
    int f;
    if (val) {
      y[lo] |= 0x4000;
      y[hi] |= 0x4000;
      if (val >= room) f = hr > lr ? val - lr + pred : pred - val + hr - 1;
      else f = (val & 1) ? pred - ((val + 1) >> 1) : pred + (val >> 1);
      if (f < 0 || f >= range) return -kErrFloorRange;
      y[i] = (int16_t)(f | 0x4000);
    } else {
      y[i] = (int16_t)pred;
    }
  }
  // the points the curve passes through, in increasing x
  int cnt = 0;
  const int* order = fl + kFlOrder;
  for (int k = 0; k < values; ++k) {
    const int i = order[k];
    if (y[i] & 0x4000) list[1 + cnt++] = (int)(((uint32_t)X[i] << 16) | (uint32_t)((y[i] & 0x3FFF) * mult));
  }
  list[0] = cnt;
  return 1;
}

// residue decode of one submap: ch vectors (their slot pointers), skip flags; returns 0, -1 (end of packet) or -code
__device__ __forceinline__ int residue_decode(LsbBits& br, const Setup& st, const int* rs, float* v0, float* v1,
                                              bool skip0, bool skip1, int ch, int n2, uint8_t* __restrict__ classes) {
  const int type = rs[kRsType];
  if (skip0 && (ch == 1 || skip1)) return 0;
  const int nvec = type == 2 ? 1 : ch;
  const int size = type == 2 ? n2 * ch : n2;
  const int lb = min(rs[kRsBegin], size), le = min(rs[kRsEnd], size);
  const int psize = rs[kRsPsize], ncls = rs[kRsClasses];
  const int cb = rs[kRsClassbook];
  const int cw = st.book(cb)[0];
  const int nparts = le > lb ? (le - lb) / psize : 0;
  if (nparts == 0) return 0;
  for (int pass = 0; pass < 8; ++pass) {
    int pc = 0;
    while (pc < nparts) {
      if (pass == 0) {
        for (int j = 0; j < nvec; ++j) {
          if (type != 2 && (j ? skip1 : skip0)) continue;
          int t = read_entry(br, st, cb);
          if (t == -1) return -1;
          if (t < 0) return -kErrCodeword;
          for (int i = cw - 1; i >= 0; --i) {
            if (pc + i < nparts) classes[j * size + pc + i] = (uint8_t)(t % ncls);
            t /= ncls;
          }
        }
      }
      for (int i = 0; i < cw && pc < nparts; ++i, ++pc) {
        for (int j = 0; j < nvec; ++j) {
          if (type != 2 && (j ? skip1 : skip0)) continue;
          const int book = rs[kRsBooks + classes[j * size + pc] * 8 + pass];
          if (book < 0) continue;
          const int* bk = st.book(book);
          const int dims = bk[0];
          const float* V = st.vec + bk[4];
          const int off = lb + pc * psize;
          if (type == 0) {
            const int step = psize / dims;
            for (int k = 0; k < step; ++k) {
              const int e = read_entry(br, st, book);
              if (e == -1) return -1;
              if (e < 0) return -kErrCodeword;
              for (int d = 0; d < dims; ++d) (j ? v1 : v0)[off + k + d * step] += __ldg(V + e * dims + d);
            }
          } else {
            for (int k = 0; k < psize; k += dims) {
              const int e = read_entry(br, st, book);
              if (e == -1) return -1;
              if (e < 0) return -kErrCodeword;
              for (int d = 0; d < dims && k + d < psize; ++d) {
                const int pos = off + k + d;
                const float v = __ldg(V + e * dims + d);
                if (type == 1) (j ? v1 : v0)[pos] += v;
                else if (ch == 1 || !(pos & 1)) v0[pos / ch] += v;
                else v1[pos >> 1] += v;
              }
            }
          }
        }
      }
    }
  }
  return 0;
}

}  // namespace

// one thread per packet
__global__ void __launch_bounds__(kParseThreads, 1) vorbis_parse_kernel(const uint8_t* __restrict__ d, int64_t n_bytes,
                                                                     const int64_t* __restrict__ table, int n_packets,
                                                                     const int* __restrict__ setup, int shared_codes,
                                                                     float* __restrict__ spec,
                                                                     uint8_t* __restrict__ classes,
                                                                     int* __restrict__ lists,
                                                                     int64_t* __restrict__ status) {
  extern __shared__ __align__(16) uint32_t s_codes[];
  __shared__ int16_t s_y[kParseThreads][kMaxValues + 1];
  Setup st{setup, reinterpret_cast<const uint32_t*>(setup + setup[kHdrOffCodes]),
           reinterpret_cast<const uint32_t*>(setup + setup[kHdrOffInfo]),
           reinterpret_cast<const float*>(setup + setup[kHdrOffVec])};
  const int n_codes = setup[kHdrCodes];
  if (shared_codes) {
    for (int i = threadIdx.x; i < n_codes; i += blockDim.x) {
      s_codes[i] = st.codes[i];
      s_codes[n_codes + i] = st.info[i];
    }
    __syncthreads();
    st.codes = s_codes;
    st.info = s_codes + n_codes;
  }
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_packets) return;
  const int64_t* row = table + (int64_t)p * 5;
  const int C = setup[kHdrChannels];
  LsbBits br{d, n_bytes, row[0] * 8, (row[0] + row[1]) * 8};
  int64_t stat = 0;
  int* list = lists + (int64_t)p * C * kListWords;
  for (int c = 0; c < C; ++c) list[c * kListWords] = -1;   // unused floor
  const int mode_bits = setup[kHdrModeBits];
  const int type = (int)br.read(1);
  const int mode = (int)br.read(mode_bits);
  if (br.over() || row[1] == 0) {
    status[p] = frame_status(kErrHeader, 0);
    return;
  }
  if (type) {
    status[p] = frame_status(kErrType, 0);
    return;
  }
  if (mode >= setup[kHdrModes]) {
    status[p] = frame_status(kErrMode, 1);
    return;
  }
  const int* md = setup + setup[kHdrOffModes] + 2 * mode;
  const int bf = md[0];
  if (bf) {
    br.read(2);
    if (br.over()) {
      status[p] = frame_status(kErrHeader, 0);
      return;
    }
  }
  const int n2 = setup[bf ? kHdrBs1 : kHdrBs0] / 2;
  const int* mp = st.mapping(md[1]);
  bool no_res0 = true, no_res1 = true;
  for (int c = 0; c < C && !stat; ++c) {
    const int sub = mp[kMpMux + c];
    const int64_t at = br.pos;
    const int r = floor1_decode(br, st, st.floor(mp[kMpFloor + sub]), s_y[threadIdx.x], list + c * kListWords);
    if (r < 0) stat = frame_status(-r, at);
    else if (r == 1) (c ? no_res1 : no_res0) = false;
    else list[c * kListWords] = -1;
  }
  if (!stat) {
    for (int s = mp[kMpSteps] - 1; s >= 0; --s) {
      const int m = mp[kMpCoupling + 2 * s], a = mp[kMpCoupling + 2 * s + 1];
      const bool used = !(m ? no_res1 : no_res0) || !(a ? no_res1 : no_res0);
      if (used) no_res0 = (m == 0 || a == 0) ? false : no_res0, no_res1 = (m == 1 || a == 1) ? false : no_res1;
    }
    float* slot = spec + row[3];
    uint8_t* cls = classes + row[3];
    for (int s = 0; s < mp[kMpSubmaps]; ++s) {
      // the submap's channels in order (at most two)
      const bool in0 = mp[kMpMux] == s, in1 = C == 2 && mp[kMpMux + 1] == s;
      const int ch = (int)in0 + (int)in1;
      if (!ch) continue;
      float* v0 = slot + (in0 ? 0 : n2);
      float* v1 = slot + n2;
      const bool skip0 = in0 ? no_res0 : no_res1, skip1 = no_res1;
      const int64_t at = br.pos;
      const int r = residue_decode(br, st, st.residue(mp[kMpResidue + s]), v0, v1, skip0, skip1, ch, n2, cls);
      if (r == -1) break;
      if (r < 0) {
        stat = frame_status(-r, at);
        break;
      }
    }
  }
  if (stat) {
    for (int c = 0; c < C; ++c) list[c * kListWords] = -1;
    stat = (stat & ~0xFFFFFFFFFFLL) | ((stat & 0xFFFFFFFFFFLL) - row[0] * 8);
  }
  status[p] = stat;
}

// one CTA per packet
__global__ void __launch_bounds__(256) vorbis_synth_kernel(const int64_t* __restrict__ table, int n_packets,
                                                           const int* __restrict__ setup, const int* __restrict__ lists,
                                                           float* __restrict__ spec, float* __restrict__ out,
                                                           int64_t n_out) {
  __shared__ float2 buf[2048];
  __shared__ float2 tw[1024];
  __shared__ uint32_t pts[kListWords];
  const int p = blockIdx.x;
  const int64_t* row = table + (int64_t)p * 5;
  const int C = setup[kHdrChannels], bs0 = setup[kHdrBs0];
  const int bf = (int)row[4] & 1;
  const int n = setup[bf ? kHdrBs1 : kHdrBs0], n2 = n / 2, q = n / 4;
  float* slot = spec + row[3];
  // row[4]: block flag | previous window flag << 1 | next window flag << 2 | mapping << 8, read on the host
  const int* mp = setup + setup[kHdrOffMaps] + (int)(row[4] >> 8) * kMapWords;
  const int prev = (int)(row[4] >> 1) & 1, next = (int)(row[4] >> 2) & 1;
  // inverse coupling, last step first
  for (int s = mp[kMpSteps] - 1; s >= 0; --s) {
    float* M = slot + (int64_t)mp[kMpCoupling + 2 * s] * n2;
    float* A = slot + (int64_t)mp[kMpCoupling + 2 * s + 1] * n2;
    for (int j = threadIdx.x; j < n2; j += blockDim.x) {
      const float m = M[j], a = A[j];
      float nm, na;
      if (m > 0.0f) {
        if (a > 0.0f) { nm = m; na = m - a; }
        else { na = m; nm = m + a; }
      } else {
        if (a > 0.0f) { nm = m; na = m + a; }
        else { na = m; nm = m - a; }
      }
      M[j] = nm;
      A[j] = na;
    }
    __syncthreads();
  }
  const int logq = 31 - __clz(q);
  for (int j = threadIdx.x; j < q / 2; j += blockDim.x) {
    float sn, cs;
    sincospif(-2.0f * (float)j / (float)q, &sn, &cs);
    tw[j] = make_float2(cs, sn);
  }
  // window slopes (the specification's, for the packet's flags)
  int ls = 0, ln = n2, rs = n2, rn = n2;
  if (bf && !prev) { ls = n / 4 - bs0 / 4; ln = bs0 / 2; }
  if (bf && !next) { rs = 3 * n / 4 - bs0 / 4; rn = bs0 / 2; }
  const int64_t end = row[2], start = end - n2;   // the block's centre is the end of the packet's output range
  const int64_t range_a = p ? table[(int64_t)(p - 1) * 5 + 2] : end;
  for (int c = 0; c < C; ++c) {
    __syncthreads();
    const int* L = lists + ((int64_t)p * C + c) * kListWords;
    const int cnt = L[0];
    for (int i = threadIdx.x; i < kListWords; i += blockDim.x) pts[i] = (uint32_t)L[i];
    __syncthreads();
    float* X = slot + (int64_t)c * n2;
    // pre-twiddle of (X[2k] + i X[M-1-2k]) times the floor, into bit-reversed order
    for (int k = threadIdx.x; k < q; k += blockDim.x) {
      float v[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int idx = h ? n2 - 1 - 2 * k : 2 * k;
        float f = 0.0f;
        if (cnt > 0) {
          int a = 0, span = cnt;
          while (span > 1) {
            const int half = span >> 1;
            if ((int)(pts[1 + a + half] >> 16) <= idx) a += half;
            span -= half;
          }
          const int x0 = (int)(pts[1 + a] >> 16), y0 = (int)(pts[1 + a] & 0xFFFF);
          int y = y0;
          if (a + 1 < cnt) y = render_point(x0, y0, (int)(pts[2 + a] >> 16), (int)(pts[2 + a] & 0xFFFF), idx);
          f = kVorbisInverseDb[min(max(y, 0), 255)] * X[idx];
        }
        v[h] = f;
      }
      float sn, cs;
      sincospif(-(float)(4 * k + 1) / (float)(2 * n), &sn, &cs);
      buf[__brev((unsigned)k) >> (32 - logq)] = make_float2(v[0] * cs - v[1] * sn, v[0] * sn + v[1] * cs);
    }
    // radix-2 forward FFT (e^{-2 pi i nk / q})
    for (int half = 1; half < q; half *= 2) {
      __syncthreads();
      for (int j = threadIdx.x; j < q / 2; j += blockDim.x) {
        const int pos = j & (half - 1), i0 = (j - pos) * 2 + pos, i1 = i0 + half;
        const float2 w = tw[pos * (q / (2 * half))];
        const float2 a = buf[i0], b = buf[i1];
        const float2 bw = make_float2(b.x * w.x - b.y * w.y, b.x * w.y + b.y * w.x);
        buf[i0] = make_float2(a.x + bw.x, a.y + bw.y);
        buf[i1] = make_float2(a.x - bw.x, a.y - bw.y);
      }
    }
    __syncthreads();
    // post-twiddle -> u[2k] = Re, u[M-1-2k] = -Im; u[m] lands at y[3M/2-1-m] = -u[m] and at y[m-M/2] = u[m] (m >= M/2)
    // or y[m+3M/2] = -u[m] (m < M/2); then the window, the left half to out and the right half over the slot
    float* o = out + (int64_t)c * n_out;
    for (int k = threadIdx.x; k < q; k += blockDim.x) {
      float sn, cs;
      sincospif(-(float)k / (float)n2, &sn, &cs);
      const float2 z = buf[k];
      const float re = z.x * cs - z.y * sn, im = z.x * sn + z.y * cs;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = h ? n2 - 1 - 2 * k : 2 * k;
        const float u = h ? -im : re;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          int i;
          float val;
          if (t == 0) {
            i = 3 * n2 / 2 - 1 - m;
            val = -u;
          } else if (m >= n2 / 2) {
            i = m - n2 / 2;
            val = u;
          } else {
            i = m + 3 * n2 / 2;
            val = -u;
          }
          float w;
          if (i < ls) w = 0.0f;
          else if (i < ls + ln) {
            const float s = sinpif(((float)(i - ls) + 0.5f) / (float)(2 * ln));
            w = sinpif(0.5f * s * s);
          } else if (i < rs) w = 1.0f;
          else if (i < rs + rn) {
            const float s = sinpif(((float)(i - rs) + 0.5f) / (float)(2 * rn) + 0.5f);
            w = sinpif(0.5f * s * s);
          } else w = 0.0f;
          val *= w;
          if (i < n2) {
            const int64_t at = start + i;
            if (at >= range_a && at < end) o[at] = val;
          } else {
            X[i - n2] = val;
          }
        }
      }
    }
  }
}

// one CTA per packet past the first: its output range += the previous packet's tail
__global__ void __launch_bounds__(256) vorbis_overlap_kernel(const int64_t* __restrict__ table, int C,
                                                             const int* __restrict__ setup,
                                                             const float* __restrict__ spec, float* __restrict__ out,
                                                             int64_t n_out) {
  const int p = blockIdx.x + 1;
  const int64_t* prow = table + (int64_t)(p - 1) * 5;
  const int64_t a = prow[2], b = table[(int64_t)p * 5 + 2];
  const int pn2 = setup[(prow[4] & 1) ? kHdrBs1 : kHdrBs0] / 2;
  const int64_t len = min(b - a, (int64_t)pn2);
  for (int c = 0; c < C; ++c) {
    const float* tail = spec + prow[3] + (int64_t)c * pn2;
    for (int64_t i = threadIdx.x; i < len; i += blockDim.x) out[(int64_t)c * n_out + a + i] += tail[i];
  }
}

namespace {

struct VorbisWorkspace {
  int* lists;
  uint8_t* classes;
  float* spec;
  int64_t bytes;
};

VorbisWorkspace vorbis_carve(uint8_t* base, int64_t n_packets, int C, int64_t slot_floats) {
  VorbisWorkspace w{};
  Carver c{base};
  w.lists = c.take<int>(n_packets * C * kListWords * 4);
  w.classes = c.take<uint8_t>(slot_floats);
  w.spec = c.take<float>(slot_floats * 4);
  w.bytes = c.bytes;
  return w;
}

}  // namespace

int64_t vorbis_workspace_bytes(int64_t n_packets, int channels, int64_t slot_floats) {
  if (n_packets < 0 || channels < 1 || channels > 2 || slot_floats < 0) return -1;
  return vorbis_carve(nullptr, n_packets, channels, slot_floats).bytes;
}

cudaError_t launch_vorbis_decode(const uint8_t* data, int64_t n_bytes, const int64_t* table, int n_packets,
                                 const int* setup, int setup_words, int channels, int n_codes, int64_t slot_floats,
                                 void* workspace, int64_t workspace_bytes, float* out, int64_t n_out, int64_t* status,
                                 cudaStream_t stream) {
  if (!data || !table || !setup || !workspace || !out || !status || n_packets < 1 || channels < 1 || channels > 2 ||
      setup_words < kHdrWords || n_codes < 0 ||
      workspace_bytes < vorbis_workspace_bytes(n_packets, channels, slot_floats))
    return cudaErrorInvalidValue;
  VorbisWorkspace w = vorbis_carve(static_cast<uint8_t*>(workspace), n_packets, channels, slot_floats);
  cudaError_t e = cudaMemsetAsync(w.spec, 0, (size_t)slot_floats * 4, stream);
  if (e == cudaSuccess && n_out) e = cudaMemsetAsync(out, 0, (size_t)n_out * channels * 4, stream);
  if (e != cudaSuccess) return e;
  // every book's codes and info in shared memory when they fit, else read from global memory
  const int64_t code_bytes = (int64_t)n_codes * 8;
  const int shared_codes = code_bytes <= kSharedCodeBytes;
  const size_t smem = shared_codes ? (size_t)code_bytes : 0;
  if (smem > 48 * 1024) {
    e = cudaFuncSetAttribute(vorbis_parse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  vorbis_parse_kernel<<<(n_packets + kParseThreads - 1) / kParseThreads, kParseThreads, smem, stream>>>(
      data, n_bytes, table, n_packets, setup, shared_codes, w.spec, w.classes, w.lists, status);
  vorbis_synth_kernel<<<n_packets, 256, 0, stream>>>(table, n_packets, setup, w.lists, w.spec, out, n_out);
  if (n_packets > 1)
    vorbis_overlap_kernel<<<n_packets - 1, 256, 0, stream>>>(table, channels, setup, w.spec, out, n_out);
  return cudaGetLastError();
}

}  // namespace vr
