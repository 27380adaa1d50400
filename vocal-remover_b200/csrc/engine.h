// Host-side engine: owns the device arena, the packed checkpoint and the per-layer launch plan of
// the CascadedNet forward (reference lib/nets.py:44-141) and the Separator glue (inference.py:16-102).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace vr {

// Owner of one cudaMalloc allocation.  It is freed on destruction, so the device it was made on must be current then.
template <class T>
class DevPtr {
 public:
  DevPtr() = default;
  DevPtr(DevPtr&& o) noexcept : p_(o.p_) { o.p_ = nullptr; }
  DevPtr(const DevPtr&) = delete;
  DevPtr& operator=(const DevPtr&) = delete;
  ~DevPtr() { reset(); }
  // frees what it holds, then allocates `bytes` (not initialised)
  cudaError_t alloc(size_t bytes) {
    reset();
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) p_ = static_cast<T*>(p);
    return e;
  }
  void reset() {
    if (p_) cudaFree(p_);
    p_ = nullptr;
  }
  T* get() const { return p_; }

 private:
  T* p_ = nullptr;
};

// Allocations that live as long as their owner: the engine's weights and activation buffers, or a test hook's
// temporaries.
typedef std::vector<DevPtr<void>> Arena;

// Grow-only workspace of T: ensure(n) keeps an allocation of at least n elements, else frees it and allocates exactly n.
// The contents are neither kept nor zeroed.
template <class T>
class GrowArray {
 public:
  cudaError_t ensure(int64_t n) {
    if (n <= cap_) return cudaSuccess;
    cap_ = 0;
    const cudaError_t e = mem_.alloc(sizeof(T) * (size_t)n);
    if (e == cudaSuccess) cap_ = n;
    return e;
  }
  T* get() const { return mem_.get(); }

 private:
  DevPtr<T> mem_;
  int64_t cap_ = 0;
};

// Synchronous host-to-device copy of weights or tables; on failure sets err and returns false.
bool upload(void* dst, const void* src, size_t bytes, std::string& err);

struct HostTensor {
  std::vector<int64_t> shape;
  std::vector<float> data;
};

struct Buffer {   // a whole NHWC split-bf16 allocation
  bf16* hi = nullptr;
  bf16* lo = nullptr;
  int N = 0, H = 0, W = 0, C = 0;
  int Wp = 0;   // row pitch in pixels (>= W): the Wp - W trailing pixels of every row are permanent zeros
  ActView view(int n, int h0, int h, int c0, int c) const {
    ActView v;
    const int64_t off = (int64_t)h0 * Wp * C + c0;
    v.hi = hi + off;
    v.lo = lo + off;
    v.N = n; v.H = h; v.W = W; v.C = c;
    v.sn = (int64_t)H * Wp * C;
    v.sh = (int64_t)Wp * C;
    v.sw = C;
    return v;
  }
  ActView all(int n) const { return view(n, 0, H, 0, C); }
};

struct TcConv;   // tensor-core plan (conv_tc.cu)

// A prepared layer holds the device weights of the one kernel that runs it: w / bias are non-null exactly when tc is
// null.  No host copy of its weights is kept.
struct ConvLayer {
  std::string name;
  int Cin = 0, CinPad = 0, Cout = 0, CoutPad = 0;
  int k = 1, stride = 1, dil_h = 1, dil_w = 1, act = ACT_RELU;
  float* w = nullptr;      // CUDA-core kernel: device fp32 [taps][CinPad][CoutPad]
  float* bias = nullptr;   // CUDA-core kernel: device fp32 [CoutPad]
  std::shared_ptr<TcConv> tc;    // the tensor-core kernel and its packed weights; null -> CUDA-core kernel
};

// Work one convolution launch does besides the layer; the default is none.  Only the row kernel implements it (what a
// plan can fuse: TcConv::fuses_*); every other path rejects a launch that asks for any.
struct ConvFusion {
  const ActView* up = nullptr;           // the leading up->C input channels are the x2 upsample of *up; `in` the rest
  const ActView* last_chunk = nullptr;   // the last channel chunk is read from here, zero-filled up to the chunk
  // sum_c dot_w[c] * y[c] of every output pixel is added to the pre-zeroed plane dot_out[n][h][w] (the LSTM branch's
  // 1x1 input convolution fused into dec2)
  const float* dot_w = nullptr;
  float* dot_out = nullptr;
  // stage 3's dec1: only the output columns [mask->offset, W - mask->offset) are computed, and the network's mask is
  // written there (mask_out_kernel's work) instead of the layer
  const MaskOutParams* mask = nullptr;
  bool empty() const { return !up && !last_chunk && !dot_w && !dot_out && !mask; }
};

struct LstmPlan {
  int C = 0, bins = 0, hid = 0, T = 0;
  float* conv_w = nullptr;   // [C] folded
  float conv_bias = 0.f;
  float* wih = nullptr;      // [8*hid][bins]  (forward rows then reverse rows)
  float* bih = nullptr;      // [8*hid]        bias_ih + bias_hh
  float* whh = nullptr;      // [2][4*hid][hid]
  float* wd = nullptr;       // [bins][2*hid]
  float* dscale = nullptr;   // [bins]  BatchNorm1d scale
  float* dshift = nullptr;   // [bins]  scale*linear_bias + BatchNorm1d shift
  float* l0 = nullptr;       // [N][bins][T]  1x1 convolution, pre-activation
  float* xp = nullptr;       // [N][T][8*hid]
  float* hs = nullptr;       // [N][T][2*hid]
  float* y = nullptr;        // [bins][N][T]  the branch output at half resolution
};

struct BaseNetPlan {
  std::string prefix;
  int n = 0, H = 0, W = 0;
  ConvLayer enc1, enc_a[4], enc_b[4], aspp1, aspp2, aspp_d[3], bott, dec[4];   // dec[0]=dec4 .. dec[3]=dec1
  LstmPlan lstm;
  // A decoder is fused when its plan produces its up-sampled input channels inside the row kernel
  // (TcConv::fuses_upsample); its concat buffer then holds only the reduction channels no kernel produces on the fly.
  //   dec2 reduces over [up(d3) 4n | e2 2n]: cat2 = [up(d3) 4n | e2 2n], or [e2 2n] when fused.
  //   dec1 reduces over [up(d2) Up | e1 n | zeros up to Lp = round_up(Up + n, 16) | up(lstm) 1 + 15 zeros], where
  //   d2 = [h 2n | zeros up to Up = round_up(2n, 32)] (whole chunks, which the row kernel can up-sample): cat1 holds
  //   channels [fused1 ? Up : 0, Lp + 16) of it.  up(lstm) is up-sampled from lstm.y (half resolution, fp32 plane) into
  //   its group by a small kernel.  When dec1 is fused and n % 32 == 0 the group is instead an 8-channel buffer lstm_up
  //   of its own, so that cat1 = [e1 n] stays dense for enc2.conv1; the row kernel reads it as its last chunk through a
  //   second tensor map whose box TMA zero-fills.
  bool fused2 = false, fused1 = false;   // dec2 / dec1 fuse their upsample
  bool dot2 = false;                     // dec2's epilogue computes the LSTM branch's 1x1 input convolution (fuses_dot)
  bool lstm_own = false;                 // the up(lstm) group is lstm_up, not in cat1
  int lstm_coff = 0;                     // channel offset of the up(lstm) group in cat1 (when not lstm_own)
  Buffer cat1, t2, cat2, t3, cat3, t4, cat4, t5, e5, pool, f1, acat, ao, d4, d3, d2, lstm_up;
};

struct Config {
  int device = 0;
  int n_fft = 2048, hop = 1024, nout = 32, nout_lstm = 128, cropsize = 256, max_batch = 4;
  int offset = 64;
  int conv_mode = 0;   // 0: wgmma where eligible, 1: CUDA-core kernel everywhere (validation)
};

// Every method but the constructor and the destructor runs on the current device, which the caller makes cfg().device;
// the methods that run the net (predict_mask, separate_windows, separate, separate_wave[_host], validation_loss) need
// ready().  api.cu does both for every entry point.
class Engine {
 public:
  explicit Engine(const Config& cfg);
  ~Engine();

  std::string err;

  bool load_tensor(const char* name, int dtype, int ndim, const int64_t* shape, const void* data);
  bool finalize();
  bool ready() const { return finalized_; }

  // ---- reference-surface operations (device pointers) ----
  bool stft(const float* wave, int64_t L, float2* spec, int64_t T, float* absmax, cudaStream_t s);
  bool istft(const float2* spec, const float* mask, int64_t T, float* wave_a, float* wave_b, cudaStream_t s);
  bool stft_range(const float* wave, int64_t L, float2* spec, int64_t T, int64_t t0, int64_t t1, cudaStream_t s);
  bool normaliser_range(const float2* spec, int64_t T, int64_t t0, int64_t t1, float* out, cudaStream_t s);
  bool istft_range(const float2* spec, const float* mask, int64_t T, int64_t k0, int64_t k1, float* wave_a,
                   float* wave_b, cudaStream_t s);
  bool predict_mask(const float* mag, int N, float* mask_out, int offset, cudaStream_t s);
  // windows [first, first+count) of the padded spectrogram -> mask frames; see include/vr_b200.h
  bool separate_windows(const float2* spec, int64_t T, const float* norm, int pad_l, int first, int count,
                        float* mask, int64_t mask_T, int64_t frame_shift, int accumulate, cudaStream_t s,
                        bool final_pass = false);
  bool separate(const float2* spec, int64_t T, int tta, float* mask, cudaStream_t s);
  bool apply_mask(const float2* spec, const float* mask, int64_t T, float2* y, float2* v, cudaStream_t s);
  // --postprocess: per-frame minimum of mask [2][bins][T], then the mask pulled towards 1 by per-frame weights
  bool mask_frame_min(const float* mask, int64_t T, float* frame_min, cudaStream_t s);
  bool mask_apply_weight(float* mask, int64_t T, const float* weight, cudaStream_t s);
  bool separate_wave(const float* wave, int64_t L, int tta, float* inst, float* voc, cudaStream_t s);
  // img_inst / img_voc: HOST [bins][T][3] uint8 spectrogram images of the two stems, or nullptr for none
  bool separate_wave_host(const float* wave, int64_t L, int tta, float* inst, float* voc, cudaStream_t s,
                          unsigned char* img_inst = nullptr, unsigned char* img_voc = nullptr);
  // spectrogram images of mask * spec and (1 - mask) * spec (mask == nullptr: of spec itself, img_b unused)
  bool spec_image(const float2* spec, const float* mask, int64_t T, unsigned char* img_a, unsigned char* img_b,
                  cudaStream_t s);
  // dataset tools: image of the vocal residual of a track pair, and out = a - b; see include/vr_b200.h
  bool vocal_image(const float2* spec_x, const float2* spec_y, int64_t T, unsigned char* img, cudaStream_t s);
  bool spec_sub(const float2* a, const float2* b, int64_t T, float2* out, cudaStream_t s);
  // evaluate.py --oracle: the ideal instruments mask of a (mixture, instruments) pair; see vr_oracle_mask
  bool oracle_mask(const float2* spec_x, const float2* spec_y, int64_t T, int kind, float* mask, cudaStream_t s);
  bool normaliser(const float2* spec, int64_t T, int mode, float* out, cudaStream_t s);
  // validation loss of one (mixture, instruments) pair; see vr_validation_loss in include/vr_b200.h
  bool validation_loss(const float2* spec_x, const float2* spec_y, int64_t T, float* coef_out, double* window_sums,
                       cudaStream_t s);
  // --wiener_iterations: EM refinement of the stems' spectrograms y / v in place; see vr_wiener in include/vr_b200.h
  bool wiener(const float2* spec, float2* y, float2* v, int64_t T, int iterations, cudaStream_t s);

  // debug / tests: run one reference Conv2DBNActiv-shaped layer through a chosen kernel
  bool debug_conv(const float* x_nchw, int N, int Cin, int H, int W, const float* w, const float* bias, int Cout,
                  int k, int stride, int dil_h, int dil_w, int act, int use_tc, float* y_nchw, cudaStream_t s);
  bool debug_decoder(const float* low_nchw, int N, int Cl, int h, int w, const float* skip_nchw, int Cs, const float* wgt,
                     const float* bias, int Cout, int act, int fused, float* y_nchw, cudaStream_t s);
  // debug / tests: images [n0, n0 + n) of an activation buffer or LSTM plane as the last forward left it; see
  // vr_debug_tensor in include/vr_b200.h.  out == nullptr: only shape4 is filled.
  bool debug_tensor(const std::string& name, int n0, int n, float* out, int64_t* shape4, cudaStream_t s);

  const Config& cfg() const { return cfg_; }
  int bins() const { return cfg_.n_fft / 2 + 1; }
  int roi() const { int r = cfg_.cropsize - 2 * cfg_.offset; return r == 0 ? cfg_.cropsize : r; }
  int64_t launches = 0;   // kernels launched by this engine (bench 'gpu_launches'); counted by timed and run_conv

  // optional CUDA-event timing of every launch (bench.py roofline object and --layers table)
  void profile_enable(bool on);
  // sums over the events recorded since enable: [0] tensor-core conv ms, [1] tensor-core conv algorithmic FLOPs,
  // [2] tensor-core launches, [3] CUDA-core conv ms, [4] CUDA-core conv FLOPs, [5] CUDA-core launches
  bool profile_read(double* out6);
  bool profile_dump(std::string& text);   // one line per profiled launch: name N H W tc ms gflop

 private:
  Config cfg_;
  bool finalized_ = false;
  bool warned_simt_ = false;   // the CUDA-core fallback warning was printed
  std::map<std::string, HostTensor> sd_;
  Arena arena_;   // weights, tables and activation buffers
  // tc: 1 = tensor-core convolution, 0 = CUDA-core convolution, 2 = any other kernel of the path
  struct ProfRec { cudaEvent_t a, b; double flops; int tc; std::string name; int N, H, W; };
  bool profiling_ = false;
  std::vector<ProfRec> prof_;
  int prof_begin(const std::string& name, int kind, double flops, int N, int H, int W, cudaStream_t s);
  void prof_end(int idx, cudaStream_t s);
  // Every launch that is not a convolution (those go through run_conv): `launch` enqueues `kernels` kernels on s,
  // which are counted and, while profiling is on, bracketed by one CUDA-event pair.
  template <class F>
  bool timed(const char* name, int kernels, int N, int H, int W, cudaStream_t s, F&& launch) {
    launches += kernels;
    const int i = prof_begin(name, 2, 0.0, N, H, W, s);
    const bool ok = launch();
    prof_end(i, s);
    return ok;
  }

  // whole-track workspaces
  GrowArray<float2> ws_spec_;
  GrowArray<float> ws_mask_;
  GrowArray<float> ws_frames_;
  GrowArray<float> ws_wave_;   // [2][L] in + 2 x [2][Lo] out (host-buffer entry)
  float* ws_norm_ = nullptr;            // [4] floats: absmax, lexmax-abs
  unsigned long long* ws_lex_ = nullptr;
  unsigned int* ws_img_range_ = nullptr;   // [4] min / max keys of the spectrogram image pass (first use)
  GrowArray<unsigned char> ws_img_;   // two [bins][T][3] images (host-buffer entry)
  GrowArray<double> ws_val_;   // per-slice partial sums of the validation loss
  GrowArray<double> ws_wiener_;   // per-slice moments, per-bin covariances and the scale of the Wiener filter

  // the high-band BaseNets of stages 1-2 run on their own stream next to the low-band chain (independent until
  // stage 3, lib/nets.py:88-99); disabled while per-kernel profiling is on so event timings stay per-kernel
  cudaStream_t s_hi_ = nullptr;
  // host-buffer entry: finished output spans are copied back on their own stream while the next window batch computes
  cudaStream_t s_copy_ = nullptr;
  cudaEvent_t ev_span_ = nullptr;
  std::function<bool(int64_t)> on_frames_final_;   // called after a batch of the last pass: mask frames [0, f) are final
  cudaEvent_t ev_fork_ = nullptr, ev_join_ = nullptr, ev_lstm_fork_ = nullptr, ev_lstm_join_ = nullptr;

  float2* twiddle_ = nullptr;
  float* window_ = nullptr;

  Buffer in3_;                 // (Nb, max_bin, W, C3): [aux2 | aux1 | x | pad]
  int pos_aux2_ = 0, pos_aux1_ = 0, pos_x_ = 0;
  Buffer o1_, o2_;             // low-band BaseNet outputs before the 1x1 bridge (stage 1 / stage 2)
  Buffer f3_;                  // stage-3 output (Nb, max_bin, W, nout)
  BaseNetPlan nets_[5];        // stg1_low, stg1_high, stg2_low, stg2_high, stg3_full
  int last_n_ = 0;             // window batch of the last forward: the row stride of every LSTM plane y
  ConvLayer bridge1_, bridge2_;
  float* out_w_ = nullptr;     // [2][nout]

  // zero-filled allocation in `arena`, holding a copy of host[0, bytes) when host is given; nullptr (err set) on failure
  void* dalloc(Arena& arena, size_t bytes, const void* host = nullptr);
  Buffer make_buffer(Arena& arena, int N, int H, int W, int C, int pad_w = 0);
  bool need(const std::string& key, std::initializer_list<int64_t> shape, const HostTensor** out);
  // The eval-mode BatchNorm at `bn` (its weight, bias, running_mean, running_var and num_batches_tracked, C channels)
  // after a layer with bias pre_bias (nullptr: none) as y = scale * x + shift per channel, in double:
  // scale = gamma / sqrt(var + eps), shift = scale * (pre_bias - mean) + beta.
  bool fold_bn(const std::string& bn, int C, const float* pre_bias, std::vector<double>& scale,
               std::vector<double>& shift);
  // H x W: the layer's output maps, from which tc_prepare chooses its kernel (rows_wide: see tc_prepare).
  // The layer's padded input width is perm.size().
  bool make_conv(ConvLayer& L, const std::string& prefix, const std::vector<int>& perm, int k, int stride, int dh,
                 int dw, int act, int H, int W, bool rows_wide = false);
  // Makes the device weights of L's kernel from its host-packed weights wp [tap][CinPad][CoutPad] and bias bp
  // [CoutPad]: use_tc lets tc_prepare plan a tensor-core kernel for output maps of H x W; a layer left on the CUDA-core
  // kernel gets wp / bp uploaded to L.w / L.bias in `arena`.
  bool prepare_conv(ConvLayer& L, Arena& arena, const std::vector<float>& wp, const std::vector<float>& bp,
                    bool use_tc, int H, int W, bool rows_wide);
  // test hooks: pack_conv and prepare_conv of the caller's device weights / bias, unscaled
  bool debug_weights(ConvLayer& L, Arena& arena, const float* w, const float* bias, int Cout, int Cin,
                     const std::vector<int>& perm, bool use_tc, int H, int W, bool rows_wide, cudaStream_t s);
  bool to_nchw(const ActView& v, int C, float* y_nchw, cudaStream_t s);
  bool build_basenet(BaseNetPlan& P, const std::string& prefix, const std::vector<int>& in_perm, int n, int H, int W,
                     int nin_lstm, int nout_lstm);
  bool run_conv(const ConvLayer& L, const ActView& in, const ActView& out, cudaStream_t s, const ConvFusion& f = {});
  // Decoder (lib/layers.py:51-64): conv(cat[up(low), skip]) -> out.  fused: the row kernel produces up(low) itself and
  // `cat` holds only the skip channels; else up(low) is first written into channels [0, low.C) of `cat`.
  bool run_decoder(const ConvLayer& L, const ActView& low, const Buffer& cat, int N, const ActView& out, bool fused,
                   cudaStream_t s, ConvFusion f = {});
  // mask != nullptr: dec1 writes the network's mask in its epilogue instead of `out` (dec1.tc->fuses_mask)
  bool run_basenet(BaseNetPlan& P, const ActView& in, const ActView& out, int N, cudaStream_t s,
                   cudaStream_t side = nullptr, const MaskOutParams* mask = nullptr);
  // in3_ x-channels already packed for N windows -> the mask of frames [mask.offset, W - mask.offset) of every window,
  // written as mask describes (mask.f3 = f3_.all(N))
  bool forward(int N, const MaskOutParams& mask, cudaStream_t s);
  bool ensure_ws(int64_t T);
  bool ck(cudaError_t e, const char* what);
};

// conv_tc.cu: plans L.tc for output maps of H x W (left null when the layer stays on the CUDA-core kernel) and uploads
// its weights from the host-packed w [tap][L.CinPad][L.CoutPad] and bias [L.Cout].
// rows_wide: the row kernel may use its 64-output-channel tile (decoder layers whose upsample it fuses).
bool tc_prepare(ConvLayer& L, const float* w, const float* bias, int H, int W, bool rows_wide, std::string& err);
cudaError_t tc_launch(const ConvLayer& L, const ActView& in, const ActView& out, cudaStream_t s, std::string& err,
                      const ConvFusion& f);

}  // namespace vr
