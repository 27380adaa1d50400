// extern "C" surface of libvr_b200.so; declarations and the reference call each entry replaces are in
// include/vr_b200.h.
#include <stdio.h>
#include <string.h>

#include <string>

#include "../../include/vr_b200.h"
#include "engine.h"
#include "kernels.h"
#include "tc_plan.h"

struct vr_ctx {
  vr::Engine* eng;
  std::string err;
};

static std::string g_create_err;

// The calls that need no model (resampling, FLAC and PCM, BSS Eval) take a ctx that may be NULL: audio is usually
// loaded, and stems scored, before a model context exists.  Such a call then runs on the calling thread's current
// device, and its error message is read with vr_last_error(NULL).
static int fail(vr_ctx* c, const std::string& m) {
  (c ? c->err : g_create_err) = m;
  return -1;
}
static void use_device(const vr_ctx* c) {
  if (c && c->eng) cudaSetDevice(c->eng->cfg().device);
}
static int done(vr_ctx* c, bool ok) {
  if (ok) return 0;
  c->err = c->eng->err;
  return -1;
}
static int cuda_result(vr_ctx* c, const char* what, cudaError_t e) {
  return e == cudaSuccess ? 0 : fail(c, std::string(what) + ": " + cudaGetErrorString(e));
}
// Every entry point that takes a context runs on the context's device ...
#define CHECK_CTX(c)                  \
  if (!(c) || !(c)->eng) return -2;   \
  use_device(c);
// ... and one that runs the net needs its weights finalized.
#define CHECK_NET(c) \
  CHECK_CTX(c)       \
  if (!(c)->eng->ready()) return fail(c, "weights not finalized");

extern "C" {

int vr_create(const vr_config* cfg, vr_ctx** out) {
  if (!cfg || !out) return -2;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    g_create_err = "no CUDA device visible: libvr_b200 has no CPU path";
    return -1;
  }
  if (cfg->device < 0 || cfg->device >= ndev) {
    g_create_err = "invalid device ordinal";
    return -1;
  }
  int nf = cfg->n_fft;
  if (nf < 64 || nf > 4096 || (nf & (nf - 1))) {
    g_create_err = "n_fft must be a power of two in [64, 4096]";
    return -1;
  }
  if (cfg->hop_length <= 0 || cfg->hop_length > nf) {
    g_create_err = "hop_length must be in (0, n_fft]";
    return -1;
  }
  if (cfg->max_batch <= 0 || cfg->cropsize <= 0) {
    g_create_err = "max_batch and cropsize must be positive";
    return -1;
  }
  vr::Config c;
  c.device = cfg->device; c.n_fft = cfg->n_fft; c.hop = cfg->hop_length; c.nout = cfg->nout;
  c.nout_lstm = cfg->nout_lstm; c.cropsize = cfg->cropsize; c.max_batch = cfg->max_batch;
  c.conv_mode = cfg->conv_mode;
  vr_ctx* ctx = new vr_ctx();
  ctx->eng = new vr::Engine(c);
  if (!ctx->eng->err.empty()) {
    g_create_err = ctx->eng->err;
    delete ctx->eng;
    delete ctx;
    return -1;
  }
  *out = ctx;
  return 0;
}

void vr_destroy(vr_ctx* ctx) {
  if (!ctx) return;
  delete ctx->eng;
  delete ctx;
}

const char* vr_last_error(const vr_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

int vr_load_tensor(vr_ctx* ctx, const char* name, int32_t dtype, int32_t ndim, const int64_t* shape,
                   const void* host_data) {
  CHECK_CTX(ctx);
  if (!name || (!host_data) || ndim < 0 || ndim > 8) return fail(ctx, "vr_load_tensor: bad arguments");
  return done(ctx, ctx->eng->load_tensor(name, dtype, ndim, shape, host_data));
}

int vr_finalize_weights(vr_ctx* ctx) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->finalize());
}

int vr_stft(vr_ctx* ctx, const float* wave, int64_t L, void* spec, int64_t T, float* absmax, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->stft(wave, L, (float2*)spec, T, absmax, (cudaStream_t)stream));
}

int vr_istft(vr_ctx* ctx, const void* spec, int64_t T, float* wave, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->istft((const float2*)spec, nullptr, T, wave, nullptr, (cudaStream_t)stream));
}

int vr_predict_mask(vr_ctx* ctx, const float* mag, int32_t N, float* mask, void* stream) {
  CHECK_NET(ctx);
  return done(ctx, ctx->eng->predict_mask(mag, N, mask, ctx->eng->cfg().offset, (cudaStream_t)stream));
}

int vr_forward(vr_ctx* ctx, const float* mag, int32_t N, float* mask, void* stream) {
  CHECK_NET(ctx);
  return done(ctx, ctx->eng->predict_mask(mag, N, mask, 0, (cudaStream_t)stream));
}

int vr_normaliser(vr_ctx* ctx, const void* spec, int64_t T, int32_t norm_mode, float* out, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->normaliser((const float2*)spec, T, norm_mode, out, (cudaStream_t)stream));
}

int vr_separate_windows(vr_ctx* ctx, const void* spec, int64_t T, const float* norm, int32_t pad_l,
                        int32_t first_window, int32_t n_windows, float* mask, int64_t mask_T, int64_t frame_shift,
                        int32_t accumulate, void* stream) {
  CHECK_NET(ctx);
  return done(ctx, ctx->eng->separate_windows((const float2*)spec, T, norm, pad_l, first_window, n_windows, mask,
                                              mask_T, frame_shift, accumulate, (cudaStream_t)stream));
}

int vr_separate(vr_ctx* ctx, const void* spec, int64_t T, int32_t tta, float* mask, void* stream) {
  CHECK_NET(ctx);
  return done(ctx, ctx->eng->separate((const float2*)spec, T, tta, mask, (cudaStream_t)stream));
}

int vr_apply_mask(vr_ctx* ctx, const void* spec, const float* mask, int64_t T, void* y_spec, void* v_spec,
                  void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->apply_mask((const float2*)spec, mask, T, (float2*)y_spec, (float2*)v_spec,
                                        (cudaStream_t)stream));
}

int vr_mask_frame_min(vr_ctx* ctx, const float* mask, int64_t T, float* frame_min, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->mask_frame_min(mask, T, frame_min, (cudaStream_t)stream));
}

int vr_mask_apply_weight(vr_ctx* ctx, float* mask, int64_t T, const float* weight, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->mask_apply_weight(mask, T, weight, (cudaStream_t)stream));
}

int vr_apply_mask_istft(vr_ctx* ctx, const void* spec, const float* mask, int64_t T, float* wave_inst,
                        float* wave_voc, void* stream) {
  CHECK_CTX(ctx);
  if (!mask) return fail(ctx, "vr_apply_mask_istft: mask is NULL");
  return done(ctx, ctx->eng->istft((const float2*)spec, mask, T, wave_inst, wave_voc, (cudaStream_t)stream));
}

int vr_stft_range(vr_ctx* ctx, const float* wave, int64_t L, void* spec, int64_t T, int64_t t0, int64_t t1,
                  void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->stft_range(wave, L, (float2*)spec, T, t0, t1, (cudaStream_t)stream));
}

int vr_normaliser_range(vr_ctx* ctx, const void* spec, int64_t T, int64_t t0, int64_t t1, float* out, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->normaliser_range((const float2*)spec, T, t0, t1, out, (cudaStream_t)stream));
}

int vr_apply_mask_istft_range(vr_ctx* ctx, const void* spec, const float* mask, int64_t T, int64_t k0, int64_t k1,
                              float* wave_inst, float* wave_voc, void* stream) {
  CHECK_CTX(ctx);
  if (!mask) return fail(ctx, "vr_apply_mask_istft_range: mask is NULL");
  return done(ctx, ctx->eng->istft_range((const float2*)spec, mask, T, k0, k1, wave_inst, wave_voc,
                                         (cudaStream_t)stream));
}

int vr_separate_wave(vr_ctx* ctx, const float* wave, int64_t L, int32_t tta, float* wave_inst, float* wave_voc,
                     void* stream) {
  CHECK_NET(ctx);
  return done(ctx, ctx->eng->separate_wave(wave, L, tta, wave_inst, wave_voc, (cudaStream_t)stream));
}

int vr_separate_wave_host(vr_ctx* ctx, const float* wave_host, int64_t L, int32_t tta, float* inst_host,
                          float* voc_host, void* stream) {
  CHECK_NET(ctx);
  return done(ctx, ctx->eng->separate_wave_host(wave_host, L, tta, inst_host, voc_host, (cudaStream_t)stream));
}

int vr_separate_wave_host_images(vr_ctx* ctx, const float* wave_host, int64_t L, int32_t tta, float* inst_host,
                                 float* voc_host, uint8_t* img_inst_host, uint8_t* img_voc_host, void* stream) {
  CHECK_NET(ctx);
  return done(ctx, ctx->eng->separate_wave_host(wave_host, L, tta, inst_host, voc_host, (cudaStream_t)stream,
                                                img_inst_host, img_voc_host));
}

int vr_spec_image(vr_ctx* ctx, const void* spec, const float* mask, int64_t T, uint8_t* img_a, uint8_t* img_b,
                  void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->spec_image((const float2*)spec, mask, T, img_a, img_b, (cudaStream_t)stream));
}

int vr_vocal_image(vr_ctx* ctx, const void* spec_x, const void* spec_y, int64_t T, uint8_t* img, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->vocal_image((const float2*)spec_x, (const float2*)spec_y, T, img, (cudaStream_t)stream));
}

int vr_spec_sub(vr_ctx* ctx, const void* a, const void* b, int64_t T, void* out, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->spec_sub((const float2*)a, (const float2*)b, T, (float2*)out, (cudaStream_t)stream));
}

int vr_oracle_mask(vr_ctx* ctx, const void* spec_x, const void* spec_y, int64_t T, int32_t kind, float* mask,
                   void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->oracle_mask((const float2*)spec_x, (const float2*)spec_y, T, kind, mask,
                                         (cudaStream_t)stream));
}

int vr_validation_loss(vr_ctx* ctx, const void* spec_x, const void* spec_y, int64_t T, float* coef_out,
                       double* window_sums, void* stream) {
  CHECK_NET(ctx);
  return done(ctx, ctx->eng->validation_loss((const float2*)spec_x, (const float2*)spec_y, T, coef_out, window_sums,
                                             (cudaStream_t)stream));
}

int vr_wiener(vr_ctx* ctx, const void* spec, void* y_spec, void* v_spec, int64_t T, int32_t iterations, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->wiener((const float2*)spec, (float2*)y_spec, (float2*)v_spec, T, iterations,
                                    (cudaStream_t)stream));
}

int vr_resample(vr_ctx* ctx, const float* x, int32_t channels, int64_t n_in, float* y, int64_t n_out, double sample_ratio,
                const double* win, const double* delta, int32_t nwin, int32_t table_per_crossing, void* stream) {
  if (!x || !y || !win || !delta) return fail(ctx, "vr_resample: null pointer");
  if (n_out != (int64_t)((double)n_in * sample_ratio))
    return fail(ctx, "vr_resample: n_out must be int(n_in * sample_ratio) (resampy.core.resample)");
  use_device(ctx);
  return cuda_result(ctx, "vr_resample",
                     vr::launch_resample_sinc(x, channels, n_in, y, n_out, sample_ratio, win, delta, nwin,
                                              table_per_crossing, (cudaStream_t)stream));
}

int vr_flac_scan(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, int64_t begin, int64_t* cands, int32_t max_cands,
                 int32_t* count, void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_flac_scan",
                     vr::launch_flac_scan(data, n_bytes, begin, cands, max_cands, count, (cudaStream_t)stream));
}

int vr_flac_decode(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, const int64_t* frames, int32_t n_frames,
                   int32_t channels, int64_t n_samples, float* out, int64_t* status, void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_flac_decode",
                     vr::launch_flac_decode(data, n_bytes, frames, n_frames, channels, n_samples, out, status,
                                            (cudaStream_t)stream));
}

int64_t vr_mp3_workspace(int64_t n_frames, int32_t channels, int64_t md_bytes) {
  return vr::mp3_workspace_bytes(n_frames, channels, md_bytes);
}

int vr_mp3_scan(vr_ctx* ctx, const uint8_t* data, int64_t begin, int64_t end, int64_t* cands, int32_t max_cands,
                int32_t* count, void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_mp3_scan", vr::launch_mp3_scan(data, begin, end, cands, max_cands, count,
                                                             (cudaStream_t)stream));
}

int vr_mp3_decode(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, const int64_t* frames, const int64_t* md_off,
                  int32_t n_frames, int32_t channels, int32_t rate_index, int64_t md_bytes, void* workspace,
                  int64_t workspace_bytes, float* out, int64_t* status, void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_mp3_decode",
                     vr::launch_mp3_decode(data, n_bytes, frames, md_off, n_frames, channels, rate_index, md_bytes,
                                           workspace, workspace_bytes, out, status, (cudaStream_t)stream));
}

int64_t vr_aac_workspace(int64_t n_packets, int32_t channels) { return vr::aac_workspace_bytes(n_packets, channels); }

int vr_aac_decode(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, const int64_t* table, int32_t n_packets,
                  int32_t channels, int32_t rate_index, void* workspace, int64_t workspace_bytes, float* out,
                  int64_t* status, void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_aac_decode",
                     vr::launch_aac_decode(data, n_bytes, table, n_packets, channels, rate_index, workspace,
                                           workspace_bytes, out, status, (cudaStream_t)stream));
}

int64_t vr_vorbis_workspace(int64_t n_packets, int32_t channels, int64_t slot_floats) {
  return vr::vorbis_workspace_bytes(n_packets, channels, slot_floats);
}

int vr_vorbis_decode(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, const int64_t* table, int32_t n_packets,
                     const int32_t* setup, int32_t setup_words, int32_t channels, int32_t n_codes, int64_t slot_floats,
                     void* workspace, int64_t workspace_bytes, float* out, int64_t n_out, int64_t* status,
                     void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_vorbis_decode",
                     vr::launch_vorbis_decode(data, n_bytes, table, n_packets, setup, setup_words, channels, n_codes,
                                              slot_floats, workspace, workspace_bytes, out, n_out, status,
                                              (cudaStream_t)stream));
}

int vr_flac_encode_analyse(vr_ctx* ctx, const float* x, int32_t channels, int64_t n, int32_t rate_code, int32_t bits,
                           void* pcm, int32_t* plan, void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_flac_encode_analyse",
                     vr::launch_flac_encode_analyse(x, channels, n, rate_code, bits, pcm, plan, (cudaStream_t)stream));
}

int vr_flac_encode_pack(vr_ctx* ctx, const void* pcm, int32_t channels, int64_t n, int32_t bits, const int32_t* plan,
                        const int64_t* offsets, int32_t rate_code, int32_t rate_value, uint8_t* out, int32_t* status,
                        void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_flac_encode_pack",
                     vr::launch_flac_encode_pack(pcm, channels, n, bits, plan, offsets, rate_code, rate_value, out,
                                                 status, (cudaStream_t)stream));
}

int vr_pcm_pack(vr_ctx* ctx, const float* x, int32_t channels, int64_t n, int32_t bits, uint8_t* out, void* stream) {
  use_device(ctx);
  return cuda_result(ctx, "vr_pcm_pack", vr::launch_pcm_pack(x, channels, n, bits, out, (cudaStream_t)stream));
}

static int64_t bss_workspace(bool framewise, int32_t K, int32_t C, int64_t N, int32_t L, int64_t window, int64_t hop,
                             int32_t frames_per_batch) {
  std::string err;
  const int64_t bytes = vr::bss_eval_workspace(framewise, K, C, N, L, window, hop, frames_per_batch, err);
  if (bytes < 0) fail(nullptr, err);
  return bytes;
}

static int bss_run(vr_ctx* ctx, bool framewise, const float* refs, const float* ests, int32_t K, int32_t C, int64_t N,
                   int32_t L, int64_t window, int64_t hop, int32_t frames_per_batch, void* workspace,
                   int64_t workspace_bytes, double* frames_host, double* corr_host, double* loading_host,
                   double* phase_ms, void* stream) {
  use_device(ctx);
  std::string err;
  return vr::bss_eval(framewise, refs, ests, K, C, N, L, window, hop, frames_per_batch, workspace, workspace_bytes,
                      frames_host, corr_host, loading_host, phase_ms, (cudaStream_t)stream, err)
             ? 0
             : fail(ctx, err);
}

int64_t vr_bss_eval_workspace(int32_t K, int32_t C, int64_t N, int32_t L, int64_t window, int64_t hop) {
  return bss_workspace(false, K, C, N, L, window, hop, 1);
}

int vr_bss_eval(vr_ctx* ctx, const float* refs, const float* ests, int32_t K, int32_t C, int64_t N, int32_t L,
                int64_t window, int64_t hop, void* workspace, int64_t workspace_bytes, double* frames_host,
                double* corr_host, double* loading_host, double* phase_ms, void* stream) {
  return bss_run(ctx, false, refs, ests, K, C, N, L, window, hop, 1, workspace, workspace_bytes, frames_host,
                 corr_host, loading_host, phase_ms, stream);
}

int64_t vr_bss_eval_framewise_workspace(int32_t K, int32_t C, int64_t N, int32_t L, int64_t window, int64_t hop,
                                        int32_t frames_per_batch) {
  return bss_workspace(true, K, C, N, L, window, hop, frames_per_batch);
}

int vr_bss_eval_framewise(vr_ctx* ctx, const float* refs, const float* ests, int32_t K, int32_t C, int64_t N,
                          int32_t L, int64_t window, int64_t hop, int32_t frames_per_batch, void* workspace,
                          int64_t workspace_bytes, double* frames_host, double* corr_host, double* loading_host,
                          double* phase_ms, void* stream) {
  return bss_run(ctx, true, refs, ests, K, C, N, L, window, hop, frames_per_batch, workspace, workspace_bytes,
                 frames_host, corr_host, loading_host, phase_ms, stream);
}

int vr_shared_alloc(vr_ctx* ctx, int64_t bytes, void** dev_ptr, unsigned char* handle64) {
  CHECK_CTX(ctx);
  if (!dev_ptr || !handle64 || bytes <= 0) return fail(ctx, "vr_shared_alloc: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle is 64 bytes");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, (size_t)bytes);
  if (e != cudaSuccess) return fail(ctx, std::string("vr_shared_alloc: cudaMalloc: ") + cudaGetErrorString(e));
  cudaIpcMemHandle_t h;
  e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    return fail(ctx, std::string("vr_shared_alloc: cudaIpcGetMemHandle: ") + cudaGetErrorString(e));
  }
  memcpy(handle64, &h, 64);
  *dev_ptr = p;
  return 0;
}

int vr_shared_open(vr_ctx* ctx, const unsigned char* handle64, void** dev_ptr) {
  CHECK_CTX(ctx);
  if (!dev_ptr || !handle64) return fail(ctx, "vr_shared_open: bad arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return fail(ctx, std::string("vr_shared_open: cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
  *dev_ptr = p;
  return 0;
}

int vr_shared_close(vr_ctx* ctx, void* dev_ptr, int32_t owner) {
  CHECK_CTX(ctx);
  if (!dev_ptr) return 0;
  cudaError_t e = owner ? cudaFree(dev_ptr) : cudaIpcCloseMemHandle(dev_ptr);
  if (e != cudaSuccess) return fail(ctx, std::string("vr_shared_close: ") + cudaGetErrorString(e));
  return 0;
}

int64_t vr_launch_count(const vr_ctx* ctx) { return ctx && ctx->eng ? ctx->eng->launches : 0; }

int vr_profile_enable(vr_ctx* ctx, int32_t on) {
  CHECK_CTX(ctx);
  ctx->eng->profile_enable(on != 0);
  return 0;
}

int vr_profile_read(vr_ctx* ctx, double* out6) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->profile_read(out6));
}

int vr_profile_dump(vr_ctx* ctx, char* text, int64_t cap, int64_t* needed) {
  CHECK_CTX(ctx);
  std::string t;
  if (!ctx->eng->profile_dump(t)) return done(ctx, false);
  if (needed) *needed = (int64_t)t.size() + 1;
  if (text && cap > 0) {
    const size_t n = t.size() < (size_t)cap - 1 ? t.size() : (size_t)cap - 1;
    memcpy(text, t.data(), n);
    text[n] = 0;
  }
  return 0;
}

int vr_debug_conv(vr_ctx* ctx, const float* x, int32_t N, int32_t Cin, int32_t H, int32_t W, const float* w,
                  const float* bias, int32_t Cout, int32_t k, int32_t stride, int32_t dil_h, int32_t dil_w, int32_t act,
                  int32_t use_tc, float* y, void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->debug_conv(x, N, Cin, H, W, w, bias, Cout, k, stride, dil_h, dil_w, act, use_tc, y,
                                        (cudaStream_t)stream));
}

int vr_debug_decoder(vr_ctx* ctx, const float* low, int32_t N, int32_t Cl, int32_t h, int32_t w, const float* skip,
                     int32_t Cs, const float* wgt, const float* bias, int32_t Cout, int32_t act, int32_t fused, float* y,
                     void* stream) {
  CHECK_CTX(ctx);
  return done(ctx, ctx->eng->debug_decoder(low, N, Cl, h, w, skip, Cs, wgt, bias, Cout, act, fused, y,
                                           (cudaStream_t)stream));
}

int vr_debug_tensor(vr_ctx* ctx, const char* name, int32_t n0, int32_t n, float* out, int64_t* shape4, void* stream) {
  CHECK_NET(ctx);
  if (!name || !shape4) return fail(ctx, "vr_debug_tensor: name and shape4 are required");
  return done(ctx, ctx->eng->debug_tensor(name, n0, n, out, shape4, (cudaStream_t)stream));
}

int vr_debug_set(int32_t key, int32_t value) {
  int* knob = key == 0 ? &vr::g_debug.trace : key == 2 ? &vr::g_debug.rows_wide : key == 3 ? &vr::g_debug.halo
            : key == 6 ? &vr::g_debug.kskip : key == 7 ? &vr::g_debug.crop_mask
            : key == 8 ? &vr::g_debug.pair : key == 9 ? &vr::g_debug.pair_stores : nullptr;
  if (!knob) return -1;
  *knob = value;
  return 0;
}

int vr_debug_last_conv(int32_t* out8) {
  if (!out8) return -1;
  const vr::TcLastConv& c = vr::g_last_conv;
  const int32_t v[8] = {c.kind, c.KB, c.BN, c.n_tiles, c.pair, c.MB, c.up, c.vec16};
  memcpy(out8, v, sizeof(v));
  return 0;
}

int64_t vr_debug_trace(uint64_t* host_out, int64_t capacity) {
  return vr::tc_rows_read_trace((unsigned long long*)host_out, (long long)capacity);
}

}  // extern "C"
