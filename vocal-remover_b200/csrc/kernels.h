// Host-side launch prototypes for the hand-written sm_90a kernels of the hot path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "common.cuh"

namespace vr {

// ---- convolution (conv_simt.cu / conv_tc.cu) -------------------------------------------------
cudaError_t launch_conv_simt(const ConvParams& p, cudaStream_t stream);

// ---- bandwidth kernels (elementwise.cu) ------------------------------------------------------
// |X|/norm of window g = first_window + n, frame tw -> dst channels [0,2) ; spec is complex64 [2][bins][T]
cudaError_t launch_pack_mag_from_spec(const float2* spec, int bins, int64_t T, int max_bin, int W, int roi,
                                      int pad_l, int first_window, const float* norm, ActView dst,
                                      cudaStream_t stream);
// mag is float32 NCHW [N][2][bins][W] (the reference predict_mask input, lib/nets.py:124)
cudaError_t launch_pack_mag_from_float(const float* mag, int bins, int max_bin, ActView dst, cudaStream_t stream);
cudaError_t launch_nchw_to_act(const float* x, int C, ActView dst, cudaStream_t stream);
cudaError_t launch_act_to_nchw(ActView src, int C, float* y, cudaStream_t stream);
cudaError_t launch_upsample2x(ActView in, ActView out, cudaStream_t stream);
// fp32 plane in[(n) in_sn][(row) in_sh][col] (inH x inW per image) -> channel 0 of the 16- or 8-channel group `out`
// (the other channels written as zeros), same interpolation arithmetic as launch_upsample2x
cudaError_t launch_upsample2x_c1(const float* in, int inH, int inW, int64_t in_sn, int64_t in_sh, ActView out,
                                 cudaStream_t stream);
cudaError_t launch_pool_freq_mean(ActView in, ActView out, cudaStream_t stream);
cudaError_t launch_broadcast_rows(ActView in, ActView out, cudaStream_t stream);

struct MaskOutParams {
  ActView f3;          // (N, max_bin, W, nout)
  const float* w;      // [2][nout]  (CascadedNet.out.weight, lib/nets.py:79)
  float* out;
  int64_t stride_n, stride_c, stride_bin;  // element strides of the destination; frames are contiguous
  int offset;          // model.offset (64): frames [offset, W-offset) are kept (lib/nets.py:127-129)
  int64_t t_base0;     // destination frame index of frame `offset` of window 0, before stride_n is applied
  int64_t t_limit;     // frames with (t_base0 + n*roi_t + tw-offset) outside [0, t_limit) are dropped
  int roi_t;           // per-window frame advance used only for the limit test
  int accumulate;      // 1: out = (out + mask) * 0.5  (TTA average, inference.py:98)
};
cudaError_t launch_mask_out(const MaskOutParams& p, cudaStream_t stream);

// accumulate: max with what *out_absmax holds (a non-negative float) instead of starting from 0
cudaError_t launch_absmax(const float2* spec, int64_t n, float* out_absmax, cudaStream_t stream,
                          bool accumulate = false);
// max |spec[r][t]| over rows r < nrows and frames t in [t0, t1) of a [nrows][T] array
cudaError_t launch_absmax_range(const float2* spec, int nrows, int64_t T, int64_t t0, int64_t t1, float* out_absmax,
                                cudaStream_t stream);
cudaError_t launch_lexmax_abs(const float2* spec, int64_t n, unsigned long long* scratch, float* out_norm,
                              cudaStream_t stream);
cudaError_t launch_mask_frame_min(const float* mask, int rows, int64_t T, float* out, cudaStream_t stream);
cudaError_t launch_mask_apply_weight(float* mask, int rows, int64_t T, const float* weight, cudaStream_t stream);
cudaError_t launch_apply_mask(const float2* spec, const float* mask, int64_t n, float2* y, float2* v,
                              cudaStream_t stream);
// spectrogram images (reference spec_utils.spectrogram_to_image): spec / mask [2][plane] with plane = bins * T ->
// img_a / img_b [plane][3] uint8 (instruments / vocals; mask == nullptr: img_a = image of spec, img_b unused);
// range: 4 unsigned ints of scratch
cudaError_t launch_spec_image(const float2* spec, const float* mask, int64_t plane, unsigned int* range,
                              unsigned char* img_a, unsigned char* img_b, cudaStream_t stream);
// the same image of the vocal residual v = |X| - |y|, kept where v > |y| (reference lib/dataset.py:280-287), of
// spec_x / spec_y [2][plane] -> img [plane][3]; range: 4 unsigned ints of scratch
cudaError_t launch_vocal_image(const float2* spec_x, const float2* spec_y, int64_t plane, unsigned int* range,
                               unsigned char* img, cudaStream_t stream);
// out[i] = a[i] - b[i] over n complex elements
cudaError_t launch_spec_sub(const float2* a, const float2* b, int64_t n, float2* out, cudaStream_t stream);
// oracle masks (evaluate.py --oracle, DESIGN.md §12): mask[i] in [0, 1] of the mixture spec_x and the true instruments
// spec_y over n complex elements; kind 0 iam, 1 ibm, 2 irm1, 3 irm2
cudaError_t launch_oracle_mask(const float2* spec_x, const float2* spec_y, int64_t n, int kind, float* mask,
                               cudaStream_t stream);
// validation loss (reference train.py:108-134): window_sums[j] = sum over (channel, bin, frames [j*roi, (j+1)*roi) of
// the track) of |mask * |X| / coef - |y| / coef|, spec_x / spec_y [2][bins][T], mask [2][bins][n_windows * roi],
// *coef on the device; partial: validation_l1_scratch(n_windows) doubles of scratch
int64_t validation_l1_scratch(int n_windows);
cudaError_t launch_validation_l1(const float2* spec_x, const float2* spec_y, const float* mask, int bins, int64_t T,
                                 int roi, int n_windows, const float* coef, double* partial, double* window_sums,
                                 cudaStream_t stream);

// ---- multichannel Wiener filter (wiener.cu), DESIGN.md §11 ------------------------------------------------------------
// `iterations` EM refinements of the estimates y / v [2][bins][T] (complex64, in place) of the mixture spec [2][bins][T];
// scratch: wiener_scratch(bins) doubles.  1 + 3 * iterations kernels.
int64_t wiener_scratch(int bins);
cudaError_t launch_wiener(const float2* spec, float2* y, float2* v, int bins, int64_t T, int iterations,
                          double* scratch, cudaStream_t stream);

// ---- LSTM branch (lstm.cu), reference lib/layers.py:108-133 ------------------------------------
// 1x1 conv (C -> 1), pre-activation sums as an fp32 plane l0[n][bin][t] (dec2's epilogue accumulates the same sums
// instead where its plan can: ConvFusion::dot_w in engine.h, TcConv::fuses_dot)
cudaError_t launch_lstm_inconv(ActView in, const float* w, float* l0, cudaStream_t stream);
// xp[(n,t)][gates] = relu(l0[n][:][t] + conv_bias) . wih[gates][:]^T + bih   (gates = 8 * hid)
cudaError_t launch_lstm_input_projection(const float* l0, float conv_bias, const float* wih, const float* bih, float* xp,
                                         int N, int T, int bins, int gates, cudaStream_t stream);
// xp: [n][t][2][4*hid] gate pre-activations (input projection + both biases), whh: [2][4*hid][hid]
// hs: [n][t][2*hid]
cudaError_t launch_lstm_recurrence(const float* xp, const float* whh, float* hs, int N, int T, int hid,
                                   cudaStream_t stream);
// y[bin][(n,t)] = relu(scale[bin] * (wd[bin][:] . hs[(n,t)][:]) + shift[bin]),  wd: [bins][K], NT = N * T
cudaError_t launch_lstm_dense(const float* hs, const float* wd, const float* scale, const float* shift, int NT, int K,
                              int bins, float* y, cudaStream_t stream);

// ---- STFT / iSTFT (fft.cu), reference lib/spec_utils.py:26-31,157-165 (librosa semantics, SURVEY App. A)
// frames [t0, t1) only (the full-track call is t0 = 0, t1 = T)
cudaError_t launch_stft(const float* wave, int64_t L, int n_fft, int hop, float2* spec, int64_t T, int64_t t0,
                        int64_t t1, const float2* twiddle, const float* window, cudaStream_t stream);
// frames_a[c][t][:] = hann * irfft(spec * mask), frames_b = hann * irfft(spec * (1 - mask));
// mask == nullptr: frames_a = hann * irfft(spec), frames_b unused
// frames [t_first, t_first + nfr) of the track into a scratch laid out [c][nfr][n_fft]
cudaError_t launch_istft_frames(const float2* spec, const float* mask, int n_fft, int64_t T, int64_t t_first,
                                int64_t nfr, float* frames_a, float* frames_b, const float2* twiddle,
                                const float* window, cudaStream_t stream);
// overlap-add + window-sum-square normalisation + centre trim of output samples [s0, s1) of wave [2][hop*(T-1)]
cudaError_t launch_istft_ola(const float* frames_a, const float* frames_b, int n_fft, int hop, int64_t T,
                             int64_t t_first, int64_t nfr, int64_t s0, int64_t s1, float* wave_a, float* wave_b,
                             const float* window, cudaStream_t stream);

// ---- sample-rate conversion (resample.cu), resampy.resample(filter='kaiser_fast') behind librosa.load ----------
// x [C][n_in] -> y [C][n_out], n_out = int(n_in * sample_ratio); win / delta: the (ratio-scaled) half filter table and
// its first difference, nwin entries, num_table entries per zero crossing (oracle/resample_oracle.py: prepare)
cudaError_t launch_resample_sinc(const float* x, int C, int64_t n_in, float* y, int64_t n_out, double sample_ratio,
                                 const double* win, const double* delta, int nwin, int num_table, cudaStream_t stream);

// ---- FLAC frame decoding (flac.cu), the decode in front of the path for .flac input (lib/flac.py) --------------------
// scan: every frame-header candidate at byte offsets [begin, n_bytes) -> cands[*count][4] (at most max_cands written;
// *count is zeroed first and counts them all); decode: one warp per chained frame, frames[n_frames][4] = (start byte,
// next frame's start byte or n_bytes, first sample, block size | header length << 17 | channel code << 24 |
// bps << 28) -> out [channels][n_samples] float32, status[n_frames]
cudaError_t launch_flac_scan(const uint8_t* data, int64_t n_bytes, int64_t begin, int64_t* cands, int max_cands,
                             int* count, cudaStream_t stream);
cudaError_t launch_flac_decode(const uint8_t* data, int64_t n_bytes, const int64_t* frames, int n_frames, int channels,
                               int64_t n_samples, float* out, int64_t* status, cudaStream_t stream);

// ---- MPEG-4 AAC-LC decoding (aac.cu), the decode in front of the path for .m4a / .mp4 input (lib/aac.py) -----------
// table[n_packets][2] = (byte offset, byte size) of each raw_data_block in data -> out [channels][1024 * n_packets]
// (no trim), status[n_packets]; the workspace (aac_workspace_bytes) holds the descriptors, quantised values and spectra
int64_t aac_workspace_bytes(int64_t n_packets, int channels);
cudaError_t launch_aac_decode(const uint8_t* data, int64_t n_bytes, const int64_t* table, int n_packets, int channels,
                              int rate_index, void* workspace, int64_t workspace_bytes, float* out, int64_t* status,
                              cudaStream_t stream);

// ---- Vorbis I decoding (vorbis.cu), the decode in front of the path for .ogg input (lib/vorbis.py) ----------------
// table[n_packets][5] (vr_b200.h) and the flattened setup -> out [channels][n_out] (no trim), status[n_packets]; the
// workspace (vorbis_workspace_bytes) holds the floor points, the residue classes and the spectrum slots
int64_t vorbis_workspace_bytes(int64_t n_packets, int channels, int64_t slot_floats);
cudaError_t launch_vorbis_decode(const uint8_t* data, int64_t n_bytes, const int64_t* table, int n_packets,
                                 const int* setup, int setup_words, int channels, int n_codes, int64_t slot_floats,
                                 void* workspace, int64_t workspace_bytes, float* out, int64_t n_out, int64_t* status,
                                 cudaStream_t stream);

// ---- MPEG-1 Layer III decoding (mp3.cu), the decode in front of the path for .mp3 input (lib/mp3.py) ---------------
// scan: every 11-bit sync at byte offsets [begin, end - 4] -> cands[*count][2] = (offset, the 4 header bytes
// big-endian); decode: frames[n_frames][2] = (offset, header word) of the chained frames, md_off[n_frames + 1] = the
// exclusive scan of their main-data byte counts (md_bytes = md_off[n_frames]) -> out [channels][1152 * n_frames],
// status[n_frames]; the workspace (mp3_workspace_bytes) holds the reservoir buffer and every intermediate
int64_t mp3_workspace_bytes(int64_t n_frames, int channels, int64_t md_bytes);
cudaError_t launch_mp3_scan(const uint8_t* data, int64_t begin, int64_t end, int64_t* cands, int max_cands, int* count,
                            cudaStream_t stream);
cudaError_t launch_mp3_decode(const uint8_t* data, int64_t n_bytes, const int64_t* frames, const int64_t* md_off,
                              int n_frames, int channels, int rate_index, int64_t md_bytes, void* workspace,
                              int64_t workspace_bytes, float* out, int64_t* status, cudaStream_t stream);

// ---- FLAC frame encoding (flac_encode.cu), the encode behind --output_format flac (lib/flac.py) ----------------------
// analyse: one CTA per 4096-sample frame of x [channels][n] -> pcm [n][channels] (int16 for bits = 16, int32 for 24),
// plan [frames][192] int32 (the frame's size in bytes first); pack: plan + each frame's byte offset -> the frames' bytes
// in out, status[frames]; pcm_pack: x -> the same integers as interleaved little-endian bits / 8-byte PCM in out
cudaError_t launch_flac_encode_analyse(const float* x, int channels, int64_t n, int rate_code, int bits, void* pcm,
                                       int32_t* plan, cudaStream_t stream);
cudaError_t launch_flac_encode_pack(const void* pcm, int channels, int64_t n, int bits, const int32_t* plan,
                                    const int64_t* offsets, int rate_code, int rate_value, uint8_t* out,
                                    int32_t* status, cudaStream_t stream);
cudaError_t launch_pcm_pack(const float* x, int channels, int64_t n, int bits, uint8_t* out, cudaStream_t stream);

// ---- BSS Eval (bsseval.cu): workspace bytes, or -1 with err set; the whole evaluation of one track, synchronous ------
// framewise: BSS Eval v3, every frame scored as a signal of its own, frames_per_batch frames per batch; otherwise one
// set of filters for the whole track (v4), and frames_per_batch is not read
int64_t bss_eval_workspace(bool framewise, int K, int C, int64_t N, int L, int64_t window, int64_t hop,
                           int64_t frames_per_batch, std::string& err);
bool bss_eval(bool framewise, const float* refs, const float* ests, int K, int C, int64_t N, int L, int64_t window,
              int64_t hop, int64_t frames_per_batch, void* workspace, int64_t workspace_bytes, double* frames_host,
              double* corr_host, double* loading_host, double* phase_ms, cudaStream_t stream, std::string& err);

}  // namespace vr
