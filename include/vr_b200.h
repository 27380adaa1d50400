/* vr_b200.h - C ABI of the H100-native vocal-remover inference hot path (libvr_b200.so).
 *
 * The reference (tsurumeso/vocal-remover @ 99f92fe) is pure Python and has NO plugin / FFI interface;
 * the drop-in boundary is the Python call surface used by inference.py:130-176 and pseudo.py:32-67.
 * Each entry point below names the reference call it replaces.  The Python mirror that binds these
 * with ctypes lives in vocal-remover_b200/lib/_native.py (see INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes only (no torch types); every function returns 0 on success and a
 * negative value on error, with the message available from vr_last_error(); `stream` is a cudaStream_t
 * passed as void* (NULL = legacy default stream); unless stated otherwise pointers are DEVICE pointers on
 * the context's GPU and calls are asynchronous on `stream`.  A context is bound to one GPU and is not
 * thread-safe.  There is no CPU path: vr_create fails if no CUDA device is present.
 *
 * Array layouts are the reference's (row-major / C order):
 *   wave  float32    [2][L]
 *   spec  complex64  [2][bins][T]        bins = n_fft/2+1, T = 1 + L/hop       (lib/spec_utils.py:26-31)
 *   mask  float32    [2][bins][T]
 *   mag   float32    [N][2][bins][W]     W = cropsize                          (lib/nets.py:124)
 */
#ifndef VR_B200_H_
#define VR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define VR_API __attribute__((visibility("default")))
#else
#define VR_API
#endif

typedef struct vr_ctx vr_ctx;

typedef struct vr_config {
  int32_t device;      /* CUDA device ordinal                                   (inference.py:124-129)  */
  int32_t n_fft;       /* --n_fft, power of two in [64, 4096]                    (inference.py:113)      */
  int32_t hop_length;  /* --hop_length                                           (inference.py:114)      */
  int32_t nout;        /* CascadedNet nout (32)                                  (inference.py:130)      */
  int32_t nout_lstm;   /* CascadedNet nout_lstm (128)                            (inference.py:130)      */
  int32_t cropsize;    /* --cropsize, multiple of 16, > 128                      (inference.py:116)      */
  int32_t max_batch;   /* windows per forward launch sequence (--batchsize)      (inference.py:115)      */
  int32_t conv_mode;   /* 0 = wgmma tensor-core conv where the tile fits,  1 = CUDA-core conv only     */
} vr_config;

/* nets.CascadedNet(n_fft, hop, nout, nout_lstm).to(device)                      (lib/nets.py:46-80)     */
VR_API int vr_create(const vr_config* cfg, vr_ctx** out);
VR_API void vr_destroy(vr_ctx* ctx);
/* Message of the last failed call on ctx (ctx may be NULL for a failed vr_create). */
VR_API const char* vr_last_error(const vr_ctx* ctx);

/* model.load_state_dict(...) (inference.py:131): one call per state_dict entry with its PyTorch key,
 * HOST pointer; dtype 0 = float32, 1 = int64.  vr_finalize_weights is strict (missing / unexpected key or
 * shape mismatch -> error), folds eval-mode BatchNorm into the convolutions and packs for the kernels.  */
VR_API int vr_load_tensor(vr_ctx* ctx, const char* name, int32_t dtype, int32_t ndim, const int64_t* shape,
                   const void* host_data);
VR_API int vr_finalize_weights(vr_ctx* ctx);

/* spec_utils.wave_to_spectrogram(wave, hop, n_fft) (lib/spec_utils.py:26-31).  absmax (device float*,
 * may be NULL) receives max|spec| = the normaliser of inference.py:74.                                  */
VR_API int vr_stft(vr_ctx* ctx, const float* wave, int64_t L, void* spec, int64_t T, float* absmax, void* stream);

/* spec_utils.spectrogram_to_wave(spec, hop) (lib/spec_utils.py:157-165): wave [2][hop*(T-1)].           */
VR_API int vr_istft(vr_ctx* ctx, const void* spec, int64_t T, float* wave, void* stream);

/* model.predict_mask(x) (lib/nets.py:124-131): mag [N][2][bins][W] -> mask [N][2][bins][W-2*64].        */
VR_API int vr_predict_mask(vr_ctx* ctx, const float* mag, int32_t N, float* mask, void* stream);

/* model.forward(x) / model(x) (lib/nets.py:82-117): the un-cropped mask [N][2][bins][W].                */
VR_API int vr_forward(vr_ctx* ctx, const float* mag, int32_t N, float* mask, void* stream);

/* norm_mode 0: max|spec| (Separator.separate, inference.py:74); 1: |lexicographic complex max| as numpy's
 * complex .max() gives in Separator.separate_tta (inference.py:87,94).  out = device float*.            */
VR_API int vr_normaliser(vr_ctx* ctx, const void* spec, int64_t T, int32_t norm_mode, float* out, void* stream);

/* Separator._separate over a shard of windows (inference.py:42-68): windows [first_window,
 * first_window+n_windows) of the spectrogram padded by pad_l zeros on the left, normalised by *norm
 * (device), are run through the net; mask frame j of the concatenated result is written to
 * mask[:, :, j - frame_shift] if that lies in [0, mask_T).  accumulate=1 averages with what is there
 * ((old+new)/2, the TTA combine of inference.py:98).  `mask` may be a peer-mapped pointer on another GPU
 * (multi-GPU gather written by the epilogue kernel itself over NVLink).                                 */
VR_API int vr_separate_windows(vr_ctx* ctx, const void* spec, int64_t T, const float* norm, int32_t pad_l,
                        int32_t first_window, int32_t n_windows, float* mask, int64_t mask_T,
                        int64_t frame_shift, int32_t accumulate, void* stream);

/* Mask of Separator.separate (tta=0, inference.py:70-77) / separate_tta (tta=1, inference.py:83-98).    */
VR_API int vr_separate(vr_ctx* ctx, const void* spec, int64_t T, int32_t tta, float* mask, void* stream);

/* Separator._postprocess without --postprocess (inference.py:32-36): y = mask*spec, v = (1-mask)*spec.  */
VR_API int vr_apply_mask(vr_ctx* ctx, const void* spec, const float* mask, int64_t T, void* y_spec, void* v_spec,
                  void* stream);

/* --postprocess / spec_utils.merge_artifacts (lib/spec_utils.py:60-93, inference.py:27-30) without moving the mask
 * off the device: frame_min[t] = min over (channel, bin) of mask[:, :, t] (device float[T]); the caller finds the
 * long above-threshold runs on the host from those T floats (lib/spec_utils.py:artifact_weights) and hands back one
 * fade weight per frame, which vr_mask_apply_weight applies in place: mask += weight[t] * (1 - mask).           */
VR_API int vr_mask_frame_min(vr_ctx* ctx, const float* mask, int64_t T, float* frame_min, void* stream);
VR_API int vr_mask_apply_weight(vr_ctx* ctx, float* mask, int64_t T, const float* weight, void* stream);

/* y/v waves straight from spec and mask: _postprocess + 2x spectrogram_to_wave fused
 * (inference.py:32-36,171,176).  wave_inst / wave_voc: [2][hop*(T-1)].                                 */
VR_API int vr_apply_mask_istft(vr_ctx* ctx, const void* spec, const float* mask, int64_t T, float* wave_inst,
                        float* wave_voc, void* stream);

/* Shard-sized pieces of the three calls above for the multi-GPU path (lib/distributed.py): the STFT of frames
 * [t0, t1) only, max|spec| over those frames (ranks all-reduce it to the normaliser of inference.py:74), and the
 * masked inverse STFT of output hops [k0, k1) = samples [hop*k0, hop*k1) of wave_inst / wave_voc [2][hop*(T-1)],
 * which may be peer-mapped buffers on another GPU (the overlap-add kernel then stores over NVLink).
 * spec / mask are the full-size [2][bins][T] arrays; only the columns the range touches are read / written.  */
VR_API int vr_stft_range(vr_ctx* ctx, const float* wave, int64_t L, void* spec, int64_t T, int64_t t0, int64_t t1,
                  void* stream);
VR_API int vr_normaliser_range(vr_ctx* ctx, const void* spec, int64_t T, int64_t t0, int64_t t1, float* out,
                        void* stream);
VR_API int vr_apply_mask_istft_range(vr_ctx* ctx, const void* spec, const float* mask, int64_t T, int64_t k0,
                              int64_t k1, float* wave_inst, float* wave_voc, void* stream);

/* Whole hot path with everything resident in HBM (inference.py:147-176 minus file I/O).                 */
VR_API int vr_separate_wave(vr_ctx* ctx, const float* wave, int64_t L, int32_t tta, float* wave_inst,
                     float* wave_voc, void* stream);

/* Same with HOST buffers (pinned recommended); copies in, runs, copies out and synchronises.            */
VR_API int vr_separate_wave_host(vr_ctx* ctx, const float* wave_host, int64_t L, int32_t tta, float* inst_host,
                          float* voc_host, void* stream);

/* vr_separate_wave_host plus the --output_image spectrogram images of both stems (inference.py:180-185), built on
 * the device from the final spectrogram and mask: img_inst_host / img_voc_host are HOST uint8 [bins][T][3] buffers,
 * or NULL for none (both NULL = vr_separate_wave_host).  The stems are the same as vr_separate_wave_host's.      */
VR_API int vr_separate_wave_host_images(vr_ctx* ctx, const float* wave_host, int64_t L, int32_t tta, float* inst_host,
                                        float* voc_host, uint8_t* img_inst_host, uint8_t* img_voc_host, void* stream);

/* spec_utils.spectrogram_to_image(spec) in magnitude mode (lib/spec_utils.py:34-57) for spec [2][bins][T]:
 * img [bins][T][3] uint8 = {max(L, R), L, R} of trunc(255 * (l - min l) / (max l - min l)), l = log10(|s|^2 + 1e-8),
 * min / max over the whole array.  mask != NULL: img_a = image of mask * spec (y_spec of inference.py:32-36) and
 * img_b = image of (1 - mask) * spec (v_spec); mask == NULL: img_a = image of spec, img_b unused.  A constant
 * array (max == min, e.g. a silent track) gives an all-zero image (the reference's cast then sees NaN).          */
VR_API int vr_spec_image(vr_ctx* ctx, const void* spec, const float* mask, int64_t T, uint8_t* img_a, uint8_t* img_b,
                         void* stream);

/* The vocal JPG of the dataset inspection tool (lib/dataset.py:280-287): spectrogram_to_image(v_mag) with
 * v_mag = |X| - |y|, kept where v_mag > |y| (zero elsewhere), for the mixture spec_x and instruments spec_y, both
 * device complex64 [2][bins][T].  img: device uint8 [bins][T][3], levels, min / max and constant-array rule as in
 * vr_spec_image.                                                                                              */
VR_API int vr_vocal_image(vr_ctx* ctx, const void* spec_x, const void* spec_y, int64_t T, uint8_t* img, void* stream);

/* v_spec = X_spec - y_spec of the pair check (lib/spec_utils.py:186): out = a - b elementwise over the device
 * complex64 [2][bins][T] arrays a, b, out (IEEE fp32 subtraction, numpy's bits).                               */
VR_API int vr_spec_sub(vr_ctx* ctx, const void* a, const void* b, int64_t T, void* out, void* stream);

/* evaluate.py --oracle (DESIGN.md §12): the instruments mask of an ideal separation, from the mixture spec_x and the
 * true instruments spec_y (device complex64 [2][bins][T]); the true vocals are V = spec_x - spec_y with vr_spec_sub's
 * fp32 bits.  mask: device float32 [2][bins][T] in [0, 1].  kind: 0 iam, 1 ibm, 2 irm1, 3 irm2; anything else, T < 1
 * or a NULL pointer is an error.  Needs no weights.  Bit-identical from call to call.                           */
VR_API int vr_oracle_mask(vr_ctx* ctx, const void* spec_x, const void* spec_y, int64_t T, int32_t kind, float* mask,
                          void* stream);

/* train.py:108-134 validate_epoch over lib/dataset.py:220-248 make_validation_set, one track pair:
 * window_sums[j], j < ceil(T/roi), = sum over (2, bins, roi) of |mask*|X|/coef - |y|/coef| for patch j,
 * coef = max(max|X|, max|y|) written to *coef_out (device float, may be NULL).
 * spec_x / spec_y: device complex64 [2][bins][T] (mixture / instruments); window_sums: device double[ceil(T/roi)].
 * mask is the net's mask of patch j (X/coef padded by make_padding, the 1025th bin replicating the 1024th), frames
 * past T count as zero.  Each patch's loss is window_sums[j] / (2 * bins * roi); the sums are bit-identical from
 * call to call.  A zero or non-finite coef gives inv = 0 (all sums 0): the caller must reject such a pair.       */
VR_API int vr_validation_loss(vr_ctx* ctx, const void* spec_x, const void* spec_y, int64_t T,
                              float* coef_out, double* window_sums, void* stream);

/* --wiener_iterations (DESIGN.md §11): norbert 0.2's wiener(v, x, iterations, use_softmask=False) for two channels and
 * two sources.  spec is the mixture, y_spec / v_spec the initial estimates (vr_apply_mask's outputs), all device
 * complex64 [2][bins][T]; y_spec and v_spec are refined in place by `iterations` rounds of expectation-maximisation:
 * per bin the spatial covariance R_j of each source over the whole track, then per (bin, frame)
 * y_j = v_j R_j (sum_k v_k R_k + sqrt(eps) I)^-1 x, in fp64 on the mixture scaled by max(1, max|X| / 10), the estimates
 * stored as complex64 between iterations.  iterations = 0 leaves them unchanged.  iterations < 0, T < 1 or a NULL
 * pointer is an error.  The results are bit-identical from call to call.                                        */
VR_API int vr_wiener(vr_ctx* ctx, const void* spec, void* y_spec, void* v_spec, int64_t T, int32_t iterations,
                     void* stream);

/* The sample-rate conversion inside librosa.load(path, sr=args.sr, res_type='kaiser_fast') (inference.py:136-138,
 * pseudo.py:47-50) = resampy.resample(y, orig_sr, sr, filter='kaiser_fast'): x [channels][n_in] -> y [channels][n_out],
 * n_out = (int64)(n_in * sample_ratio), sample_ratio = sr / orig_sr.  win / delta: DEVICE float64 arrays of nwin entries -
 * the half filter table (already multiplied by sample_ratio when it is < 1) and its first difference - with
 * table_per_crossing entries per zero crossing, as resampy.core.resample prepares them (lib/audio_io.py builds the
 * documented kaiser_fast table; a table taken from an installed resampy can be passed instead).  ctx may be NULL
 * (audio is loaded before a model exists): the call then runs on the calling thread's current device and its error
 * message is read with vr_last_error(NULL).  SURVEY 8(f) rank 2.                                            */
VR_API int vr_resample(vr_ctx* ctx, const float* x, int32_t channels, int64_t n_in, float* y, int64_t n_out,
                       double sample_ratio, const double* win, const double* delta, int32_t nwin,
                       int32_t table_per_crossing, void* stream);

/* FLAC decoding on the device (RFC 9639; lib/flac.py is the caller, oracle/flac_oracle.py restates the format).  All
 * buffers are DEVICE memory owned by the caller; neither call allocates.  ctx may be NULL, as for vr_resample: the
 * call then runs on the calling thread's current device and its error message is read with vr_last_error(NULL).
 *
 * vr_flac_scan: every frame-header candidate (sync 0xFFF8 / 0xFFF9, a parsable header, matching CRC-8) at a byte
 * offset in [begin, n_bytes) of data.  Writes min(count, max_cands) rows of 4 int64, in no particular order:
 * (offset, coded frame or sample number, block size | header length << 17 | variable-strategy bit << 22,
 * header byte 2 | byte 3 << 8 | coded sample-rate value << 16); *count (one int32) is set to the number found.
 *
 * vr_flac_decode: one warp per frame.  frames: n_frames rows of 4 int64 (start byte, the next frame's start byte or,
 * for the last frame, the end of the audio data, first sample, block size | header length << 17 | channel code << 24 |
 * bits per sample << 28).  out: [channels][n_samples] float32, float32(x) / 2^(bps-1).  status: one
 * int64 per frame, 0 when the frame decoded, ends 2 bytes before the next frame's start and its CRC-16 matches, else
 * code << 40 | bit offset in the frame (codes: lib/flac.py).  Malformed bytes never fault: they give a status. */
VR_API int vr_flac_scan(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, int64_t begin, int64_t* cands,
                        int32_t max_cands, int32_t* count, void* stream);
VR_API int vr_flac_decode(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, const int64_t* frames, int32_t n_frames,
                          int32_t channels, int64_t n_samples, float* out, int64_t* status, void* stream);

/* MPEG-1 Audio Layer III decoding on the device (ISO/IEC 11172-3, 32 / 44.1 / 48 kHz; lib/mp3.py is the caller,
 * oracle/mp3_oracle.py restates the standard).  All buffers are DEVICE memory owned by the caller; no call allocates.
 * ctx may be NULL, as for vr_flac_scan.
 *
 * vr_mp3_scan: every 11-bit frame sync at a byte offset in [begin, end - 4] of data.  Writes min(count, max_cands)
 * rows of 2 int64, in no particular order: (offset, the 4 header bytes as a big-endian word); *count (one int32) is
 * set to the number found.  Header fields are not judged: the host chains the frames and rejects what it does not take.
 *
 * vr_mp3_workspace: bytes of the workspace vr_mp3_decode needs for n_frames frames of channels (1 or 2) channels
 * holding md_bytes bytes of main data in all (-1 for invalid arguments).
 *
 * vr_mp3_decode: frames: n_frames rows of 2 int64 (offset, header word) of consecutive MPEG-1 Layer III frames of one
 * rate (rate_index 0 / 1 / 2 = 44.1 / 48 / 32 kHz) and one channel mode; md_off: n_frames + 1 int64, the exclusive
 * scan of the frames' main-data byte counts (frame length less header, CRC and side info), md_off[n_frames] =
 * md_bytes.  out: [channels][1152 * n_frames] float32, the synthesis output at full scale 1, not clipped, with zero
 * filterbank state before the first frame.  status: one int64 per frame, 0 or code << 40 | bit offset (codes:
 * lib/mp3.py); code 1 (main data begins before the first frame) is not an error: that frame decodes as an all-zero
 * spectrum and the synthesis carries on through it.  Malformed bytes never fault: they give a status and zeros. */
VR_API int64_t vr_mp3_workspace(int64_t n_frames, int32_t channels, int64_t md_bytes);
VR_API int vr_mp3_scan(vr_ctx* ctx, const uint8_t* data, int64_t begin, int64_t end, int64_t* cands, int32_t max_cands,
                       int32_t* count, void* stream);
VR_API int vr_mp3_decode(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, const int64_t* frames,
                         const int64_t* md_off, int32_t n_frames, int32_t channels, int32_t rate_index,
                         int64_t md_bytes, void* workspace, int64_t workspace_bytes, float* out, int64_t* status,
                         void* stream);

/* MPEG-4 AAC-LC decoding on the device (ISO/IEC 14496-3 subpart 4, the twelve sampling-frequency indices, 1 or 2
 * channels, 1024-sample frames; lib/aac.py is the caller and walks the MP4 container, oracle/aac_oracle.py restates
 * the standard).  All buffers are DEVICE memory owned by the caller; no call allocates.
 *
 * vr_aac_workspace: bytes of the workspace vr_aac_decode needs for n_packets packets of channels (1 or 2) channels
 * (-1 for invalid arguments).
 *
 * vr_aac_decode: table: n_packets rows of 2 int64 (byte offset in data, byte size) of consecutive raw_data_blocks of
 * one track (rate_index 0..11, the AudioSpecificConfig's samplingFrequencyIndex).  out: [channels][1024 * n_packets]
 * float32 at full scale 1, not clipped, with zero filterbank state before the first packet and no edit-list trim.
 * status: one int64 per packet, 0 or code << 40 | bit offset in the packet (codes: lib/aac.py).  Malformed bytes never
 * fault: they give a status and a finite output. */
VR_API int64_t vr_aac_workspace(int64_t n_packets, int32_t channels);
VR_API int vr_aac_decode(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, const int64_t* table, int32_t n_packets,
                         int32_t channels, int32_t rate_index, void* workspace, int64_t workspace_bytes, float* out,
                         int64_t* status, void* stream);

/* Vorbis I decoding on the device (1 or 2 channels, block sizes 64..8192, floor 1, residues 0-2; lib/vorbis.py is
 * the caller, reads the Ogg pages and flattens the setup header; oracle/vorbis_oracle.py restates the specification).
 * All buffers are DEVICE memory owned by the caller; no call allocates.
 *
 * vr_vorbis_workspace: bytes of the workspace vr_vorbis_decode needs for n_packets packets of channels (1 or 2)
 * channels whose spectrum slots take slot_floats floats in all (the sum over packets of channels * blocksize / 2; -1
 * for invalid arguments).
 *
 * vr_vorbis_decode: table: n_packets rows of 5 int64: byte offset in data, byte size, end of the packet's output range
 * (the samples from the centre of the first block to the centre of this one), offset of its spectrum slot in floats,
 * block flag | previous window flag << 1 | next window flag << 2 | mapping << 8.  setup: setup_words int32 in
 * lib/vorbis.py's layout, holding n_codes codewords in all.  out: [channels][n_out] float32 at full scale 1, not
 * clipped, no granule trim; n_out is the last row's output end.  status: one int64 per packet, 0 or code << 40 | bit
 * offset in the packet (codes: lib/vorbis.py).  Malformed bytes never fault: they give a status and a finite
 * output. */
VR_API int64_t vr_vorbis_workspace(int64_t n_packets, int32_t channels, int64_t slot_floats);
VR_API int vr_vorbis_decode(vr_ctx* ctx, const uint8_t* data, int64_t n_bytes, const int64_t* table,
                            int32_t n_packets, const int32_t* setup, int32_t setup_words, int32_t channels,
                            int32_t n_codes, int64_t slot_floats, void* workspace, int64_t workspace_bytes, float* out,
                            int64_t n_out, int64_t* status, void* stream);

/* FLAC encoding on the device (RFC 9639 streamable subset; lib/flac.py is the caller, oracle/flac_oracle.py decodes
 * the result independently): fixed block size FLAC_ENCODE_BLOCK (the last block shorter), bits = 16 or 24 bits per
 * sample (anything else is an error), one or two channels.  All buffers are DEVICE memory owned by the caller; no call
 * allocates.  ctx may be NULL, as for vr_flac_scan.  frames = ceil(n / FLAC_ENCODE_BLOCK); rate_code is the frame
 * header's sample-rate code (1-11 from the table, 12-14 with rate_value written after the header as RFC 9639 section
 * 9.1.2 gives).  Both encoder calls of one stream take the same bits.
 *
 * The integers: q(x) = clip(rint(x * T), -T - 1, T) with T = 2^(bits-1) - 1 (32767 or 8388607), the product rounded
 * once in fp32 and rint to even, NaN -> 0.  A subframe holds bits-wide samples, except the side channel S = L - R of a
 * left/side, side/right or mid/side frame, which takes bits + 1 (25 at 24 bits).
 *
 * vr_flac_encode_analyse: one CTA per frame.  x: [channels][n] float32, quantised into pcm: [n][channels], int16 for
 * bits = 16 and int32 for bits = 24 (interleaved; vr_flac_encode_pack reads it back).  Chooses
 * every subframe's coding and the channel assignment by exact size and writes plan: frames rows of
 * FLAC_ENCODE_PLAN_INTS int32, plan[f * FLAC_ENCODE_PLAN_INTS] = frame f's size in bytes (the rest is private to
 * vr_flac_encode_pack).  The plan, and with it every byte, is the same on every run.
 *
 * vr_flac_encode_pack: one CTA per frame.  offsets: frames int64, the byte offset of each frame in out (the exclusive
 * scan of the plan's sizes, plus the caller's header length); writes each frame, CRC-8 and CRC-16 included, to its
 * span.  status: frames int32, 0 when the frame filled exactly the size the plan gave, else nonzero.
 *
 * vr_pcm_pack: the quantiser alone.  x: [channels][n] float32 -> out: n * channels * bits / 8 bytes, q(x) interleaved
 * as little-endian 2- or 3-byte integers: the data chunk of a PCM WAV file and the bytes the STREAMINFO MD5 is taken
 * over.  out must be 16-byte aligned.                                                                        */
#define FLAC_ENCODE_BLOCK 4096
#define FLAC_ENCODE_PLAN_INTS 192
VR_API int vr_flac_encode_analyse(vr_ctx* ctx, const float* x, int32_t channels, int64_t n, int32_t rate_code,
                                  int32_t bits, void* pcm, int32_t* plan, void* stream);
VR_API int vr_flac_encode_pack(vr_ctx* ctx, const void* pcm, int32_t channels, int64_t n, int32_t bits,
                               const int32_t* plan, const int64_t* offsets, int32_t rate_code, int32_t rate_value,
                               uint8_t* out, int32_t* status, void* stream);
VR_API int vr_pcm_pack(vr_ctx* ctx, const float* x, int32_t channels, int64_t n, int32_t bits, uint8_t* out,
                       void* stream);

/* BSS Eval images with time-invariant distortion filters (lib/bsseval.py is the caller, oracle/bsseval_oracle.py the
 * float64 restatement, DESIGN.md section 10 the contract): K sources of C channels, M = K * C <= BSS_EVAL_MAX_SIGNALS,
 * filters of L <= BSS_EVAL_MAX_FILTER taps, N >= window samples.  refs / ests: DEVICE float32 [K][C][N] on the calling
 * thread's current device (or the context's, when ctx is not NULL; ctx may be NULL, as for vr_resample).
 *
 * vr_bss_eval_workspace: the bytes of device workspace vr_bss_eval needs for these sizes, or -1 (message from
 * vr_last_error(NULL)) for sizes it does not take.
 *
 * vr_bss_eval: frames = (N - window + hop) / hop windows, frame w = samples [w * hop, w * hop + window).  Writes to the
 * HOST array frames_host [K][frames][8] the float64 sums over frame w and the C channels of source j of
 *   s^2, (P_j - s)^2, (shat - s)^2, P_j^2, (P_all - P_j)^2, P_all^2, (shat - P_all)^2, shat^2
 * with s / shat the reference / estimate and P_all / P_j the estimate's projections on the delayed references of all
 * sources / of source j; the four ratios and the silence rule follow from these on the host.  corr_host (HOST, may be
 * NULL) receives r[a][b](l) = sum_u s_a(u) y_b(u + l), [M][2M][L], y = the M references then the M estimates: G and d.
 * The systems are G + eps I over all K*C*L unknowns and each source's block + eps I, eps = scale * max diag G with
 * scale = 2^-40, raised by 2^8 per retry for a system whose Cholesky factorisation meets a non-positive pivot (G is only
 * positive semidefinite), up to 2^-20; loading_host (HOST, may be NULL) receives the K + 1 scales used (all unknowns,
 * then source 0, 1, ...).  phase_ms (HOST, may be NULL) receives the CUDA-event times of {correlations, assembly +
 * Cholesky + solves, projections + frame sums, all}; "all" runs from the start of the call to the end of its last
 * projections, and alone includes the input check and the upload of the task list.  Synchronises the stream; the
 * results are bit-identical from call to call.  NaN or Inf in refs or ests, or a system still not factored at 2^-20,
 * is an error.
 *
 * Both calls run one host driver (csrc/bsseval.cu): this one scores the whole track as a single segment, the
 * framewise one below scores each frame as a segment of its own, in batches.                                     */
#define BSS_EVAL_MAX_SIGNALS 8
#define BSS_EVAL_MAX_FILTER 1024
VR_API int64_t vr_bss_eval_workspace(int32_t K, int32_t C, int64_t N, int32_t L, int64_t window, int64_t hop);
VR_API int vr_bss_eval(vr_ctx* ctx, const float* refs, const float* ests, int32_t K, int32_t C, int64_t N, int32_t L,
                       int64_t window, int64_t hop, void* workspace, int64_t workspace_bytes, double* frames_host,
                       double* corr_host, double* loading_host, double* phase_ms, void* stream);

/* BSS Eval images with framewise distortion filters (BSS Eval v3, museval's mode 'v3'; DESIGN.md section 10,
 * "Framewise filters (v3)"): the same frames, K, C, L, refs and ests as vr_bss_eval, but each frame w is scored as a
 * signal of its own: the window samples from w * hop, zero outside them, with its own Gram matrix, loadings, filters
 * and projections, on its own timeline of window + L - 1 samples.  Requires window >= L.
 *
 * vr_bss_eval_framewise_workspace: the bytes of device workspace for frames_per_batch frames at a time (clamped to
 * [1, min(frames, 4096)]; about frames_per_batch * ((K*C*L)^2 + K (C*L)^2) * 8 bytes), or -1 (vr_last_error(NULL)).
 *
 * vr_bss_eval_framewise: frames_host [K][frames][8] receives the eight sums of vr_bss_eval, in the same order, over
 * the window + L - 1 samples of each frame's timeline and the source's channels; corr_host (may be NULL) each frame's
 * correlations [frames][M][2M][L] of its window samples; loading_host (may be NULL) each frame's K + 1 loading scales
 * [frames][K + 1], NaN for a frame in which a reference source or an estimate is all zeros (its systems are the
 * identity and are not factored); phase_ms as vr_bss_eval's, the first three summed over the batches.  Synchronises the
 * stream; the results are bit-identical from call to call and for every frames_per_batch.  NaN or Inf in refs or
 * ests, or a system still not factored at 2^-20, is an error.                                                      */
VR_API int64_t vr_bss_eval_framewise_workspace(int32_t K, int32_t C, int64_t N, int32_t L, int64_t window,
                                               int64_t hop, int32_t frames_per_batch);
VR_API int vr_bss_eval_framewise(vr_ctx* ctx, const float* refs, const float* ests, int32_t K, int32_t C, int64_t N,
                                 int32_t L, int64_t window, int64_t hop, int32_t frames_per_batch, void* workspace,
                                 int64_t workspace_bytes, double* frames_host /* [K][nwin][8] */,
                                 double* corr_host /* [nwin][M][2M][L] or NULL */,
                                 double* loading_host /* [nwin][K+1] or NULL */, double* phase_ms, void* stream);

/* Multi-GPU mask exchange over NVLink peer memory (one process per GPU).  The owner (rank 0) allocates the
 * whole-track mask with vr_shared_alloc and publishes the 64-byte CUDA IPC handle; every other rank maps it
 * with vr_shared_open and passes the mapped pointer as `mask` to vr_separate_windows, so the mask epilogue
 * kernel itself stores its shard into rank 0's HBM - the "gather" of Separator._separate's concatenate
 * (inference.py:63-66) fused into the producing kernel.  vr_shared_close unmaps (owner=0) or frees (owner=1). */
VR_API int vr_shared_alloc(vr_ctx* ctx, int64_t bytes, void** dev_ptr, unsigned char* handle64);
VR_API int vr_shared_open(vr_ctx* ctx, const unsigned char* handle64, void** dev_ptr);
VR_API int vr_shared_close(vr_ctx* ctx, void* dev_ptr, int32_t owner);

/* Number of kernels launched by this context so far (bench.py 'gpu_launches').                           */
VR_API int64_t vr_launch_count(const vr_ctx* ctx);

/* CUDA-event timing of every convolution launch between enable(1) and read (bench.py roofline):
 * out[0..2] = tensor-core conv {ms, algorithmic FLOPs, launches}, out[3..5] = CUDA-core conv likewise.    */
VR_API int vr_profile_enable(vr_ctx* ctx, int32_t on);
VR_API int vr_profile_read(vr_ctx* ctx, double* out6);
/* Per-launch detail as text, one line per timed launch in launch order, convolutions and every other kernel of the
 * path: "<name> N Hout Wout kind ms gflop".  A convolution is named by the state_dict prefix of its layer (+ "+up"
 * when it produces its upsampled input itself) and has kind 1 (tensor cores) or 0 (CUDA cores); any other kernel has
 * kind 2 and gflop 0, and one line may time a group of kernels launched together (e.g. the two of the lexmax
 * normaliser).  Writes at most cap bytes (NUL-terminated) and stores the size needed in *needed (either may be
 * NULL / 0 to query).                                                                                       */
VR_API int vr_profile_dump(vr_ctx* ctx, char* text, int64_t cap, int64_t* needed);

/* ---- validation hooks used by tests/ (not part of the reference surface) ---------------------------- */
/* One Conv2DBNActiv-shaped layer (lib/layers.py:8-26; BN already folded into w/bias by the caller):
 * x [N][Cin][H][W] -> y [N][Cout][Ho][Wo]; use_tc selects the wgmma kernel (error if tile does not fit). */
VR_API int vr_debug_conv(vr_ctx* ctx, const float* x, int32_t N, int32_t Cin, int32_t H, int32_t W, const float* w,
                  const float* bias, int32_t Cout, int32_t k, int32_t stride, int32_t dil_h, int32_t dil_w,
                  int32_t act, int32_t use_tc, float* y, void* stream);
/* One Decoder-shaped layer (lib/layers.py:51-64, BN folded by the caller): low [N][Cl][h][w] is bilinearly
 * upsampled x2 (align_corners=True), concatenated with skip [N][Cs][2h][2w] and convolved 3x3 -> y [N][Cout][2h][2w];
 * fused = 1 runs the upsample inside the row-streaming tensor-core kernel, 0 as a separate kernel.              */
VR_API int vr_debug_decoder(vr_ctx* ctx, const float* low, int32_t N, int32_t Cl, int32_t h, int32_t w, const float* skip,
                     int32_t Cs, const float* wgt, const float* bias, int32_t Cout, int32_t act, int32_t fused, float* y,
                     void* stream);
/* Images [n0, n0 + n) of one tensor the last forward (vr_predict_mask, vr_forward, vr_separate*) left on the device,
 * copied to out (device float32) asynchronously on stream; synchronise the forward first.  Names:
 *   "in3", "o1", "o2", "f3"         the stage-input buffer, the stage-1 / stage-2 low-band outputs, stage 3's output
 *   "<prefix>.<buf>"                a BaseNet buffer, <prefix> its state_dict prefix (e.g. "stg3_full_band_net") and
 *                                   <buf> one of cat1 lstm_up t2 cat2 t3 cat3 t4 cat4 t5 e5 pool f1 acat ao d4 d3 d2
 *   "<prefix>.lstm.{l0,xp,hs,y}"    the LSTM branch's planes
 * An activation buffer comes back as NCHW [n][C][H][W] with every channel of the buffer, pads included; its channel
 * layout is DESIGN.md section 4's.  The LSTM planes come back as l0 / y [n][bins][T] (l0: the 1x1 input convolution
 * before its bias), xp [n][T][8*hid] (gate pre-activations, forward then reverse) and hs [n][T][2*hid], with
 * shape4[3] = 1.  out == NULL only fills shape4 = {n, C, H, W}.  Fails for an unknown name, n0 < 0, n0 + n > max_batch,
 * "lstm_up" in a BaseNet whose up(lstm) group lives in cat1, and y images the last forward did not compute.      */
VR_API int vr_debug_tensor(vr_ctx* ctx, const char* name, int32_t n0, int32_t n, float* out, int64_t* shape4,
                           void* stream);
/* Process-wide debug knobs of the tensor-core kernels: key 0 = 1 makes CTA 0 of the row-streaming kernel record a
 * timeline (builds with -DVR_TRACE), key 2 = 1 makes vr_debug_conv use its 64-channel output tile, key 3 = 1 sends the
 * layers prepared afterwards (every vr_debug_conv call prepares its layer) from the halo-tile kernel to the generic
 * one, key 3 = 2 / 3 makes the halo-tile kernel use MB = 1 / 2, key 6 = 1 (default) skips channel groups whose weights
 * are all zero, key 7 = 1 (default) lets stage 3's last convolution compute only the frames the mask keeps and write
 * the mask itself (0: every frame, then a separate output-layer kernel), key 8 chooses the generic kernel's pairing
 * (0 = automatic per launch, 1 = never, 2 / 3 = two m-tiles / both N tiles per CTA wherever the layer allows it),
 * key 9 chooses the epilogue stores of the three tensor-core kernels (0 = 16-byte stores of 8 channels wherever the
 * output allows them, 1 = 4-byte stores of channel pairs everywhere; both write the same values).
 * Returns -1 for any other key.                                                                                    */
VR_API int vr_debug_set(int32_t key, int32_t value);
/* The last convolution launch of this process (any context), as its launcher decided it: out8 = {kind (0 CUDA-core,
 * 1 generic, 2 row-streaming, 3 halo-tile tensor-core kernel), KB (channels per chunk), BN (output channels per tile),
 * n_tiles, pairing (0 none, 1 PAIR_M, 2 PAIR_N), MB (halo kernel), UP (row kernel with fused upsample), 16-byte
 * epilogue stores (0/1)}; fields the kernel does not have are 0.  Returns -1 if out8 is NULL.                        */
VR_API int vr_debug_last_conv(int32_t* out8);
/* timeline of CTA 0 of the last row-kernel launch made with vr_debug_set(0, 1): 3 roles x 2048 events x 3 clock64 stamps
 * (unused / TMA producer / interpolation warp 0), copied to HOST memory; returns the number of values or -1 */
VR_API int64_t vr_debug_trace(uint64_t* host_out, int64_t capacity);

#ifdef __cplusplus
}
#endif
#endif /* VR_B200_H_ */
