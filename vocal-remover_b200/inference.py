"""H100-native drop-in for the reference's inference.py (Separator + CLI).

Same command line (12 flags, inference.py:109-120), same output files and stage banners, same
``Separator(model, device, batchsize, cropsize, postprocess).separate / separate_tta`` contract
(numpy complex64 (2, bins, T) in, (y_spec, v_spec) out), but the sliding-window STFT -> CascadedNet ->
mask -> inverse-STFT path runs in hand-written sm_90a CUDA (libvr_b200.so, include/vr_b200.h).
``Separator.separate_wave`` is the fused device-resident form of the same path used by ``main``.
"""
import argparse
import os

import numpy as np
import torch

from lib import _native
from lib import audio_io
from lib import dataset
from lib import flac
from lib import nets
from lib import spec_utils
from lib import utils


class Separator(object):

    def __init__(self, model, device=None, batchsize=1, cropsize=256, postprocess=False, wiener_iterations=0):
        self.model = model
        self.offset = model.offset
        self.device = device
        self.batchsize = batchsize
        self.cropsize = cropsize
        self.postprocess = postprocess
        # an extension of the reference: > 0 refines both stems with that many iterations of a multichannel Wiener
        # filter (vr_wiener, DESIGN.md §11) once the mask is final
        if wiener_iterations < 0:
            raise ValueError('wiener_iterations must be >= 0, got %d' % wiener_iterations)
        self.wiener_iterations = int(wiener_iterations)
        if device is not None:
            model.to(device)

    # ---- helpers ------------------------------------------------------------------------------------
    def _ctx(self):
        return self.model.native_context(self.cropsize, self.batchsize)

    def _dev(self):
        return torch.device('cuda', self._ctx().device_index)

    @staticmethod
    def _check_spec(X_spec):
        X_spec = np.asarray(X_spec)
        if X_spec.ndim != 3 or X_spec.shape[0] != 2:
            raise ValueError('X_spec must have shape (2, bins, frames)')
        return np.ascontiguousarray(X_spec.astype(np.complex64, copy=False))

    def _mask_device(self, d_spec, tta):
        ctx = self._ctx()
        T = d_spec.shape[2]
        d_mask = torch.empty((2, d_spec.shape[1], T), dtype=torch.float32, device=d_spec.device)
        ctx.check(ctx.lib.vr_separate(ctx.handle, _native.ptr(d_spec), T, 1 if tta else 0, _native.ptr(d_mask),
                                      _native.stream_ptr()), 'vr_separate')
        if self.postprocess:
            # --postprocess (inference.py:27-30): only T floats leave the device, the run detection of
            # merge_artifacts runs on the host, the fade weights are applied on the device
            frame_min = torch.empty(T, dtype=torch.float32, device=d_spec.device)
            ctx.check(ctx.lib.vr_mask_frame_min(ctx.handle, _native.ptr(d_mask), T, _native.ptr(frame_min),
                                                _native.stream_ptr()), 'vr_mask_frame_min')
            weight = torch.from_numpy(spec_utils.artifact_weights(frame_min.cpu().numpy())).to(d_spec.device)
            ctx.check(ctx.lib.vr_mask_apply_weight(ctx.handle, _native.ptr(d_mask), T, _native.ptr(weight),
                                                   _native.stream_ptr()), 'vr_mask_apply_weight')
        return d_mask

    def _run(self, X_spec, tta):
        X_spec = self._check_spec(X_spec)
        ctx = self._ctx()
        dev = self._dev()
        with torch.cuda.device(dev):
            d_spec = torch.from_numpy(X_spec).to(dev)
            d_mask = self._mask_device(d_spec, tta)
            y = torch.empty_like(d_spec)
            v = torch.empty_like(d_spec)
            ctx.check(ctx.lib.vr_apply_mask(ctx.handle, _native.ptr(d_spec), _native.ptr(d_mask), d_spec.shape[2],
                                            _native.ptr(y), _native.ptr(v), _native.stream_ptr()), 'vr_apply_mask')
            self._wiener(d_spec, y, v)
            return y.cpu().numpy(), v.cpu().numpy()

    def _wiener(self, d_spec, y, v):
        """--wiener_iterations: y / v refined in place (nothing to do for 0)."""
        if self.wiener_iterations > 0:
            ctx = self._ctx()
            ctx.check(ctx.lib.vr_wiener(ctx.handle, _native.ptr(d_spec), _native.ptr(y), _native.ptr(v),
                                        d_spec.shape[2], self.wiener_iterations, _native.stream_ptr()), 'vr_wiener')

    # ---- reference surface --------------------------------------------------------------------------
    def _separate(self, X_spec_pad, roi_size):
        """inference.py:42-68: mask for an already padded + normalised spectrogram."""
        X = self._check_spec(X_spec_pad)
        ctx = self._ctx()
        dev = self._dev()
        patches = (X.shape[2] - 2 * self.offset) // roi_size
        with torch.cuda.device(dev):
            d_spec = torch.from_numpy(X).to(dev)
            one = torch.ones(1, dtype=torch.float32, device=dev)
            d_mask = torch.empty((2, X.shape[1], patches * roi_size), dtype=torch.float32, device=dev)
            ctx.check(ctx.lib.vr_separate_windows(ctx.handle, _native.ptr(d_spec), X.shape[2], _native.ptr(one), 0, 0,
                                                  patches, _native.ptr(d_mask), patches * roi_size, 0, 0,
                                                  _native.stream_ptr()), 'vr_separate_windows')
            return d_mask.cpu().numpy()

    def separate(self, X_spec):
        """inference.py:70-81."""
        return self._run(X_spec, tta=False)

    def separate_tta(self, X_spec):
        """inference.py:83-102."""
        return self._run(X_spec, tta=True)

    # ---- fused device-resident path -----------------------------------------------------------------
    def separate_wave(self, wave, tta=False, images=False):
        """float32 (2, L) wave -> (instruments, vocals) float32 (2, hop*(T-1)) waves.

        Equivalent to wave_to_spectrogram -> separate[_tta] -> 2x spectrogram_to_wave
        (inference.py:147,158-161,171,176) without leaving the GPU in between.  ``wave`` may be a numpy
        array (host; copied in and out) or a CUDA tensor (returns CUDA tensors).  ``images=True`` also returns the
        --output_image spectrogram images of both stems (spectrogram_to_image of y_spec / v_spec, inference.py:180-185)
        as uint8 (bins, T, 3): (inst, voc, img_inst, img_voc); the stems are the same as with ``images=False``.
        """
        ctx = self._ctx()
        if self.postprocess or self.wiener_iterations > 0:
            # staged on the device: STFT -> mask (+ postprocess) [-> Wiener filter] -> inverse STFT
            return self._separate_wave_staged(wave, tta, images)
        dev = self._dev()
        hop = self.model.hop_length
        with torch.cuda.device(dev):
            if torch.is_tensor(wave) and wave.is_cuda:
                if images:
                    # the engine calls vr_separate_wave makes, with the spectrogram and mask kept for the images
                    return self._separate_wave_staged(wave, tta, images)
                w = wave.contiguous().float()
                L = w.shape[1]
                Lo = hop * (L // hop)
                inst = torch.empty((2, Lo), dtype=torch.float32, device=dev)
                voc = torch.empty((2, Lo), dtype=torch.float32, device=dev)
                ctx.check(ctx.lib.vr_separate_wave(ctx.handle, _native.ptr(w), L, 1 if tta else 0, _native.ptr(inst),
                                                   _native.ptr(voc), _native.stream_ptr()), 'vr_separate_wave')
                return inst, voc
            w = np.ascontiguousarray(np.asarray(wave, dtype=np.float32))
            L = w.shape[1]
            Lo = hop * (L // hop)
            inst = np.empty((2, Lo), dtype=np.float32)
            voc = np.empty((2, Lo), dtype=np.float32)
            if images:
                shape = (self.model.n_fft // 2 + 1, 1 + L // hop, 3)
                img_inst = np.empty(shape, dtype=np.uint8)
                img_voc = np.empty(shape, dtype=np.uint8)
                ctx.check(ctx.lib.vr_separate_wave_host_images(ctx.handle, w.ctypes.data, L, 1 if tta else 0,
                                                               inst.ctypes.data, voc.ctypes.data, img_inst.ctypes.data,
                                                               img_voc.ctypes.data, _native.stream_ptr()),
                          'vr_separate_wave_host_images')
                return inst, voc, img_inst, img_voc
            ctx.check(ctx.lib.vr_separate_wave_host(ctx.handle, w.ctypes.data, L, 1 if tta else 0, inst.ctypes.data,
                                                    voc.ctypes.data, _native.stream_ptr()), 'vr_separate_wave_host')
            return inst, voc

    def _separate_wave_staged(self, wave, tta, images):
        ctx = self._ctx()
        dev = self._dev()
        hop, n_fft = self.model.hop_length, self.model.n_fft
        with torch.cuda.device(dev):
            host = not (torch.is_tensor(wave) and wave.is_cuda)
            w = (torch.from_numpy(np.ascontiguousarray(np.asarray(wave, dtype=np.float32))).to(dev) if host
                 else wave.contiguous().float())
            L = w.shape[1]
            T = 1 + L // hop
            d_spec = torch.empty((2, n_fft // 2 + 1, T), dtype=torch.complex64, device=dev)
            ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(w), L, _native.ptr(d_spec), T, None,
                                      _native.stream_ptr()), 'vr_stft')
            d_mask = self._mask_device(d_spec, tta)
            inst = torch.empty((2, hop * (T - 1)), dtype=torch.float32, device=dev)
            voc = torch.empty_like(inst)
            if self.wiener_iterations > 0:
                # the filtered stems' spectrograms, then one inverse STFT (and image) per stem
                y = torch.empty_like(d_spec)
                v = torch.empty_like(d_spec)
                ctx.check(ctx.lib.vr_apply_mask(ctx.handle, _native.ptr(d_spec), _native.ptr(d_mask), T,
                                                _native.ptr(y), _native.ptr(v), _native.stream_ptr()), 'vr_apply_mask')
                self._wiener(d_spec, y, v)
                for spec, wave_out in ((y, inst), (v, voc)):
                    ctx.check(ctx.lib.vr_istft(ctx.handle, _native.ptr(spec), T, _native.ptr(wave_out),
                                               _native.stream_ptr()), 'vr_istft')
            else:
                ctx.check(ctx.lib.vr_apply_mask_istft(ctx.handle, _native.ptr(d_spec), _native.ptr(d_mask), T,
                                                      _native.ptr(inst), _native.ptr(voc), _native.stream_ptr()),
                          'vr_apply_mask_istft')
            out = [inst, voc]
            if images:
                img_inst = torch.empty((n_fft // 2 + 1, T, 3), dtype=torch.uint8, device=dev)
                img_voc = torch.empty_like(img_inst)
                if self.wiener_iterations > 0:
                    for spec, img in ((y, img_inst), (v, img_voc)):
                        ctx.check(ctx.lib.vr_spec_image(ctx.handle, _native.ptr(spec), None, T, _native.ptr(img), None,
                                                        _native.stream_ptr()), 'vr_spec_image')
                else:
                    ctx.check(ctx.lib.vr_spec_image(ctx.handle, _native.ptr(d_spec), _native.ptr(d_mask), T,
                                                    _native.ptr(img_inst), _native.ptr(img_voc), _native.stream_ptr()),
                              'vr_spec_image')
                out += [img_inst, img_voc]
            return tuple(t.cpu().numpy() for t in out) if host else tuple(out)


MODEL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'models')
DEFAULT_MODEL_PATH = os.path.join(MODEL_DIR, 'baseline.pth')
JPEG_MAX_WIDTH = utils.JPEG_MAX_WIDTH


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument('--gpu', '-g', type=int, default=-1)
    p.add_argument('--pretrained_model', '-P', type=str, default=DEFAULT_MODEL_PATH)
    p.add_argument('--input', '-i', required=True)
    p.add_argument('--sr', '-r', type=int, default=44100)
    p.add_argument('--n_fft', '-f', type=int, default=2048)
    p.add_argument('--hop_length', '-H', type=int, default=1024)
    p.add_argument('--batchsize', '-B', type=int, default=4)
    p.add_argument('--cropsize', '-c', type=int, default=256)
    p.add_argument('--output_image', '-I', action='store_true')
    p.add_argument('--tta', '-t', action='store_true')
    p.add_argument('--postprocess', '-p', action='store_true')
    p.add_argument('--output_dir', '-o', type=str, default="")
    # an extension of the reference CLI: lossless FLAC stems, encoded on the GPU (lib/flac.py)
    p.add_argument('--output_format', choices=['wav', 'flac'], default='wav')
    # an extension of the reference CLI too: bits per written sample of either format; 24 keeps the depth of a 24-bit
    # input, which the float32 stems carry and 16-bit output throws away
    p.add_argument('--output_bits', type=int, choices=[16, 24], default=16)
    # an extension as well: refine both stems with a multichannel Wiener filter (DESIGN.md §11) after the mask is final
    p.add_argument('--wiener_iterations', type=non_negative_int, default=0,
                   help="EM iterations of a multichannel Wiener filter applied to both stems (0: none; 1 is norbert's "
                        "default)")
    return p


def non_negative_int(text):
    value = int(text)
    if value < 0:
        raise argparse.ArgumentTypeError('must be >= 0, got {}'.format(value))
    return value


def main():
    args = build_parser().parse_args()

    # missing requirements fail before any heavy work (model load, audio decode, output directory)
    if args.output_image:
        try:
            import cv2  # noqa: F401  (the JPEG encoder of lib/utils.imwrite)
        except ImportError as e:
            raise ImportError('--output_image needs OpenCV (the cv2 module) to encode the JPGs: %s' % e) from e
    if not torch.cuda.is_available():
        raise RuntimeError('no CUDA device: the H100 build of vocal-remover has no CPU path')
    if args.gpu < 0:
        # the reference's default (--gpu -1) means CPU; this build has no CPU path
        print('note: --gpu {} selects the CPU in the reference; this build has no CPU path and uses cuda:0'.format(args.gpu))

    print('loading model...', end=' ')
    device = torch.device('cuda:{}'.format(max(args.gpu, 0)))
    model = nets.CascadedNet(args.n_fft, args.hop_length, 32, 128)
    model.load_state_dict(torch.load(args.pretrained_model, map_location='cpu'))
    model.to(device)
    spec_utils.set_device(device.index)
    print('done')

    print('loading wave source...', end=' ')
    X, sr = audio_io.load(args.input, sr=args.sr, mono=False, dtype=np.float32, device=device)
    basename = os.path.splitext(os.path.basename(args.input))[0]
    print('done')

    if X.ndim == 1:
        # mono to stereo
        X = np.asarray([X, X])

    sp = Separator(
        model=model,
        device=device,
        batchsize=args.batchsize,
        cropsize=args.cropsize,
        postprocess=args.postprocess,
        wiener_iterations=args.wiener_iterations
    )

    print('validating output directory...', end=' ')
    output_dir = args.output_dir
    if output_dir != "":  # modifies output_dir if theres an arg specified
        output_dir = output_dir.rstrip('/') + '/'
        os.makedirs(output_dir, exist_ok=True)
    print('done')

    images = args.output_image
    n_frames = 1 + X.shape[1] // args.hop_length
    if images and n_frames > JPEG_MAX_WIDTH:
        # the reference's cv2.imencode refuses the image and imwrite returns False: no JPG, the WAVs are still written
        print('skipping {0}_Instruments.jpg and {0}_Vocals.jpg: {1} frames exceed the {2}-pixel width limit of '
              'JPEG'.format(basename, n_frames, JPEG_MAX_WIDTH))
        images = False

    print('stft of wave source, separation, inverse stft of instruments and vocals...', end=' ')
    flac_out = args.output_format == 'flac'
    # FLAC and 24-bit WAV: the stems stay on the device for the encoder or the PCM packer, and only the file's bytes
    # come back
    on_device = flac_out or args.output_bits == 24
    out = sp.separate_wave(torch.from_numpy(np.ascontiguousarray(X)).to(device) if on_device else X, tta=args.tta,
                           images=images)
    wave_inst, wave_voc = out[:2]
    print('done')
    writer = audio_io.AsyncWriter()   # the two stems (and images) are encoded and written concurrently
    if flac_out:
        writer.run(flac.encode, wave_inst, sr, '{}{}_Instruments.flac'.format(output_dir, basename), True,
                   args.output_bits)
        writer.run(flac.encode, wave_voc, sr, '{}{}_Vocals.flac'.format(output_dir, basename), True, args.output_bits)
    else:
        writer.write('{}{}_Instruments.wav'.format(output_dir, basename), wave_inst.T, sr, args.output_bits)
        writer.write('{}{}_Vocals.wav'.format(output_dir, basename), wave_voc.T, sr, args.output_bits)
    if on_device:
        out = [t.cpu().numpy() if i >= 2 else t for i, t in enumerate(out)]
    if images:
        writer.run(utils.imwrite, '{}{}_Instruments.jpg'.format(output_dir, basename), out[2])
        writer.run(utils.imwrite, '{}{}_Vocals.jpg'.format(output_dir, basename), out[3])
    writer.join()


if __name__ == '__main__':
    main()
