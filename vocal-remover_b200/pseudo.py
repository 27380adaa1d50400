"""H100-native drop-in for the reference's pseudo.py (pseudo-label generation over a directory of track pairs), the
second caller of ``Separator.separate_tta`` (pseudo.py:56-74) and the many-file front-end of the hot path.

Same command line (pseudo.py:17-28) and the same outputs (``pseudo/{basename}_PseudoInstruments.npy`` + the empty
``.wav`` marker).  Per pair: load both tracks, ``align_wave_head_and_tail``, STFT of both, ``separate_tta(X - y)``,
``pseudo_inst = y + a_spec``.  The two STFTs, the difference, the TTA separation and the final sum run on the GPU without
leaving it in between (``PseudoLabeler.pseudo_instruments``); only the aligned waves go in and the result comes out.

Many files, many GPUs: under ``torchrun --nproc-per-node N pseudo.py ...`` every rank takes the files
``filelist[rank::N]`` (``dataset.shard_files``): whole files per GPU, no exchange between ranks - tracks are independent,
so file-level sharding replaces the window-level sharding of ``lib/distributed.py`` when there are at least N files.
"""
import argparse
import os

import numpy as np
import torch

from lib import _native
from lib import audio_io
from lib import dataset
from lib import nets
from lib import spec_utils

import inference


class PseudoLabeler(object):
    """Device-resident body of the reference loop (pseudo.py:56-71)."""

    def __init__(self, model, device, batchsize=4, cropsize=256, postprocess=False):
        self.sp = inference.Separator(model, device, batchsize, cropsize, postprocess)
        self.model = model

    def pseudo_instruments(self, X_wave, y_wave):
        """aligned float32 (2, L) mixture and instrument waves -> complex64 (2, bins, T) pseudo instruments."""
        sp = self.sp
        ctx = sp._ctx()
        dev = sp._dev()
        hop, n_fft = self.model.hop_length, self.model.n_fft
        with torch.cuda.device(dev):
            specs = []
            for w in (X_wave, y_wave):
                d_w = torch.from_numpy(np.ascontiguousarray(np.asarray(w, dtype=np.float32))).to(dev)
                L = d_w.shape[1]
                T = 1 + L // hop
                d_s = torch.empty((2, n_fft // 2 + 1, T), dtype=torch.complex64, device=dev)
                ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(d_w), L, _native.ptr(d_s), T, None,
                                          _native.stream_ptr()), 'vr_stft')
                specs.append(d_s)
            X, y = specs
            D = X - y                                          # pseudo.py:66: the residual the model separates
            mask = sp._mask_device(D, True)                    # separate_tta (inference.py:83-98), mask on the device
            a_spec = torch.empty_like(D)
            v_spec = torch.empty_like(D)
            ctx.check(ctx.lib.vr_apply_mask(ctx.handle, _native.ptr(D), _native.ptr(mask), D.shape[2],
                                            _native.ptr(a_spec), _native.ptr(v_spec), _native.stream_ptr()), 'vr_apply_mask')
            return (y + a_spec).cpu().numpy()                  # pseudo.py:69


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--gpu', '-g', type=int, default=-1)
    p.add_argument('--pretrained_model', '-P', type=str, default='models/baseline.pth')
    p.add_argument('--mixtures', '-m', required=True)
    p.add_argument('--instruments', '-i', required=True)
    p.add_argument('--sr', '-r', type=int, default=44100)
    p.add_argument('--n_fft', '-f', type=int, default=2048)
    p.add_argument('--hop_length', '-H', type=int, default=1024)
    p.add_argument('--batchsize', '-B', type=int, default=4)
    p.add_argument('--cropsize', '-c', type=int, default=256)
    p.add_argument('--postprocess', '-p', action='store_true')
    p.add_argument('--output_dir', '-o', type=str, default='pseudo')
    args = p.parse_args()

    if not torch.cuda.is_available():
        raise RuntimeError('no CUDA device: the H100 build of vocal-remover has no CPU path')
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    # one process per GPU under torchrun; a single process uses --gpu (the reference's -1 = CPU means cuda:0 here)
    index = local if world > 1 else max(args.gpu, 0)
    if world == 1 and args.gpu < 0:
        print('note: --gpu {} selects the CPU in the reference; this build has no CPU path and uses cuda:0'.format(args.gpu))

    print('loading model...', end=' ')
    device = torch.device('cuda:{}'.format(index))
    model = nets.CascadedNet(args.n_fft, args.hop_length)
    model.load_state_dict(torch.load(args.pretrained_model, map_location='cpu'))
    model.to(device)
    spec_utils.set_device(index)
    print('done')

    os.makedirs(args.output_dir, exist_ok=True)
    labeler = PseudoLabeler(model, device, args.batchsize, args.cropsize, args.postprocess)
    filelist = dataset.shard_files(dataset.make_pair(args.mixtures, args.instruments), world, rank)
    for mix_path, inst_path in filelist:
        basename = os.path.splitext(os.path.basename(mix_path))[0]
        print(basename)

        print('loading wave source...', end=' ')
        X, sr = audio_io.load(mix_path, sr=args.sr, mono=False, dtype=np.float32, device=device)
        y, sr = audio_io.load(inst_path, sr=args.sr, mono=False, dtype=np.float32, device=device)
        print('done')

        if X.ndim == 1:
            # mono to stereo
            X = np.asarray([X, X])

        print('stft of wave source, separation...', end=' ')
        X, y = spec_utils.align_wave_head_and_tail(X, y, sr)
        pseudo_inst = labeler.pseudo_instruments(X, y)
        print('done')

        audio_io.write(os.path.join(args.output_dir, '{}_PseudoInstruments.wav'.format(basename)), np.zeros((1, 1)), sr)
        np.save(os.path.join(args.output_dir, '{}_PseudoInstruments.npy'.format(basename)), pseudo_inst)


if __name__ == '__main__':
    main()
