"""BSS Eval SDR, ISR, SIR and SAR of a checkpoint's separated stems over a dataset of (mixture, instruments) pairs, on
the GPU.

The numbers the SiSEC campaigns report, for the pairs validate.py would validate on (or every pair with ``--all``):
per pair, both files are loaded and aligned as ``spec_utils.cache_or_load`` does, the true stems are the instruments
``y`` and the vocals ``X - y``, the estimates are ``Separator.separate_wave`` of the mixture (kept on the device), and
``lib/bsseval.bss_eval`` scores every ``--window`` second frame, hopping ``--hop`` seconds.  Each pair prints the median
over its frames of the four ratios of both stems; the last line is the median over the pairs of those medians.
``--json`` writes every frame's values as well.  ``--framewise_filters`` scores with BSS Eval v3 instead (distortion
filters solved for each frame on its own samples; ``--window`` of at least ``--filters_len`` samples).

Split flags as validate.py (-g -s -r -H -f -d -S -v -V -P), separation flags as inference.py (-B -c -t -p).  Under
``torchrun --nproc-per-node N evaluate.py ...`` every rank scores the pairs ``dataset.shard_files(filelist, N, rank)``
and rank 0 prints them in file order; each pair is scored on one GPU, so the numbers do not depend on N.
"""
import argparse
import json
import math
import os
import random

import numpy as np
import torch

import inference
import validate
from lib import audio_io
from lib import bsseval
from lib import dataset
from lib import nets
from lib import spec_utils

STEMS = ('instruments', 'vocals')


def pair_waves(X_path, y_path, sr, device=None):
    """The aligned mixture and instruments of a pair, float32 (2, L) each, as cache_or_load aligns them."""
    X, _ = audio_io.load(X_path, sr=sr, mono=False, dtype=np.float32, device=device)
    y, _ = audio_io.load(y_path, sr=sr, mono=False, dtype=np.float32, device=device)
    X, y = (np.asarray([w, w]) if w.ndim == 1 else w for w in (X, y))
    return spec_utils.align_wave_head_and_tail(X, y, sr)


def score_pair(separator, X, y, window, hop, filters_len, tta=False, framewise=False):
    """Frame metrics of one aligned pair: the estimates of ``separator`` against references (y, X - y), both cut to
    the hop * (L // hop) samples separate_wave returns.  dict of (2, nwin) arrays, rows instruments, vocals.
    ``framewise``: BSS Eval v3 filters, solved per frame (bsseval.bss_eval)."""
    dev = separator._dev()
    with torch.cuda.device(dev):
        d_x = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(dev)
        d_y = torch.from_numpy(np.ascontiguousarray(y, dtype=np.float32)).to(dev)
        inst, voc = separator.separate_wave(d_x, tta)
        n = inst.shape[1]
        refs = torch.stack([d_y[:, :n], (d_x - d_y)[:, :n]])
        ests = torch.stack([inst, voc])
        return bsseval.bss_eval(refs, ests, window, hop, filters_len, device=dev, framewise=framewise)


def dataset_medians(per_track):
    """Median over the tracks of each per-track median (tracks with a NaN median left out): dict of (2,)."""
    out = {}
    for m in bsseval.METRICS:
        v = np.asarray([bsseval.track_medians(r)[m] for r in per_track], dtype=np.float64).reshape(-1, len(STEMS))
        out[m] = np.asarray([np.median(c[~np.isnan(c)]) if np.any(~np.isnan(c)) else np.nan for c in v.T])
    return out


def format_values(med):
    return ' '.join('{} {}'.format(stem, ' '.join('{} {:.3f}'.format(m.upper(), float(med[m][k]))
                                                  for m in ('sdr', 'isr', 'sir', 'sar')))
                    for k, stem in enumerate(STEMS))


def _nan_to_none(v):
    return [None if math.isnan(x) else float(x) for x in np.asarray(v, dtype=np.float64).ravel()]


def to_json(filelist, per_track, args_dict):
    tracks = []
    for (X_path, y_path), r in zip(filelist, per_track):
        med = bsseval.track_medians(r)
        tracks.append({'mixture': X_path, 'instruments': y_path,
                       'frames': {stem: {m: _nan_to_none(r[m][k]) for m in bsseval.METRICS}
                                  for k, stem in enumerate(STEMS)},
                       'median': {stem: {m: _nan_to_none(med[m][k:k + 1])[0] for m in bsseval.METRICS}
                                  for k, stem in enumerate(STEMS)}})
    total = dataset_medians(per_track)
    return dict(args_dict, tracks=tracks,
                median={stem: {m: _nan_to_none(total[m][k:k + 1])[0] for m in bsseval.METRICS}
                        for k, stem in enumerate(STEMS)})


def build_parser():
    p = argparse.ArgumentParser(description='BSS Eval SDR / ISR / SIR / SAR of a checkpoint over a dataset, on the GPU')
    p.add_argument('--gpu', '-g', type=int, default=-1)
    p.add_argument('--seed', '-s', type=int, default=2019)
    p.add_argument('--sr', '-r', type=int, default=44100)
    p.add_argument('--hop_length', '-H', type=int, default=1024)
    p.add_argument('--n_fft', '-f', type=int, default=2048)
    p.add_argument('--dataset', '-d', required=True)
    p.add_argument('--split_mode', '-S', type=str, choices=['random', 'subdirs'], default='random')
    p.add_argument('--val_rate', '-v', type=float, default=0.2)
    p.add_argument('--val_filelist', '-V', type=str, default=None)
    p.add_argument('--pretrained_model', '-P', type=str, required=True)
    p.add_argument('--batchsize', '-B', type=int, default=4)
    p.add_argument('--cropsize', '-c', type=int, default=256)
    p.add_argument('--tta', '-t', action='store_true')
    p.add_argument('--postprocess', '-p', action='store_true')
    p.add_argument('--all', action='store_true', help='score every pair of the dataset, not the validation split')
    p.add_argument('--window', type=float, default=1.0, help='frame length in seconds')
    p.add_argument('--hop', type=float, default=1.0, help='frame advance in seconds')
    p.add_argument('--filters_len', type=int, default=512, help='taps of the distortion filters')
    p.add_argument('--json', type=str, default=None, help='write every frame value to this file')
    p.add_argument('--framewise_filters', action='store_true',
                   help='BSS Eval v3: solve the distortion filters for each frame on its own samples (the SiSEC '
                        'campaigns before 2018), instead of once per track')
    return p


def select_pairs(p, args):
    """The pairs to score, or a parser error (before the model loads)."""
    random.seed(args.seed)   # as validate.py / train.py, before the split
    val_filelist = []
    if args.val_filelist is not None:
        with open(args.val_filelist, 'r', encoding='utf8') as f:
            val_filelist = json.load(f)
    try:
        train, val = dataset.train_val_split(args.dataset, args.split_mode, args.val_rate, val_filelist)
        if args.all:
            if args.split_mode == 'random':
                pairs = dataset.make_pair(os.path.join(args.dataset, 'mixtures'),
                                          os.path.join(args.dataset, 'instruments'))
            else:
                pairs = list(train) + list(val)
        else:
            pairs = val
    except (ValueError, OSError) as e:
        p.error(str(e))
    if len(pairs) == 0:
        p.error('no pairs to score in {}'.format(args.dataset))
    return [list(x) for x in pairs]


def main():
    p = build_parser()
    args = p.parse_args()

    # argument and dataset errors come before the model is loaded
    if not os.path.isfile(args.pretrained_model):
        p.error('--pretrained_model: no such file: {}'.format(args.pretrained_model))
    if args.batchsize < 1:
        p.error('--batchsize must be at least 1')
    if args.cropsize <= 2 * 64:
        p.error('--cropsize must exceed 128 (twice the model offset): the model keeps no frame otherwise')
    window, hop = int(round(args.window * args.sr)), int(round(args.hop * args.sr))
    if window < 1 or hop < 1:
        p.error('--window and --hop must be at least one sample')
    if not 1 <= args.filters_len <= bsseval.MAX_FILTER:
        p.error('--filters_len must be in [1, {}]'.format(bsseval.MAX_FILTER))
    if args.framewise_filters and window < args.filters_len:
        p.error('--framewise_filters needs a --window of at least --filters_len ({}) samples, got {}'.format(
            args.filters_len, window))
    if args.json is not None and not os.path.isdir(os.path.dirname(os.path.abspath(args.json))):
        p.error('--json: no such directory: {}'.format(os.path.dirname(os.path.abspath(args.json))))
    filelist = select_pairs(p, args)

    if not torch.cuda.is_available():
        raise RuntimeError('no CUDA device: the H100 build of vocal-remover has no CPU path')
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    index = local if world > 1 else max(args.gpu, 0)
    if world == 1 and args.gpu < 0:
        print('note: --gpu {} selects the CPU in the reference; this build has no CPU path and uses cuda:0'.format(args.gpu))
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group('gloo')   # only the per-frame values are exchanged, on the host

    if rank == 0:
        print('loading model...', end=' ')
    device = torch.device('cuda:{}'.format(index))
    torch.cuda.set_device(device)
    model = nets.CascadedNet(args.n_fft, args.hop_length, 32, 128)
    model.load_state_dict(torch.load(args.pretrained_model, map_location='cpu'))
    model.to(device)
    spec_utils.set_device(index)
    if rank == 0:
        print('done')
    sp = inference.Separator(model, device, args.batchsize, args.cropsize, args.postprocess)

    def report(i, result):
        X_path, y_path = filelist[i]
        print('{} {} {}'.format(i + 1, validate.pair_name(X_path, y_path), format_values(bsseval.track_medians(result))))

    local_results = []
    for k, (X_path, y_path) in enumerate(dataset.shard_files(filelist, world, rank)):
        X, y = pair_waves(X_path, y_path, args.sr, index)
        try:
            local_results.append(score_pair(sp, X, y, window, hop, args.filters_len, args.tta,
                                            args.framewise_filters))
        except ValueError as e:
            raise ValueError('{}: {}'.format(validate.pair_name(X_path, y_path), e)) from e
        if world == 1:
            report(k, local_results[-1])
    results = validate.gather_window_sums(local_results, world, rank)
    if rank == 0:
        if world > 1:
            for i, r in enumerate(results):
                report(i, r)
        print('median of {} pairs: {}'.format(len(results), format_values(dataset_medians(results))))
        if args.json is not None:
            info = {'sr': args.sr, 'window': window, 'hop': hop, 'filters_len': args.filters_len}
            if args.framewise_filters:
                info['framewise_filters'] = True
            with open(args.json, 'w') as f:
                json.dump(to_json(filelist, results, info), f)
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
