"""Validation loss of a checkpoint over a dataset of (mixture, instruments) pairs, on the GPU.

The number the reference's train.py reports once per epoch (``validate_epoch``, train.py:108-134, over
``make_validation_set`` + ``VocalRemoverValidationSet``, lib/dataset.py:220-248), without training: per pair
``X, y = cache_or_load(...)``, ``coef = max(max|X|, max|y|)``, ``ceil(T / roi)`` patches of the padded ``X / coef``
through the net, and the L1 distance of ``mask * |X| / coef`` from ``|y| / coef`` over the kept frames.  The loss is
the mean of the per-patch losses, which is what ``validate_epoch`` returns since all patches are the same size.

The patches never leave the GPU: one ``vr_validation_loss`` call per pair runs the windows through the net and
reduces each window's L1 sum on the device, so the reference's npz patch cache (``cs{..}_of{..}/`` in the working
directory) is not written.  The spectrogram caches are the reference's own (``spec_utils.cache_or_load``).

Same flags as train.py for what validation uses (-g -s -r -H -f -d -S -v -V -b -c -P; -P is required).  The split is
the reference's: ``random.seed(seed)`` and then ``train_val_split``, so ``-s`` / ``-v`` pick the pairs train.py would
validate on.  Under ``torchrun --nproc-per-node N validate.py ...`` every rank takes the pairs
``dataset.shard_files(filelist, N, rank)`` and rank 0 combines the per-window sums in file order, so the printed loss
does not depend on N.
"""
import argparse
import json
import math
import os
import random

import numpy as np
import torch

from lib import _native
from lib import dataset
from lib import nets
from lib import spec_utils


class Validator(object):
    """Per-window L1 sums of track pairs on one GPU (vr_validation_loss) for ``model`` at a cropsize and batch size."""

    def __init__(self, model, device=None, cropsize=256, batchsize=4):
        self.model = model
        self.cropsize = int(cropsize)
        self.batchsize = int(batchsize)
        self.bins = model.n_fft // 2 + 1
        self.roi = dataset.make_padding(0, self.cropsize, model.offset)[2]
        if device is not None:
            model.to(device)

    def patch_count(self, n_frames):
        return dataset.validation_patch_count(n_frames, self.cropsize, self.model.offset)

    def patch_losses(self, window_sums):
        """Per-patch L1Loss (the mean over (2, bins, roi)) from the per-window sums."""
        return np.asarray(window_sums, dtype=np.float64) / float(2 * self.bins * self.roi)

    def window_sums(self, X, y, name='pair'):
        """complex (2, bins, T) mixture / instruments spectrograms (numpy or CUDA tensors) -> float64 numpy
        (ceil(T / roi),) sums of |mask * |X| / coef - |y| / coef| per patch.  Raises ValueError naming ``name`` when
        coef = max(max|X|, max|y|) is zero or not finite (the reference's loss is NaN there)."""
        ctx = self.model.native_context(self.cropsize, self.batchsize)
        dev = torch.device('cuda', ctx.device_index)
        with torch.cuda.device(dev):
            d_x, d_y = (self._to_device(s, dev) for s in (X, y))
            if d_x.shape != d_y.shape or d_x.dim() != 3 or d_x.shape[0] != 2 or d_x.shape[1] != self.bins:
                raise ValueError('%s: X and y must both have shape (2, %d, T), got %s and %s'
                                 % (name, self.bins, tuple(d_x.shape), tuple(d_y.shape)))
            T = d_x.shape[2]
            coef = torch.empty(1, dtype=torch.float32, device=dev)
            sums = torch.empty(self.patch_count(T), dtype=torch.float64, device=dev)
            ctx.check(ctx.lib.vr_validation_loss(ctx.handle, _native.ptr(d_x), _native.ptr(d_y), T, _native.ptr(coef),
                                                 _native.ptr(sums), _native.stream_ptr()), 'vr_validation_loss')
            c = float(coef.item())
            if not (c > 0 and math.isfinite(c)):
                raise ValueError('%s: max(|X|.max(), |y|.max()) is %r, so the validation loss is undefined (the '
                                 'reference divides by it)' % (name, c))
            return sums.cpu().numpy()

    @staticmethod
    def _to_device(s, dev):
        if torch.is_tensor(s):
            if s.device != dev:
                raise ValueError('spectrogram is on %s, the model on %s' % (s.device, dev))
            return s.to(torch.complex64).contiguous()
        return torch.from_numpy(np.ascontiguousarray(np.asarray(s, dtype=np.complex64))).to(dev)


def pair_name(X_path, y_path):
    return '{} {}'.format(os.path.basename(X_path), os.path.basename(y_path))


def file_window_sums(validator, filelist, sr, hop_length, n_fft, on_pair=None):
    """Per-window sums of every pair of ``filelist``, in order; ``on_pair(k, sums)`` after pair k."""
    out = []
    for k, (X_path, y_path) in enumerate(filelist):
        X, y, _, _ = spec_utils.cache_or_load(X_path, y_path, sr, hop_length, n_fft)
        out.append(validator.window_sums(X, y, name=pair_name(X_path, y_path)))
        if on_pair is not None:
            on_pair(k, out[-1])
    return out


def combine(validator, per_file_sums):
    """The validation loss from the per-window sums of all pairs: the mean of the per-patch losses.  ``math.fsum``
    rounds the exact total once, so the result does not depend on how the pairs were spread over ranks."""
    losses = [validator.patch_losses(s) for s in per_file_sums]
    count = sum(len(l) for l in losses)
    if count == 0:
        raise ValueError('no validation pairs')
    return math.fsum(float(v) for l in losses for v in l) / count


def gather_window_sums(local, world, rank, group=None):
    """Rank ``rank``'s per-file sums (of ``dataset.shard_files(filelist, world, rank)``) -> on rank 0 the sums of all
    files in the global file order, None on the other ranks.  Host arrays are exchanged whole (8 bytes per window)."""
    local = list(local)
    if world == 1:
        return local
    import torch.distributed as dist
    gathered = [None] * world if rank == 0 else None
    dist.gather_object(local, gathered, dst=0, group=group)
    if rank != 0:
        return None
    n = sum(len(g) for g in gathered)
    # shard_files is round-robin: global file i is file i // world of rank i % world
    return [gathered[i % world][i // world] for i in range(n)]


def validation_loss(model, device, filelist, sr=44100, hop_length=1024, n_fft=2048, cropsize=256, batchsize=4):
    """train.py's ``validate_epoch`` over ``make_validation_set(filelist, cropsize, sr, hop_length, n_fft,
    model.offset)``: the mean L1 loss of ``model.predict`` over all validation patches of ``filelist``."""
    validator = Validator(model, device, cropsize, batchsize)
    return combine(validator, file_window_sums(validator, filelist, sr, hop_length, n_fft))


def main():
    p = argparse.ArgumentParser(description='validation loss of a checkpoint (train.py validate_epoch) on the GPU')
    p.add_argument('--gpu', '-g', type=int, default=-1)
    p.add_argument('--seed', '-s', type=int, default=2019)
    p.add_argument('--sr', '-r', type=int, default=44100)
    p.add_argument('--hop_length', '-H', type=int, default=1024)
    p.add_argument('--n_fft', '-f', type=int, default=2048)
    p.add_argument('--dataset', '-d', required=True)
    p.add_argument('--split_mode', '-S', type=str, choices=['random', 'subdirs'], default='random')
    p.add_argument('--val_rate', '-v', type=float, default=0.2)
    p.add_argument('--val_filelist', '-V', type=str, default=None)
    p.add_argument('--val_batchsize', '-b', type=int, default=4)
    p.add_argument('--val_cropsize', '-c', type=int, default=256)
    p.add_argument('--pretrained_model', '-P', type=str, required=True)
    args = p.parse_args()

    # argument and dataset errors come before the model is loaded
    if not os.path.isfile(args.pretrained_model):
        p.error('--pretrained_model: no such file: {}'.format(args.pretrained_model))
    if args.val_batchsize < 1:
        p.error('--val_batchsize must be at least 1')
    if args.val_cropsize <= 2 * 64:
        p.error('--val_cropsize must exceed 128 (twice the model offset): the model keeps no frame otherwise')
    random.seed(args.seed)   # train.py:170, before the split
    val_filelist = []
    if args.val_filelist is not None:
        with open(args.val_filelist, 'r', encoding='utf8') as f:
            val_filelist = json.load(f)
    try:
        _, val_filelist = dataset.train_val_split(args.dataset, args.split_mode, args.val_rate, val_filelist)
    except (ValueError, OSError) as e:
        p.error(str(e))
    if len(val_filelist) == 0:
        p.error('no validation pairs in {}'.format(args.dataset))

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
        dist.init_process_group('gloo')   # only the per-window sums are exchanged, on the host

    if rank == 0:
        print('loading model...', end=' ')
    device = torch.device('cuda:{}'.format(index))
    model = nets.CascadedNet(args.n_fft, args.hop_length, 32, 128)
    model.load_state_dict(torch.load(args.pretrained_model, map_location='cpu'))
    model.to(device)
    spec_utils.set_device(index)
    if rank == 0:
        print('done')

    validator = Validator(model, device, args.val_cropsize, args.val_batchsize)

    def report(i, sums):
        X_path, y_path = val_filelist[i]
        print('{} {} {:.6f}'.format(i + 1, pair_name(X_path, y_path), float(np.mean(validator.patch_losses(sums)))))

    local_files = dataset.shard_files(val_filelist, world, rank)
    local_sums = file_window_sums(validator, local_files, args.sr, args.hop_length, args.n_fft,
                                  on_pair=report if world == 1 else None)
    all_sums = gather_window_sums(local_sums, world, rank)
    if rank == 0:
        if world > 1:
            for i, sums in enumerate(all_sums):
                report(i, sums)
        print('validation loss = {:.6f}'.format(combine(validator, all_sums)))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
