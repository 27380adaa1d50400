"""Inference-side pieces of the reference's lib/dataset.py: the window geometry used by Separator, the file pairing
used by pseudo.py, the train / validation split and patch count used by validate.py, and the dataset inspection
tool (training-set construction is out of scope, SURVEY 2).

Run as a script, it is the reference's vocal JPG tool (lib/dataset.py:262-287): for every pair of
``make_pair(mix_dir, inst_dir)`` it writes ``<outdir>/<mix basename>_Vocal.jpg``, the image of the vocal energy the
instrumental track lacks, from the pair's cached spectrograms (``spec_utils.cache_or_load``)::

    python lib/dataset.py <mix_dir> <inst_dir> <outdir>        (or python -m lib.dataset ...)

Under ``torchrun --nproc-per-node N`` every rank takes ``shard_files(pairs, N, rank)`` on ``cuda:LOCAL_RANK``.
"""
import os
import random
import sys

if __name__ == '__main__' and not __package__:
    # run as a file: import the package this file belongs to instead of its modules as top-level ones
    _LIB_DIR = os.path.dirname(os.path.abspath(__file__))
    if sys.path and os.path.abspath(sys.path[0] or os.curdir) == _LIB_DIR:
        del sys.path[0]
    sys.path.insert(0, os.path.dirname(_LIB_DIR))
    __package__ = 'lib'

import numpy as np
import torch

from . import _native
from . import spec_utils


def make_padding(width, cropsize, offset):
    """Same contract as the reference's lib/dataset.py:198-205: returns (left, right, roi_size).

    The padded width left + width + right is a multiple of roi_size plus 2*offset, so the padded
    spectrogram splits into whole cropsize-wide windows at stride roi_size.
    """
    roi_size = cropsize - 2 * offset
    if roi_size == 0:
        roi_size = cropsize
    return offset, roi_size - (width % roi_size) + offset, roi_size


INPUT_EXTS = ['.wav', '.m4a', '.mp3', '.mp4', '.flac']


def make_pair(mix_dir, inst_dir):
    """lib/dataset.py:144-160: sorted mixture / instrument files of two directories, zipped pairwise."""
    X_list = sorted([os.path.join(mix_dir, fname) for fname in os.listdir(mix_dir)
                     if os.path.splitext(fname)[1] in INPUT_EXTS])
    y_list = sorted([os.path.join(inst_dir, fname) for fname in os.listdir(inst_dir)
                     if os.path.splitext(fname)[1] in INPUT_EXTS])
    return list(zip(X_list, y_list))


def train_val_split(dataset_dir, split_mode, val_rate, val_filelist):
    """lib/dataset.py:163-195: (train_filelist, val_filelist) of ``dataset_dir``.

    'random' pairs ``mixtures/`` with ``instruments/``, shuffles the pairs with ``random.shuffle`` (seed ``random``
    first to reproduce a split) and keeps the last ``int(len * val_rate)`` as validation, unless ``val_filelist`` (a
    list of [mixture, instruments] paths) is given: that list is then the validation set as it stands and the training
    set is every other pair.  'subdirs' pairs ``training/`` and ``validation/`` and refuses a ``val_filelist``.  As in
    the reference, a ``val_rate`` that rounds to zero pairs makes every pair a validation pair.
    """
    if split_mode == 'random':
        filelist = make_pair(os.path.join(dataset_dir, 'mixtures'), os.path.join(dataset_dir, 'instruments'))
        random.shuffle(filelist)
        if len(val_filelist) == 0:
            val_size = int(len(filelist) * val_rate)
            train_filelist = filelist[:-val_size]
            val_filelist = filelist[-val_size:]
        else:
            train_filelist = [pair for pair in filelist if list(pair) not in val_filelist]
    elif split_mode == 'subdirs':
        if len(val_filelist) != 0:
            raise ValueError('`val_filelist` option is not available with `subdirs` mode')
        train_filelist = make_pair(os.path.join(dataset_dir, 'training/mixtures'),
                                   os.path.join(dataset_dir, 'training/instruments'))
        val_filelist = make_pair(os.path.join(dataset_dir, 'validation/mixtures'),
                                 os.path.join(dataset_dir, 'validation/instruments'))
    return train_filelist, val_filelist


def validation_patch_count(n_frames, cropsize, offset):
    """Patches ``make_validation_set`` cuts from a track of ``n_frames`` frames (lib/dataset.py:236): ceil(T / roi).
    Separator cuts (W_pad - 2*offset) // roi windows instead, one more when T is a multiple of roi."""
    roi = make_padding(n_frames, cropsize, offset)[2]
    return -(-int(n_frames) // roi)


def shard_files(filelist, world, rank):
    """File-level sharding of a many-file job (pseudo.py:41-74) over ``world`` processes (one per GPU): round-robin, so
    that every rank gets a similar mix of track lengths; whole files, no exchange between ranks."""
    return [f for i, f in enumerate(filelist) if i % world == rank]


def vocal_image(X_spec, y_spec):
    """Mixture / instruments spectrograms, complex (2, bins, T) each -> uint8 (bins, T, 3) image {max(L, R), L, R} of
    ``spectrogram_to_image(v_mag)`` with ``v_mag = |X| - |y|`` kept where ``v_mag > |y|`` (lib/dataset.py:280-286).

    Built on the GPU (vr_vocal_image).  Numpy arrays give a numpy image, CUDA complex64 tensors a CUDA uint8 tensor.
    A constant ``v_mag`` (e.g. a silent pair) gives an all-zero image where the reference's uint8 cast sees NaN.
    """
    on_device = torch.is_tensor(X_spec)
    if torch.is_tensor(y_spec) != on_device:
        raise TypeError('vocal_image: X_spec and y_spec must both be numpy arrays or both CUDA tensors')
    if not on_device:
        X_spec, y_spec = np.asarray(X_spec), np.asarray(y_spec)
    for s in (X_spec, y_spec):
        if not (s.is_complex() if on_device else np.iscomplexobj(s)):
            raise ValueError('vocal_image: the spectrograms must be complex')
    if X_spec.ndim != 3 or X_spec.shape[0] != 2 or tuple(X_spec.shape) != tuple(y_spec.shape):
        raise ValueError('vocal_image: X_spec and y_spec must both have shape (2, bins, T), got %s and %s'
                         % (tuple(X_spec.shape), tuple(y_spec.shape)))
    bins, T = X_spec.shape[1], X_spec.shape[2]
    ctx = spec_utils._spectral_ctx(2 * (bins - 1), bins - 1)
    dev = torch.device('cuda', ctx.device_index)
    with torch.cuda.device(dev):
        d_x, d_y = (spec_utils._to_device(s, dev, 'vocal_image') for s in (X_spec, y_spec))
        img = torch.empty((bins, T, 3), dtype=torch.uint8, device=dev)
        ctx.check(ctx.lib.vr_vocal_image(ctx.handle, _native.ptr(d_x), _native.ptr(d_y), T, _native.ptr(img),
                                         _native.stream_ptr()), 'vr_vocal_image')
        return img if on_device else img.cpu().numpy()


def main(argv=None):
    """The reference's vocal JPG tool: ``<outdir>/<mix basename>_Vocal.jpg`` for every pair of the two directories."""
    import argparse
    from . import utils
    p = argparse.ArgumentParser(prog='lib/dataset.py',
                                description='writes <outdir>/<mix basename>_Vocal.jpg for every (mixture, '
                                            'instruments) pair: the vocal energy the instrumental track lacks')
    p.add_argument('mix_dir')
    p.add_argument('inst_dir')
    p.add_argument('outdir')
    args = p.parse_args(argv)

    # missing requirements fail before any file or directory is written
    try:
        import cv2  # noqa: F401  (the JPEG encoder of lib/utils.imwrite)
    except ImportError as e:
        raise ImportError('the vocal JPG tool needs OpenCV (the cv2 module) to encode the JPGs: %s' % e) from e
    if not torch.cuda.is_available():
        raise RuntimeError('no CUDA device: the H100 build of vocal-remover has no CPU path')
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    index = int(os.environ.get('LOCAL_RANK', '0')) if world > 1 else 0
    spec_utils.set_device(index)

    os.makedirs(args.outdir, exist_ok=True)
    # the reference's fixed spectrogram parameters, so that the caches are the ones its training reads
    sr, hop_length, n_fft = 44100, 1024, 2048
    for mix_path, inst_path in shard_files(make_pair(args.mix_dir, args.inst_dir), world, rank):
        mix_basename = os.path.splitext(os.path.basename(mix_path))[0]
        outpath = '{}/{}_Vocal.jpg'.format(args.outdir, mix_basename)
        X_spec, y_spec, _, _ = spec_utils.cache_or_load(mix_path, inst_path, sr, hop_length, n_fft)
        if X_spec.shape[2] > utils.JPEG_MAX_WIDTH:
            # the reference's cv2.imencode refuses the image and its imwrite returns False: no JPG
            print('skipping {}: {} frames exceed the {}-pixel width limit of JPEG'.format(
                outpath, X_spec.shape[2], utils.JPEG_MAX_WIDTH))
            continue
        utils.imwrite(outpath, vocal_image(X_spec, y_spec))
        print(outpath)


if __name__ == '__main__':
    main()
