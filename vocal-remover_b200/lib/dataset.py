"""Inference-side pieces of the reference's lib/dataset.py: the window geometry used by Separator, the file pairing
used by pseudo.py and the train / validation split and patch count used by validate.py (training-set construction is
out of scope, SURVEY 2)."""
import os
import random


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
