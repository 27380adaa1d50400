"""CPU oracle and golden recipe of the validation loss (validate.py).  TEST INFRASTRUCTURE.

``patch_losses`` restates the reference's validation loss (train.py:108-134 ``validate_epoch`` over
lib/dataset.py:220-248 ``make_validation_set`` + ``VocalRemoverValidationSet``) for one (mixture, instruments) pair
in numpy + ``oracle.net_oracle``; ``validation_cases`` regenerates the seeded pairs of the fixture
``tests/golden/ref_validation.partN.npz``, which ``run_validation`` writes from the UNMODIFIED reference's
``make_validation_set``, ``VocalRemoverValidationSet``, ``train.validate_epoch`` and ``train_val_split`` on CPU.  The
spectrograms are the oracle STFT's, written as the reference's ``cache_or_load`` caches so that librosa is never
called.  Regenerate with ``VR_REFERENCE_ROOT=<checkout> python -m oracle.validation_oracle`` from the repo root; it
writes only ref_validation.*.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import net_oracle, separator_oracle, stft_oracle

SR, HOP, N_FFT, CROPSIZE, OFFSET = 44100, 1024, 2048, 256, 64
# frames per pair: a multiple of roi (128), fewer than roi, and two generic lengths
FRAMES = (256, 100, 300, 131)
VAL_BATCHSIZE = 4
SPLIT_SEED, SPLIT_RATE, SPLIT_PAIRS = 2019, 0.2, 10


def validation_cases():
    """[(name, mixture wave, instruments wave)], float32 (2, L) with 1 + L // HOP = FRAMES[k]: a few tones plus noise;
    the instruments are the mixture without one tone ("the vocal") plus noise of their own."""
    rng = np.random.default_rng(7)
    cases = []
    for k, T in enumerate(FRAMES):
        L = (T - 1) * HOP + int(rng.integers(0, HOP))
        t = np.arange(L, dtype=np.float64) / SR
        tones = []
        for _ in range(4):
            f = rng.uniform(80.0, 8000.0, size=2)
            a = rng.uniform(0.05, 0.3, size=2)
            ph = rng.uniform(-np.pi, np.pi, size=2)
            tones.append(a[:, None] * np.sin(2 * np.pi * f[:, None] * t[None, :] + ph[:, None]))
        mix = sum(tones) + 0.01 * rng.standard_normal((2, L))
        inst = mix - tones[k % len(tones)] + 0.005 * rng.standard_normal((2, L))
        cases.append(('pair%d' % k, mix.astype(np.float32), inst.astype(np.float32)))
    return cases


def spectrograms():
    """[(name, X, y)] complex64 (2, 1025, T) oracle STFTs of validation_cases()."""
    return [(name, stft_oracle.wave_to_spectrogram(a, HOP, N_FFT), stft_oracle.wave_to_spectrogram(b, HOP, N_FFT))
            for name, a, b in validation_cases()]


def split_names():
    """Basenames of the synthetic dataset listing of the train_val_split case (plus one non-audio file)."""
    return ['track%02d' % i for i in range(SPLIT_PAIRS)]


def patch_losses(sd, X, y, cropsize=CROPSIZE, offset=OFFSET, n_fft=N_FFT):
    """float64 (ceil(T / roi),) losses of one pair: L1Loss(predict(|X_p|), crop_center(|y_p|)) per patch p, with
    X_p, y_p the cropsize-frame patches of X / coef, y / coef padded by make_padding (lib/dataset.py:225-247)."""
    coef = np.max([np.abs(X).max(), np.abs(y).max()])
    X, y = X / coef, y / coef
    l, r, roi = separator_oracle.make_padding(X.shape[2], cropsize, offset)
    X_pad = np.pad(X, ((0, 0), (0, 0), (l, r)), mode='constant')
    y_pad = np.pad(y, ((0, 0), (0, 0), (l, r)), mode='constant')
    out = []
    for j in range(int(np.ceil(X.shape[2] / roi))):
        s = j * roi
        x_mag = torch.from_numpy(np.abs(X_pad[None, :, :, s:s + cropsize]))
        y_mag = torch.from_numpy(np.abs(y_pad[None, :, :, s:s + cropsize]))
        pred = (x_mag * net_oracle.forward(sd, x_mag, n_fft))[:, :, :, offset:-offset]   # lib/nets.py:133-141
        y_crop = net_oracle.crop_center(y_mag, pred)
        out.append(F.l1_loss(pred, y_crop).item())
    return np.asarray(out, dtype=np.float64)


def _reference_train(ref_root):
    """The reference's train.py as a module.  It imports ``from lib import ...``: the reference's own lib (kept as
    ``_ref_lib*`` by librosa_shim.import_reference) stands in for ``lib`` while it is imported, then the previous
    ``lib`` modules come back."""
    import importlib.util
    import os
    import sys
    names = [k[len('_ref_'):] for k in sys.modules if k == '_ref_lib' or k.startswith('_ref_lib.')]
    saved = {k: sys.modules.get(k) for k in names}
    try:
        for k in names:
            sys.modules[k] = sys.modules['_ref_' + k]
        spec = importlib.util.spec_from_file_location('_ref_train', os.path.join(ref_root, 'train.py'))
        train = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(train)
    finally:
        for k, mod in saved.items():
            if mod is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = mod
    return train


def run_validation():
    """Reference per-patch losses (one validate_epoch per single-patch dataset), the val_batchsize = 4 total over all
    patches, and the train_val_split of a synthetic listing, in a temporary working directory."""
    import os
    import random
    import tempfile
    import torch.utils.data
    from oracle import librosa_shim, make_golden
    from lib import synth
    _, ref_nets, _, ref_dataset = librosa_shim.import_reference()
    train = _reference_train(librosa_shim.REFERENCE_ROOT)
    model = ref_nets.CascadedNet(N_FFT, HOP, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    model.eval()
    cpu = torch.device('cpu')
    out = {'T': np.asarray(FRAMES, dtype=np.int64)}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            filelist = []
            cache = 'sr{}_hl{}_nf{}'.format(SR, HOP, N_FFT)
            for (name, X, y), (_, a, b) in zip(spectrograms(), validation_cases()):
                out[name + '_wave_sum'] = np.stack([make_golden.checksum(a), make_golden.checksum(b)])
                out[name + '_spec_sum'] = np.stack([make_golden.checksum(X), make_golden.checksum(y)])
                pair = []
                for sub, spec in (('mixtures', X), ('instruments', y)):
                    os.makedirs(os.path.join('data', sub, cache), exist_ok=True)
                    open(os.path.join('data', sub, name + '.wav'), 'wb').close()   # never decoded: the cache hits
                    np.save(os.path.join('data', sub, cache, name + '.npy'), spec.transpose(2, 0, 1))
                    pair.append(os.path.join('data', sub, name + '.wav'))
                filelist.append(tuple(pair))
            patches = ref_dataset.make_validation_set(filelist, CROPSIZE, SR, HOP, N_FFT, model.offset)

            def epoch(patch_list, batchsize):
                loader = torch.utils.data.DataLoader(ref_dataset.VocalRemoverValidationSet(patch_list),
                                                     batch_size=batchsize, shuffle=False, num_workers=0)
                return train.validate_epoch(loader, model, cpu)
            out['patch_losses'] = np.asarray([epoch([p], 1) for p in patches], dtype=np.float64)
            out['total_b%d' % VAL_BATCHSIZE] = np.float64(epoch(patches, VAL_BATCHSIZE))

            for sub in ('mixtures', 'instruments'):
                os.makedirs(os.path.join('split', sub))
                for base in split_names():
                    open(os.path.join('split', sub, base + '.wav'), 'wb').close()
                open(os.path.join('split', sub, 'notes.txt'), 'w').close()
            random.seed(SPLIT_SEED)
            train_list, val_list = ref_dataset.train_val_split('split', 'random', SPLIT_RATE, [])
            for key, lst in (('split_train', train_list), ('split_val', val_list)):
                out[key] = np.asarray([[os.path.basename(a), os.path.basename(b)] for a, b in lst])
        finally:
            os.chdir(cwd)
    print('patch losses', out['patch_losses'], 'total', out['total_b%d' % VAL_BATCHSIZE])
    make_golden.save_parts('ref_validation', out)


if __name__ == '__main__':
    run_validation()
