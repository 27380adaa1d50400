"""CPU oracle and golden recipe of the dataset tool's vocal JPGs (lib/dataset.py run as a script).  TEST INFRASTRUCTURE.

``vocal_image`` restates the image the reference's lib/dataset.py:280-287 writes for one (mixture, instruments) pair
in float32 numpy; ``vocal_cases`` regenerates the seeded spectrogram pairs of the fixture
``tests/golden/ref_vocal_image.partN.npz``, which ``run_vocal_image`` writes by running the UNMODIFIED reference's
lib/dataset.py as ``__main__``.  The pairs are handed to it as the reference's ``cache_or_load`` caches next to empty
.wav placeholders, so that no audio is decoded, and its ``utils.imwrite`` is replaced by a function that keeps the
image instead of encoding it.  Seeded random spectrograms rather than an STFT keep the inputs bit-identical on every
machine.  Regenerate with ``VR_REFERENCE_ROOT=<checkout> python -m oracle.dataset_image_oracle`` from the repo root;
it writes only ref_vocal_image.*.
"""
import numpy as np

from . import image_oracle

SR, HOP, N_FFT = 44100, 1024, 2048   # the values the reference's script passes to cache_or_load
BINS = N_FFT // 2 + 1
FRAMES = (100, 1)


def vocal_image(X, y):
    """complex (2, bins, T) mixture / instruments -> uint8 (bins, T, 3): spectrogram_to_image(v_mag) with
    v_mag = |X| - |y| kept where v_mag > |y|.  A constant v_mag gives zeros, the rule the GPU kernels follow."""
    X_mag = np.abs(X)
    y_mag = np.abs(y)
    v_mag = X_mag - y_mag
    v_mag *= v_mag > y_mag
    # for a real array |v|^2 is v ** 2 bit for bit, so the magnitude-mode restatement applies as it stands
    return image_oracle.spectrogram_to_image(v_mag)


def vocal_cases():
    """[(name, X, y)] complex64 (2, BINS, T) for T in FRAMES.  |X| is log-uniform over 1e-4 .. 300; |y| is |X| times a
    factor uniform in [0, 1.5] with its own phase, so v > |y|, 0 <= v < |y| and v < 0 all occur.  A few elements are
    exact zeros of X, of y or of both, and about 2% are exact ties y = X / 2, where v == |y| and the strict comparison
    drops v."""
    rng = np.random.default_rng(2026)
    cases = []
    for k, T in enumerate(FRAMES):
        shape = (2, BINS, T)
        mag = 10.0 ** rng.uniform(-4.0, np.log10(300.0), size=shape)
        X = (mag * np.exp(1j * rng.uniform(-np.pi, np.pi, size=shape))).astype(np.complex64)
        factor = rng.uniform(0.0, 1.5, size=shape)
        y = (np.abs(X) * factor * np.exp(1j * rng.uniform(-np.pi, np.pi, size=shape))).astype(np.complex64)
        idx = rng.permutation(X.size)
        n_tie = max(1, X.size // 50)
        ties, zx, zy, zxy = idx[:n_tie], idx[n_tie:n_tie + 8], idx[n_tie + 8:n_tie + 16], idx[n_tie + 16:n_tie + 20]
        y.flat[ties] = X.flat[ties] / np.complex64(2)
        X.flat[zx] = 0
        y.flat[zy] = 0
        X.flat[zxy] = 0
        y.flat[zxy] = 0
        cases.append(('pair%d' % k, X, y))
    return cases


def _run_reference_script(path, argv, modules):
    """runpy of the reference script ``path`` as ``__main__`` with ``sys.argv = argv``.  ``modules`` (name -> module)
    stand in for the reference's own imports while it runs; the previous modules of those names come back after."""
    import runpy
    import sys
    saved_modules = {k: sys.modules.get(k) for k in modules}
    saved_argv = sys.argv
    try:
        sys.modules.update(modules)
        sys.argv = list(argv)
        runpy.run_path(path, run_name='__main__')
    finally:
        sys.argv = saved_argv
        for k, mod in saved_modules.items():
            if mod is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = mod


def run_vocal_image():
    """Reference vocal JPG images of vocal_cases(), captured from its lib/dataset.py run as a script over a dataset
    of cached pairs in a temporary directory."""
    import os
    import sys
    import tempfile
    import types
    from oracle import librosa_shim, make_golden
    librosa_shim.import_reference()
    # the reference script imports ``from lib import spec_utils`` and ``import utils`` (its lib/utils.py)
    ref_lib = {k[len('_ref_'):]: m for k, m in sys.modules.items() if k == '_ref_lib' or k.startswith('_ref_lib.')}
    captured = {}

    def imwrite(filename, img, params=None):
        captured[filename] = np.array(img, copy=True)
        return True
    utils = types.ModuleType('utils')
    utils.imwrite = imwrite

    out = {}
    cache = 'sr{}_hl{}_nf{}'.format(SR, HOP, N_FFT)
    with tempfile.TemporaryDirectory() as tmp:
        for name, X, y in vocal_cases():
            out[name + '_X_sum'] = make_golden.checksum(X)
            out[name + '_y_sum'] = make_golden.checksum(y)
            for sub, spec in (('mixtures', X), ('instruments', y)):
                os.makedirs(os.path.join(tmp, sub, cache), exist_ok=True)
                open(os.path.join(tmp, sub, name + '.wav'), 'wb').close()   # never decoded: the cache hits
                np.save(os.path.join(tmp, sub, cache, name + '.npy'), spec.transpose(2, 0, 1))
        outdir = os.path.join(tmp, 'out')
        _run_reference_script(os.path.join(librosa_shim.REFERENCE_ROOT, 'lib', 'dataset.py'),
                              ['dataset.py', os.path.join(tmp, 'mixtures'), os.path.join(tmp, 'instruments'), outdir],
                              dict(ref_lib, utils=utils))
        assert os.path.isdir(outdir)
        written = sorted(captured)
        assert written == ['{}/{}_Vocal.jpg'.format(outdir, name) for name, _, _ in vocal_cases()], written
        for name, _, _ in vocal_cases():
            out[name + '_vocal'] = captured['{}/{}_Vocal.jpg'.format(outdir, name)]
    make_golden.save_parts('ref_vocal_image', out)


if __name__ == '__main__':
    run_vocal_image()
