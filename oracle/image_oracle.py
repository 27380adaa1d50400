"""CPU oracle and golden recipe of the --output_image spectrogram images.  TEST INFRASTRUCTURE.

``spectrogram_to_image`` restates the reference's magnitude-mode ``spec_utils.spectrogram_to_image``
(lib/spec_utils.py:34-57) in float32 numpy; ``image_cases`` regenerates the seeded inputs of the fixture
``tests/golden/ref_image.partN.npz``, which ``run_image`` writes from the UNMODIFIED reference's
``Separator._postprocess`` (inference.py:26-40) and ``spectrogram_to_image``.  Seeded random spectrograms rather
than an STFT keep the inputs bit-identical on every machine.  Regenerate with
``VR_REFERENCE_ROOT=<checkout> python -m oracle.image_oracle`` from the repo root; it writes only ref_image.*.
"""
import numpy as np


def spectrogram_to_image(spec):
    """complex (2, bins, T) -> uint8 (bins, T, 3) = {max(L, R), L, R}.  A constant input (where the reference's uint8
    cast sees 0 * inf = NaN) gives zeros, the rule the GPU kernels follow."""
    level = np.log10(np.square(np.abs(spec)) + np.float32(1e-8))
    level -= level.min()
    top = level.max()
    if top == 0:
        img = np.zeros(level.shape, np.uint8)
    else:
        level *= np.float32(255) / top
        img = level.astype(np.uint8)
    lr = np.moveaxis(img, 0, -1)
    return np.concatenate([lr.max(axis=-1, keepdims=True), lr], axis=-1)


def image_cases():
    """[(name, X complex64 (2, bins, T), mask float32 (2, bins, T) or None)]: magnitudes log-uniform over 1e-5 .. 300
    with a few exact zeros, masks log-uniform down to 1e-6 with exact 0 and 1."""
    rng = np.random.default_rng(2024)

    def spec(bins, T):
        mag = 10.0 ** rng.uniform(-5.0, np.log10(300.0), size=(2, bins, T))
        X = (mag * np.exp(1j * rng.uniform(-np.pi, np.pi, size=(2, bins, T)))).astype(np.complex64)
        X.flat[rng.choice(X.size, min(8, X.size), replace=False)] = 0
        return X

    def mask(shape):
        m = (10.0 ** rng.uniform(-6.0, 0.0, size=shape)).astype(np.float32)
        k = rng.choice(m.size, min(40, m.size), replace=False)
        m.flat[k[:len(k) // 2]] = 0
        m.flat[k[len(k) // 2:]] = 1
        return m

    masked = spec(1025, 256)
    small = spec(257, 300)
    single = spec(1025, 1)
    return [('masked', masked, mask(masked.shape)), ('small', small, None), ('single', single, mask(single.shape))]


def run_image():
    """Reference images of image_cases(): 'masked' / 'single' -> <name>_inst / <name>_voc of y_spec / v_spec of
    Separator._postprocess (postprocess=False), 'small' -> <name>_X of the spectrogram itself."""
    import types
    from oracle import librosa_shim, make_golden
    ref_inference, _, ref_spec_utils, _ = librosa_shim.import_reference()
    sp = ref_inference.Separator(types.SimpleNamespace(offset=64), None, 1, 256, False)
    out = {}
    for name, X, m in image_cases():
        out[name + '_X_sum'] = make_golden.checksum(X)
        if m is None:
            out[name + '_X'] = ref_spec_utils.spectrogram_to_image(X)
            continue
        out[name + '_mask_sum'] = make_golden.checksum(m)
        y, v = sp._postprocess(X, m)
        out[name + '_inst'] = ref_spec_utils.spectrogram_to_image(y)
        out[name + '_voc'] = ref_spec_utils.spectrogram_to_image(v)
    make_golden.save_parts('ref_image', out)


if __name__ == '__main__':
    run_image()
