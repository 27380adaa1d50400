"""The oracle masks of ``evaluate.py --oracle`` (DESIGN.md §12) in float64 numpy.

Restates vr_oracle_mask operation by operation: the true vocals V = X - Y are a float32 subtraction per component, the
powers Re² + Im², the square roots and the quotients are float64 with each operation rounded (numpy neither fuses nor
reorders them), and the result is rounded once to float32.  So the GPU's mask equals ``mask`` bit for bit.
"""
import numpy as np

KINDS = ('iam', 'ibm', 'irm1', 'irm2')


def _power(re, im):
    re, im = np.asarray(re, np.float64), np.asarray(im, np.float64)
    return re * re + im * im


def mask(X, Y, kind):
    """float32 mask (the instruments'; the vocals get 1 - mask) of the mixture X and true instruments Y, both complex64
    arrays of one shape."""
    X, Y = np.asarray(X, np.complex64), np.asarray(Y, np.complex64)
    pY = _power(Y.real, Y.imag)
    with np.errstate(divide='ignore', invalid='ignore'):
        if kind == 'iam':
            pX = _power(X.real, X.imag)
            m = np.where(pY >= pX, 1.0, np.sqrt(pY) / np.sqrt(pX))
        else:
            pV = _power(np.subtract(X.real, Y.real, dtype=np.float32), np.subtract(X.imag, Y.imag, dtype=np.float32))
            if kind == 'ibm':
                m = np.where(pY >= pV, 1.0, 0.0)
            elif kind == 'irm1':
                a = np.sqrt(pY)
                s = a + np.sqrt(pV)
                m = np.where(s == 0.0, 0.5, a / s)
            elif kind == 'irm2':
                s = pY + pV
                m = np.where(s == 0.0, 0.5, pY / s)
            else:
                raise ValueError('unknown oracle mask %r' % (kind,))
    return m.astype(np.float32)
