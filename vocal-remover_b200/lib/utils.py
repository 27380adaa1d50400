"""Image file helpers of the --output_image JPGs (reference lib/utils.py).

cv2 is imported when a function is called, so that importing ``lib`` never needs it; a missing cv2 raises
ImportError.  Like the reference, both functions report every other failure by their return value and never raise.
"""
import os

import numpy as np

JPEG_MAX_WIDTH = 65500   # widest image the JPEG encoder accepts; one pixel per STFT frame


def imread(filename, flags=None, dtype=np.uint8):
    """Decodes an image file (cv2.IMREAD_COLOR by default); None if it cannot be read or decoded."""
    import cv2
    try:
        return cv2.imdecode(np.fromfile(filename, dtype), cv2.IMREAD_COLOR if flags is None else flags)
    except Exception as e:
        print(e)
        return None


def imwrite(filename, img, params=None):
    """Encodes ``img`` in the format of ``filename``'s extension and writes it.  Returns True on success; False, with
    nothing written, if the encoder refuses the image (a JPEG is at most 65500 pixels wide) or the file cannot be
    opened."""
    import cv2
    try:
        ok, buf = cv2.imencode(os.path.splitext(filename)[1], img, params if params is not None else [])
        if not ok:
            return False
        with open(filename, 'wb') as f:
            buf.tofile(f)
        return True
    except Exception as e:
        print(e)
        return False
