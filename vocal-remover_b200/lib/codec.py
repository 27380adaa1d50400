"""Host steps the GPU input decoders (lib/flac.py, lib/mp3.py, lib/aac.py) share: the source's name and bytes, the
size of an ID3v2 tag, the device a decode runs on, the sync scan with its retry, the per-frame status words and the
trim of the decoded samples.  Each format's own logic (metadata or boxes, frame chain, gapless or edit-list trim
range, error messages) stays in its module."""
import os

import numpy as np


def source(src):
    """(name for messages, bytes) of a file path or a bytes-like object."""
    name = src if isinstance(src, (str, os.PathLike)) else '<%d bytes>' % len(src)
    if isinstance(src, (bytes, bytearray, memoryview)):
        return name, bytes(src)
    with open(src, 'rb') as f:
        return name, f.read()


def id3v2_size(head):
    """Bytes taken by an ID3v2 tag at the start of ``head`` (0 if there is none)."""
    if len(head) < 10 or head[:3] != b'ID3':
        return 0
    return 10 + ((head[6] & 0x7F) << 21 | (head[7] & 0x7F) << 14 | (head[8] & 0x7F) << 7 | (head[9] & 0x7F)) + \
        (10 if head[5] & 0x10 else 0)


def cuda_device(name, what, device):
    """The torch device that decodes ``name`` (``device``, by default cuda:0); RuntimeError when no CUDA device is
    visible.  ``what``: the format, as the message names it."""
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError('%s: %s decoding runs on the GPU and no CUDA device is visible' % (name, what))
    return torch.device(device if device is not None else 'cuda:0')


def scan(lib, fn, d_data, a, b, width, cap):
    """The rows of ``width`` int64 that the sync scan ``fn`` (vr_flac_scan, vr_mp3_scan: ``a`` and ``b`` are their two
    byte bounds) appends for ``d_data``, as a device tensor in no particular order.  The scan runs with room for ``cap``
    rows and, when it found more, once more with room for the count it returned."""
    import torch
    from . import _native
    count = torch.zeros(1, dtype=torch.int32, device=d_data.device)
    while True:
        cands = torch.empty((cap, width), dtype=torch.int64, device=d_data.device)
        _native.check(lib, getattr(lib, fn)(None, _native.ptr(d_data), a, b, _native.ptr(cands), cap,
                                            _native.ptr(count), _native.stream_ptr()), fn)
        found = int(count.item())
        if found <= cap:
            return cands[:found]
        cap = found


def raise_first_bad(status, offsets, errors, name, unit, allowed=(), first=0, bit_note=''):
    """ValueError for the first status word (code << 40 | bit, one per frame or packet, csrc/bitstream.cuh) whose code
    is neither 0 nor in ``allowed``: '<name>: <unit> <first + k> (byte <offsets[k]>): <errors[code]> (bit
    <bit><bit_note>)'.  ``first`` numbers the words from a frame other than 0."""
    st = np.asarray(status, np.int64)
    codes = st >> 40
    keep = codes != 0
    for code in allowed:
        keep &= codes != code
    bad = np.flatnonzero(keep)
    if bad.size:
        k = int(bad[0])
        code = int(codes[k])
        raise ValueError('%s: %s %d (byte %d): %s (bit %d%s)' % (name, unit, first + k, int(offsets[k]),
                                                                 errors.get(code, 'error %d' % code),
                                                                 int(st[k]) & ((1 << 40) - 1), bit_note))


def trim(out, a, b):
    """Samples [a, b) of the decoded (channels, n) ``out``: ``out`` itself when that is all of it, else a contiguous
    copy."""
    return out if (a, b) == (0, out.shape[1]) else out[:, a:b].contiguous()
