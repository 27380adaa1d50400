"""FLAC input (RFC 9639) decoded on the GPU: ``decode(path_or_bytes, device) -> (CUDA float32 (channels, n), rate, bps)``.

The host reads the metadata (an ID3v2 prefix is skipped, STREAMINFO is read, every other block is skipped by its
length), copies the bytes to the device once, and runs two kernels of csrc/flac.cu with a host step between them:

1. ``vr_flac_scan`` lists every frame-header candidate after the metadata (sync, header, CRC-8).
2. ``build_chain`` (numpy, a few thousand rows) starts at the end of the metadata and repeatedly takes the next
   candidate whose coded number is the expected one (the frame index for a fixed-block-size stream, the first sample
   for a variable one).  That gives every frame its byte span and first sample.  A sync pattern inside frame data
   with a valid CRC-8 carries some other number and is passed over; the decode's end check would catch one that
   does not.
3. ``vr_flac_decode`` decodes one frame per warp straight into the output as ``float32(x) / 2^(bps-1)`` (the scaling
   of soundfile and of the WAV reader) and leaves a status word per frame.

Malformed input raises ``ValueError`` naming the file, the frame and its byte offset.  The MD5 in STREAMINFO is not
checked on this path (libsndfile does not check it either).

FLAC output, ``encode(x, rate, path=None, md5=True, bits=16) -> bytes``: 16 or 24 bits per sample, one or two channels,
fixed block size ``BLOCK`` (the last block shorter), inside the streamable subset.  Two kernels of csrc/flac_encode.cu
with a host step between them:

1. ``vr_flac_encode_analyse`` quantises each frame to ``bits``-wide integers and chooses every subframe's coding and
   the channel assignment by exact size; it leaves the samples (int16, or int32 for 24 bits) and a plan with each
   frame's size in bytes.
2. The host scans the frame sizes into byte offsets (numpy).
3. ``vr_flac_encode_pack`` writes every frame to its span, CRCs included.

The host puts ``fLaC`` and STREAMINFO in front; STREAMINFO's MD5 is computed with hashlib from the samples as
interleaved little-endian ``bits / 8``-byte integers: the int16 samples as they are, the 24-bit ones packed to 3 bytes
on the device by ``vr_pcm_pack`` (``pcm_bytes``), which is also what a 24-bit WAV file holds (lib/audio_io.write).

The integers are ``clip(rint(x * (2^(bits-1) - 1)))`` with the product in fp32 and NaN -> 0, for every writer.
"""
import hashlib

import numpy as np

from . import codec
from .codec import id3v2_size as _id3_size   # the name tests/test_mp3.py takes it by

BPS_CODES = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24}
MAX_BLOCK = 65535
BLOCK = 4096                 # FLAC_ENCODE_BLOCK (include/vr_b200.h)
PLAN_INTS = 192              # FLAC_ENCODE_PLAN_INTS
BITS = {16: 'int16', 24: 'int32'}   # output sample widths and the dtype of Frames.pcm for each
RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10,
              96000: 11}

# status codes of flac_decode_kernel (csrc/flac.cu)
ERRORS = {
    1: 'the frame data ends before its subframes do',
    2: 'a padding bit is not zero',
    3: 'reserved subframe type',
    4: 'predictor order larger than the block',
    5: 'LPC precision code 1111',
    6: 'negative LPC shift',
    7: 'reserved residual coding method',
    8: 'partition order does not fit the block size and predictor order',
    9: 'a Rice-coded residual does not fit 32 bits',
    10: 'a predicted sample is outside the subframe\'s bit depth',
    11: 'the subframes do not end 2 bytes before the next frame header (or the end of the stream): '
        'corrupted data or a missing or corrupted frame header after it',
    12: 'CRC-16 mismatch',
    13: 'frame shape the stream does not have',
    14: 'wasted bits leave no sample bits',
}


def sniff(path):
    """True if the file holds a FLAC stream (by content: ``fLaC``, optionally after an ID3v2 tag)."""
    try:
        with open(path, 'rb') as f:
            head = f.read(10)
            skip = _id3_size(head)
            if skip:
                f.seek(skip)
                head = f.read(4)
    except OSError:
        return False
    return head[:4] == b'fLaC'


def parse_metadata(data, name='<bytes>'):
    """(byte offset of the first frame, STREAMINFO dict with rate, channels, bps, total, md5)."""
    p = _id3_size(data)
    if data[p:p + 4] != b'fLaC':
        raise ValueError('%s: not a FLAC stream (no fLaC marker)' % name)
    p += 4
    info = None
    while True:
        if p + 4 > len(data):
            raise ValueError('%s: metadata runs past the end of the file' % name)
        hdr, ln = data[p], int.from_bytes(data[p + 1:p + 4], 'big')
        if p + 4 + ln > len(data):
            raise ValueError('%s: metadata block at byte %d runs past the end of the file' % (name, p))
        if info is None:
            if hdr & 0x7F != 0 or ln != 34:
                raise ValueError('%s: the first metadata block is not a 34-byte STREAMINFO' % name)
            b = data[p + 4:p + 38]
            packed = int.from_bytes(b[10:18], 'big')
            info = dict(min_block=int.from_bytes(b[0:2], 'big'), max_block=int.from_bytes(b[2:4], 'big'),
                        rate=packed >> 44, channels=((packed >> 41) & 7) + 1, bps=((packed >> 36) & 31) + 1,
                        total=packed & ((1 << 36) - 1), md5=bytes(b[18:34]))
        elif hdr & 0x7F == 127:
            raise ValueError('%s: invalid metadata block type 127 at byte %d' % (name, p))
        p += 4 + ln
        if hdr & 0x80:
            break
    if info['bps'] == 32:
        raise ValueError('%s: 32-bit FLAC is not supported (4 to 24 bits per sample)' % name)
    if info['bps'] < 4:
        raise ValueError('%s: STREAMINFO gives %d bits per sample (4 to 24 are supported)' % (name, info['bps']))
    if info['rate'] == 0:
        raise ValueError('%s: STREAMINFO gives a sample rate of 0' % name)
    return p, info


def build_chain(cands, audio_start, audio_end, info, name='<bytes>'):
    """Frames of the stream from the scan's candidate rows (any order; layout in include/vr_b200.h, vr_flac_scan).

    Returns (frames int64 (F, 4) as vr_flac_decode takes them, total samples).  Raises ValueError on reserved codes
    and on headers that disagree with STREAMINFO.  The length is checked after the decode (check_length), so that a
    truncated stream is reported by the frame it cuts."""
    cands = np.asarray(cands, np.int64).reshape(-1, 4)
    cands = cands[np.argsort(cands[:, 0], kind='stable')]
    cands = cands[(cands[:, 0] >= audio_start) & (cands[:, 0] < audio_end)]
    offs, nums = cands[:, 0].tolist(), cands[:, 1].tolist()
    strat = ((cands[:, 2] >> 22) & 1).tolist()
    chosen = []
    expected, samples, variable = 0, 0, None
    j = 0
    while True:
        while j < len(offs) and not (nums[j] == expected and (variable is None or strat[j] == variable)):
            j += 1
        if j == len(offs):
            break
        row = cands[j]
        k, off = len(chosen), int(row[0])
        bs, hlen = int(row[2] & 0x1FFFF), int((row[2] >> 17) & 0x1F)
        b2, b3 = int(row[3] & 0xFF), int((row[3] >> 8) & 0xFF)
        bs_code, rate_code, ch_code, bps_code = b2 >> 4, b2 & 15, b3 >> 4, (b3 >> 1) & 7
        where = '%s: frame %d (byte %d)' % (name, k, off)
        if bs_code == 0:
            raise ValueError('%s: reserved block-size code 0000' % where)
        if rate_code == 15:
            raise ValueError('%s: invalid sample-rate code 1111' % where)
        if ch_code > 10:
            raise ValueError('%s: reserved channel assignment %d' % (where, ch_code))
        if bps_code == 3:
            raise ValueError('%s: reserved sample-size code 011' % where)
        if bps_code == 7:
            raise ValueError('%s: 32-bit FLAC is not supported (4 to 24 bits per sample)' % where)
        if b3 & 1:
            raise ValueError('%s: reserved header bit set' % where)
        if bs > MAX_BLOCK:
            raise ValueError('%s: block size %d exceeds %d' % (where, bs, MAX_BLOCK))
        nch = ch_code + 1 if ch_code < 8 else 2
        bps = BPS_CODES.get(bps_code, info['bps'])
        if nch != info['channels'] or bps != info['bps']:
            raise ValueError('%s: %d channels of %d bits, STREAMINFO gives %d of %d' % (where, nch, bps, info['channels'],
                                                                                       info['bps']))
        chosen.append((off, samples, bs | (hlen << 17) | (ch_code << 24) | (bps << 28)))
        if variable is None:
            variable = strat[j]
        samples += bs
        expected = samples if variable else len(chosen)
        j += 1
    if not chosen:
        raise ValueError('%s: no audio frame follows the metadata (byte %d)' % (name, audio_start))
    frames = np.zeros((len(chosen), 4), np.int64)
    frames[:, 0] = [c[0] for c in chosen]
    frames[:-1, 1] = frames[1:, 0]
    frames[-1, 1] = audio_end
    frames[:, 2] = [c[1] for c in chosen]
    frames[:, 3] = [c[2] for c in chosen]
    return frames, samples


def check_length(info, samples, name='<bytes>'):
    """The stream's length is the sum of its block sizes; a nonzero STREAMINFO total must agree."""
    if info['total'] and info['total'] != samples:
        raise ValueError('%s: STREAMINFO gives %d samples, the frames hold %d' % (name, info['total'], samples))


def audio_end(data, start):
    """End of the frame data: the file's end, less an ID3v1 tag (128 bytes starting ``TAG``) after the frames."""
    n = len(data)
    if n - 128 >= start and data[n - 128:n - 125] == b'TAG':
        return n - 128
    return n


def decode(src, device=None):
    """FLAC file path or bytes -> (CUDA float32 tensor (channels, n), sample rate, bits per sample)."""
    import torch
    from . import _native
    name, data = codec.source(src)
    start, info = parse_metadata(data, name)
    end = audio_end(data, start)
    dev = codec.cuda_device(name, 'FLAC', device)
    lib = _native.load_library()
    with torch.cuda.device(dev):
        d_data = torch.frombuffer(bytearray(data[:end]), dtype=torch.uint8).to(dev) if end else \
            torch.zeros(1, dtype=torch.uint8, device=dev)
        # a retry with the exact count covers streams of very short frames
        cands = codec.scan(lib, 'vr_flac_scan', d_data, end, start, 4, 256 + end // 256)
        frames, total = build_chain(cands.cpu().numpy(), start, end, info, name)
        out = torch.empty((info['channels'], total), dtype=torch.float32, device=dev)
        status = torch.empty(frames.shape[0], dtype=torch.int64, device=dev)
        d_frames = torch.from_numpy(frames).to(dev)
        _native.check(lib, lib.vr_flac_decode(None, _native.ptr(d_data), end, _native.ptr(d_frames), frames.shape[0],
                                              info['channels'], total, _native.ptr(out), _native.ptr(status),
                                              _native.stream_ptr()), 'vr_flac_decode')
        st = status.cpu().numpy()
    codec.raise_first_bad(st, frames[:, 0], ERRORS, name, 'frame', bit_note=' of the frame')
    check_length(info, total, name)
    return out, info['rate'], info['bps']


# ------------------------------------------------------------------------------------------------------------- encoder


def rate_code(rate):
    """(frame-header sample-rate code, value written after the header) of ``rate``; codes 12-14 for rates that are not
    in the table, as the streamable subset requires."""
    rate = int(rate)
    if rate in RATE_CODES:
        return RATE_CODES[rate], 0
    if rate % 1000 == 0 and rate // 1000 <= 255:
        return 12, rate // 1000
    if 0 < rate <= 65535:
        return 13, rate
    if rate % 10 == 0 and rate // 10 <= 65535:
        return 14, rate // 10
    raise ValueError('FLAC output: a sample rate of %d Hz cannot be coded in a frame header' % rate)


def _check_bits(bits):
    if bits not in BITS:
        raise ValueError('output samples are 16 or 24 bits wide, not %r' % (bits,))


def stream_header(channels, total, rate, frame_sizes, md5, block=BLOCK, bits=16):
    """``fLaC`` and the one STREAMINFO block of a fixed-block-size stream: min / max block size (the last block
    excluded, unless it is the only one), min / max frame size, rate, channels, bits per sample, total samples, MD5."""
    sizes = [block] * (len(frame_sizes) - 1) + [total - block * (len(frame_sizes) - 1)]
    bmin = max(16, min(sizes[:-1] or sizes))
    bmax = min(65535, max(16, max(sizes)))
    fmin, fmax = int(min(frame_sizes)), int(max(frame_sizes))
    si = bmin.to_bytes(2, 'big') + bmax.to_bytes(2, 'big') + fmin.to_bytes(3, 'big') + fmax.to_bytes(3, 'big')
    si += ((int(rate) << 44) | ((channels - 1) << 41) | ((bits - 1) << 36) | int(total)).to_bytes(8, 'big') + bytes(md5)
    return b'fLaC' + bytes([0x80]) + len(si).to_bytes(3, 'big') + si


class Frames(object):
    """The frames of one encode: ``body`` (bytes), ``sizes`` (int64 per frame), ``pcm`` (the samples the frames code,
    (n, channels) on the device: int16 for ``bits`` 16, int32 holding the 24-bit integers for 24), ``channels``,
    ``total``, ``rate`` and ``bits``."""

    def __init__(self, body, sizes, pcm, channels, total, rate, bits=16):
        self.body, self.sizes, self.pcm = body, sizes, pcm
        self.channels, self.total, self.rate, self.bits = channels, total, rate, bits


def _on_device(x, device=None):
    """(channels, n) float samples, a CUDA tensor (kept where it is) or an array -> contiguous float32 CUDA tensor."""
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError('FLAC encoding runs on the GPU and no CUDA device is visible')
    if torch.is_tensor(x) and x.is_cuda:
        dev = x.device
    else:
        dev = torch.device(device if device is not None else 'cuda:0')
    if x.ndim != 2 or x.shape[0] not in (1, 2) or x.shape[1] < 1:
        raise ValueError('FLAC output takes (channels, n) samples with one or two channels and n >= 1, not %s'
                         % (tuple(x.shape),))
    xd = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x, np.float32))
    return xd.to(dev, torch.float32).contiguous()


def pcm_bytes(x, bits, device=None):
    """float (channels, n) -> numpy uint8 array: the samples quantised and interleaved as little-endian ``bits / 8``-byte
    integers on the device (``vr_pcm_pack``); only those bytes are copied back."""
    import torch
    from . import _native
    _check_bits(bits)
    xd = _on_device(x, device)
    lib = _native.load_library()
    with torch.cuda.device(xd.device):
        out = torch.empty(xd.numel() * (bits // 8), dtype=torch.uint8, device=xd.device)
        _native.check(lib, lib.vr_pcm_pack(None, _native.ptr(xd), int(xd.shape[0]), int(xd.shape[1]), bits,
                                           _native.ptr(out), _native.stream_ptr()), 'vr_pcm_pack')
        return out.cpu().numpy()


def encode_frames(x, rate, device=None, bits=16):
    """float (channels, n) -> Frames.  ``x``: a CUDA float32 tensor (stays on its device) or an array."""
    import torch
    from . import _native
    _check_bits(bits)
    xd = _on_device(x, device)
    dev = xd.device
    code, value = rate_code(rate)
    C, n = int(xd.shape[0]), int(xd.shape[1])
    if n >= 1 << 36:
        raise ValueError('FLAC output: %d samples per channel exceed STREAMINFO\'s 36 bits' % n)
    lib = _native.load_library()
    with torch.cuda.device(dev):
        F = (n + BLOCK - 1) // BLOCK
        pcm = torch.empty((n, C), dtype=getattr(torch, BITS[bits]), device=dev)
        plan = torch.empty((F, PLAN_INTS), dtype=torch.int32, device=dev)
        stream = _native.stream_ptr()
        _native.check(lib, lib.vr_flac_encode_analyse(None, _native.ptr(xd), C, n, code, bits, _native.ptr(pcm),
                                                      _native.ptr(plan), stream), 'vr_flac_encode_analyse')
        sizes = plan[:, 0].cpu().numpy().astype(np.int64)
        offsets = np.zeros(F, np.int64)
        np.cumsum(sizes[:-1], out=offsets[1:])
        out = torch.empty(int(sizes.sum()), dtype=torch.uint8, device=dev)
        status = torch.empty(F, dtype=torch.int32, device=dev)
        d_off = torch.from_numpy(offsets).to(dev)
        _native.check(lib, lib.vr_flac_encode_pack(None, _native.ptr(pcm), C, n, bits, _native.ptr(plan),
                                                   _native.ptr(d_off), code, value, _native.ptr(out),
                                                   _native.ptr(status), stream), 'vr_flac_encode_pack')
        body = out.cpu().numpy().tobytes()
        st = status.cpu().numpy()
    bad = np.flatnonzero(st)
    if bad.size:
        raise RuntimeError('FLAC encode: frame %d did not fill the size its plan gave (status %d)'
                           % (int(bad[0]), int(st[bad[0]])))
    return Frames(body, sizes, pcm, C, n, int(rate), bits)


def encode(x, rate, path=None, md5=True, bits=16):
    """float (channels, n) -> the whole FLAC stream (bytes): ``fLaC``, STREAMINFO, the frames; also written to ``path``
    when one is given.  ``x`` is a CUDA float32 tensor (it stays on the device; only the compressed bytes and the
    samples' bytes for the MD5 are copied back) or an array; samples are quantised as clip(rint(x * 32767)), or
    clip(rint(x * 8388607)) for ``bits=24``, NaN -> 0.
    ``md5=False`` leaves STREAMINFO's MD5 zero (unknown), which skips the copy of the samples and the hash."""
    _check_bits(bits)
    x = _on_device(x)
    fr = encode_frames(x, rate, bits=bits)
    if not md5:
        digest = bytes(16)
    elif bits == 16:
        digest = hashlib.md5(fr.pcm.cpu().numpy().astype('<i2', copy=False).tobytes()).digest()
    else:
        digest = hashlib.md5(pcm_bytes(x, bits)).digest()
    data = stream_header(fr.channels, fr.total, fr.rate, fr.sizes, digest, bits=bits) + fr.body
    if path is not None:
        with open(path, 'wb') as f:
            f.write(data)
    return data
