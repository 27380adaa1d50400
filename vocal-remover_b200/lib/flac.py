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
"""
import os

import numpy as np

BPS_CODES = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24}
MAX_BLOCK = 65535

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


def _name(src):
    return src if isinstance(src, (str, os.PathLike)) else '<%d bytes>' % len(src)


def _read(src):
    if isinstance(src, (bytes, bytearray, memoryview)):
        return bytes(src)
    with open(src, 'rb') as f:
        return f.read()


def _id3_size(head):
    """Bytes taken by an ID3v2 tag at the start of ``head`` (0 if there is none)."""
    if len(head) < 10 or head[:3] != b'ID3':
        return 0
    return 10 + ((head[6] & 0x7F) << 21 | (head[7] & 0x7F) << 14 | (head[8] & 0x7F) << 7 | (head[9] & 0x7F)) + \
        (10 if head[5] & 0x10 else 0)


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
    name = _name(src)
    data = _read(src)
    start, info = parse_metadata(data, name)
    end = audio_end(data, start)
    if not torch.cuda.is_available():
        raise RuntimeError('%s: FLAC decoding runs on the GPU and no CUDA device is visible' % name)
    dev = torch.device(device if device is not None else 'cuda:0')
    lib = _native.load_library()

    def check(rc, what):
        if rc != 0:
            raise _native.NativeError('%s failed: %s' % (what, lib.vr_last_error(None).decode()))

    with torch.cuda.device(dev):
        d_data = torch.frombuffer(bytearray(data[:end]), dtype=torch.uint8).to(dev) if end else \
            torch.zeros(1, dtype=torch.uint8, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        cap = 256 + end // 256      # a retry with the exact count covers streams of very short frames
        while True:
            cands = torch.empty((cap, 4), dtype=torch.int64, device=dev)
            check(lib.vr_flac_scan(None, _native.ptr(d_data), end, start, _native.ptr(cands), cap, _native.ptr(count),
                                   _native.stream_ptr()), 'vr_flac_scan')
            found = int(count.item())
            if found <= cap:
                break
            cap = found
        frames, total = build_chain(cands[:found].cpu().numpy(), start, end, info, name)
        out = torch.empty((info['channels'], total), dtype=torch.float32, device=dev)
        status = torch.empty(frames.shape[0], dtype=torch.int64, device=dev)
        d_frames = torch.from_numpy(frames).to(dev)
        check(lib.vr_flac_decode(None, _native.ptr(d_data), end, _native.ptr(d_frames), frames.shape[0],
                                 info['channels'], total, _native.ptr(out), _native.ptr(status), _native.stream_ptr()),
              'vr_flac_decode')
        st = status.cpu().numpy()
    bad = np.flatnonzero(st)
    if bad.size:
        k = int(bad[0])
        code, bit = int(st[k]) >> 40, int(st[k]) & ((1 << 40) - 1)
        raise ValueError('%s: frame %d (byte %d): %s (bit %d of the frame)'
                         % (name, k, int(frames[k, 0]), ERRORS.get(code, 'error %d' % code), bit))
    check_length(info, total, name)
    return out, info['rate'], info['bps']
