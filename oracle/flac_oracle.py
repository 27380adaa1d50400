"""FLAC (RFC 9639) test infrastructure: an encoder that writes valid streams from integer samples, a coverage schedule
that makes a handful of short streams exercise every coding choice the decoder has to handle, and a straightforward
decoder restating the RFC.  CPU only (numpy / pure Python); the product (lib/flac.py, csrc/flac.cu) never imports it.

The points where a shared misreading would survive a round trip are written out from the RFC, not from the product:
LPC ``s[i] = r[i] + ((sum_j c[j] * s[i-1-j]) >> shift)`` with the first coefficient on the newest sample and an
arithmetic shift; the side channel has one more bit than the frame; wasted bits are removed before coding and shifted
back after decoding; mid/side ``m = (m << 1) | (s & 1); L = (m + s) >> 1; R = (m - s) >> 1``; Rice
``u = (q << k) | low, v = (u >> 1) ^ -(u & 1)``; the first partition holds ``(blocksize >> order) - predictor_order``
samples.
"""
import hashlib
import math
import struct

import numpy as np

# ---------------------------------------------------------------------------------------------------------------- CRCs


def _crc_table(poly, width):
    top, mask = 1 << (width - 1), (1 << width) - 1
    table = []
    for b in range(256):
        c = b << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) if c & top else (c << 1)
        table.append(c & mask)
    return table


CRC8_TABLE = _crc_table(0x07, 8)
CRC16_TABLE = _crc_table(0x8005, 16)


def crc8(data):
    """CRC-8 of the frame header: poly x^8 + x^2 + x + 1, init 0, not reflected."""
    c = 0
    for b in bytes(data):
        c = CRC8_TABLE[c ^ b]
    return c


def crc16(data):
    """CRC-16 of the frame: poly x^16 + x^15 + x^2 + 1 (0x8005), init 0, not reflected (CRC-16/UMTS)."""
    c = 0
    for b in bytes(data):
        c = ((c << 8) & 0xFFFF) ^ CRC16_TABLE[(c >> 8) ^ b]
    return c


_CRC16_T16 = None


def crc16_many(chunks):
    """crc16 of each bytes object in ``chunks``, vectorised across them.  With init 0, leading zero bytes leave a CRC
    unchanged, so every chunk is left-padded to a common even length and all are advanced 16 bits per step."""
    global _CRC16_T16
    if _CRC16_T16 is None:
        t8 = np.asarray(CRC16_TABLE, np.uint32)
        w = np.arange(65536, dtype=np.uint32)
        c = t8[w >> 8]                                  # register 0, high byte in
        c = ((c << 8) & 0xFFFF) ^ t8[(c >> 8) ^ (w & 0xFF)]
        _CRC16_T16 = c.astype(np.uint32)
    n = max(len(c) for c in chunks)
    n += n & 1
    buf = np.zeros((len(chunks), n), np.uint8)
    for i, ch in enumerate(chunks):
        if len(ch):
            buf[i, n - len(ch):] = np.frombuffer(bytes(ch), np.uint8)
    words = (buf[:, 0::2].astype(np.uint32) << 8) | buf[:, 1::2]
    crc = np.zeros(len(chunks), np.uint32)
    for j in range(words.shape[1]):
        crc = _CRC16_T16[crc ^ words[:, j]]
    return [int(v) for v in crc]


# ------------------------------------------------------------------------------------------------------------ bit I/O


class BitWriter(object):
    """MSB-first bit fields; scalars and numpy arrays of fields, packed at once by ``tobytes`` (zero-padded to a byte)."""

    def __init__(self):
        self.vals, self.lens = [], []

    def put(self, value, nbits):
        if nbits:
            self.vals.append(np.array([int(value) & ((1 << nbits) - 1)], np.uint64))
            self.lens.append(np.array([nbits], np.int64))

    def put_signed_array(self, values, nbits):
        values = np.asarray(values, np.int64)
        if nbits and values.size:
            self.vals.append((values & ((1 << nbits) - 1)).astype(np.uint64))
            self.lens.append(np.full(values.size, nbits, np.int64))

    def put_fields(self, vals, lens):
        """Fields of any length; bits above bit 63 of a field are zeros (long unary prefixes)."""
        if len(vals):
            self.vals.append(np.asarray(vals, np.uint64))
            self.lens.append(np.asarray(lens, np.int64))

    def tobytes(self):
        if not self.vals:
            return b''
        vals, lens = np.concatenate(self.vals), np.concatenate(self.lens)
        lens_nz = lens > 0
        vals, lens = vals[lens_nz], lens[lens_nz]
        total = int(lens.sum())
        starts = np.cumsum(lens) - lens
        idx = np.repeat(np.arange(lens.size), lens)
        shift = lens[idx] - 1 - (np.arange(total) - starts[idx])
        bits = ((vals[idx] >> np.minimum(shift, 63).astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        bits[shift > 63] = 0
        return np.packbits(bits).tobytes()


class BitReader(object):
    """MSB-first reader over a byte string, as a '0'/'1' text so that unary runs are a str.find."""

    def __init__(self, data, pos_bits=0):
        self.bits = (np.unpackbits(np.frombuffer(bytes(data), np.uint8)) + 48).tobytes().decode('ascii')
        self.pos = pos_bits

    def read(self, n):
        if n == 0:
            return 0
        if self.pos + n > len(self.bits):
            raise ValueError('read past the end of the stream')
        v = int(self.bits[self.pos:self.pos + n], 2)
        self.pos += n
        return v

    def read_signed(self, n):
        v = self.read(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def unary(self):
        j = self.bits.find('1', self.pos)
        if j < 0:
            raise ValueError('unterminated unary code')
        q = j - self.pos
        self.pos = j + 1
        return q

    def align(self):
        self.pos = (self.pos + 7) & ~7


# ------------------------------------------------------------------------------------------------------- header codes

RATE_CODES = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000,
              11: 96000}
BPS_CODES = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}
CH_INDEPENDENT, CH_LEFT_SIDE, CH_SIDE_RIGHT, CH_MID_SIDE = 'independent', 8, 9, 10


def block_size_of_code(code, extra=None):
    if code == 1:
        return 192
    if 2 <= code <= 5:
        return 576 << (code - 2)
    if code in (6, 7):
        return extra + 1
    if code >= 8:
        return 256 << (code - 8)
    return None


def utf8_number(v):
    """The UTF-8-like coding of the frame / sample number (up to 36 bits, 1-7 bytes)."""
    if v < 0x80:
        return bytes([v])
    for n, lead in ((2, 0xC0), (3, 0xE0), (4, 0xF0), (5, 0xF8), (6, 0xFC), (7, 0xFE)):
        if v < (1 << (5 * n + 1 if n < 7 else 36)):
            out = []
            for _ in range(n - 1):
                out.append(0x80 | (v & 0x3F))
                v >>= 6
            return bytes([lead | v] + out[::-1])
    raise ValueError('frame / sample number needs more than 36 bits')


# -------------------------------------------------------------------------------------------------------------- encoder


def _zigzag(r):
    return np.where(r >= 0, r << 1, ((-r) << 1) - 1).astype(np.int64)


def _rice_param(u, limit):
    m = float(u.mean()) if u.size else 0.0
    k = int(math.floor(math.log2(m + 1.0))) if m > 0 else 0
    return min(k, limit)


def _put_residual(bw, res, order, bs, sub, stats):
    """Residual with partitioned Rice coding.  sub['rice5'], sub['porder'], sub['escape'] in ('none', 'some', 'all')."""
    rice5 = bool(sub.get('rice5'))
    porder = sub['porder']
    escape = sub.get('escape', 'none')
    u_all = _zigzag(res)
    if not rice5 and u_all.size and _rice_param(u_all, 30) > 14:
        rice5 = True                                   # a 4-bit parameter would need very long unary prefixes
    bw.put(1 if rice5 else 0, 2)
    bw.put(porder, 4)
    limit, esc = (30, 31) if rice5 else (14, 15)
    nparts = 1 << porder
    psize = bs >> porder
    start = 0
    for p in range(nparts):
        n = psize - order if p == 0 else psize
        r, u = res[start:start + n], u_all[start:start + n]
        start += n
        if escape == 'all' or (escape == 'some' and p % 2 == 1):
            raw = 0 if not r.size or not r.any() else int(max(int(r.max()).bit_length(), int((-r - 1).max()).bit_length())) + 1
            bw.put(esc, 5 if rice5 else 4)
            bw.put(raw, 5)
            bw.put_signed_array(r, raw)
            stats['escape_raw0' if raw == 0 else 'escape'] = stats.get('escape_raw0' if raw == 0 else 'escape', 0) + 1
            continue
        k = _rice_param(u, limit)
        bw.put(k, 5 if rice5 else 4)
        q = u >> k
        bw.put_fields((np.uint64(1) << np.uint64(k)) | (u & ((1 << k) - 1)).astype(np.uint64), q + 1 + k)
    stats['rice5' if rice5 else 'rice4'] = stats.get('rice5' if rice5 else 'rice4', 0) + 1
    stats.setdefault('porders', set()).add(porder)


def fixed_residual(s, order):
    s = np.asarray(s, np.int64)
    r = s.copy()
    for _ in range(order):
        r = np.diff(r)
    return r


def lpc_residual(s, coefs, shift):
    s = np.asarray(s, np.int64)
    order, n = len(coefs), len(s)
    pred = np.zeros(n - order, np.int64)
    for j, c in enumerate(coefs):
        pred += int(c) * s[order - 1 - j:n - 1 - j]
    return s[order:] - (pred >> shift)


def _put_subframe(bw, s, bps, sub, stats):
    """s: int64 samples of one subframe (side channels have bps + 1 bits)."""
    kind = sub['type']
    w = sub.get('wasted', 0)
    if w:
        assert not (s & ((1 << w) - 1)).any()
        s = s >> w
    eb = bps - w
    code = {'constant': 0, 'verbatim': 1}.get(kind)
    if kind == 'fixed':
        code = 8 + sub['order']
    elif kind == 'lpc':
        code = 32 + sub['order'] - 1
    bw.put(0, 1)
    bw.put(code, 6)
    if w:
        bw.put(1, 1)
        bw.put(1, w)                                   # w - 1 zeros then a one
    else:
        bw.put(0, 1)
    stats.setdefault('kinds', set()).add((kind, sub.get('order', 0)))
    if w:
        stats.setdefault('wasted', set()).add(w)
    if kind == 'constant':
        assert (s == s[0]).all()
        bw.put_signed_array(s[:1], eb)
    elif kind == 'verbatim':
        bw.put_signed_array(s, eb)
    elif kind == 'fixed':
        o = sub['order']
        bw.put_signed_array(s[:o], eb)
        _put_residual(bw, fixed_residual(s, o), o, len(s), sub, stats)
    else:
        o, prec, shift, coefs = sub['order'], sub['precision'], sub['shift'], sub['coefs']
        bw.put_signed_array(s[:o], eb)
        bw.put(prec - 1, 4)
        bw.put(shift, 5)
        bw.put_signed_array(coefs, prec)
        stats.setdefault('precisions', set()).add(prec)
        stats.setdefault('shifts', set()).add(shift)
        _put_residual(bw, lpc_residual(s, coefs, shift), o, len(s), sub, stats)


def subframe_signals(x, mode):
    """(channels, bs) int64 -> the signals coded in the subframes, and each one's extra bit (1 for a side channel)."""
    x = np.asarray(x, np.int64)
    if mode == CH_LEFT_SIDE:
        return [x[0], x[0] - x[1]], [0, 1]
    if mode == CH_SIDE_RIGHT:
        return [x[0] - x[1], x[1]], [1, 0]
    if mode == CH_MID_SIDE:
        return [(x[0] + x[1]) >> 1, x[0] - x[1]], [0, 1]
    return list(x), [0] * x.shape[0]


def frame_header(number, bs, bs_code, rate_code, rate, ch_code, bps_code, variable):
    h = bytearray([0xFF, 0xF9 if variable else 0xF8, (bs_code << 4) | rate_code, (ch_code << 4) | (bps_code << 1)])
    h += utf8_number(number)
    if bs_code == 6:
        h.append(bs - 1)
    elif bs_code == 7:
        h += struct.pack('>H', bs - 1)
    if rate_code == 12:
        h.append(rate // 1000)
    elif rate_code == 13:
        h += struct.pack('>H', rate)
    elif rate_code == 14:
        h += struct.pack('>H', rate // 10)
    h.append(crc8(h))
    return bytes(h)


def encode_frames(x, bps, rate, frames, variable):
    """x: int (channels, n).  frames: list of dicts {bs, bs_code, rate_code, bps_code, mode, subs}; mode is
    'independent' or a stereo code 8/9/10.  Returns (list of frame byte strings, stats)."""
    x = np.asarray(x, np.int64)
    C = x.shape[0]
    stats = {}
    bodies, headers = [], []
    pos = 0
    for k, fr in enumerate(frames):
        bs = fr['bs']
        blk = x[:, pos:pos + bs]
        mode = fr.get('mode', CH_INDEPENDENT)
        ch_code = C - 1 if mode == CH_INDEPENDENT else mode
        headers.append(frame_header(pos if variable else k, bs, fr['bs_code'], fr['rate_code'], rate, ch_code,
                                    fr['bps_code'], variable))
        stats.setdefault('bs_codes', set()).add(fr['bs_code'])
        stats.setdefault('rate_codes', set()).add(fr['rate_code'])
        stats.setdefault('bps_codes', set()).add(fr['bps_code'])
        stats.setdefault('modes', set()).add(mode if C == 2 else 'independent%d' % C)
        sigs, extra = subframe_signals(blk, mode)
        bw = BitWriter()
        for c in range(C):
            _put_subframe(bw, sigs[c], bps + extra[c], fr['subs'][c], stats)
        bodies.append(headers[-1] + bw.tobytes())
        pos += bs
    assert pos == x.shape[1], 'frames cover %d of %d samples' % (pos, x.shape[1])
    crcs = crc16_many(bodies)
    return [b + struct.pack('>H', c) for b, c in zip(bodies, crcs)], stats


def md5_of(x, bps):
    nb = (bps + 7) // 8
    inter = np.ascontiguousarray(np.asarray(x, np.int64).T).reshape(-1).astype('<i4')
    return hashlib.md5(inter.view(np.uint8).reshape(-1, 4)[:, :nb].tobytes()).digest()


def _block(btype, payload, last):
    return bytes([(0x80 if last else 0) | btype]) + struct.pack('>I', len(payload))[1:] + payload


def metadata(x, bps, rate, frames, frame_bytes, extra_blocks=True, write_total=True):
    C, n = np.asarray(x).shape
    sizes = [f['bs'] for f in frames]
    bmin = max(16, min(sizes[:-1] or sizes))
    bmax = min(65535, max(16, max(sizes)))
    flen = [len(b) for b in frame_bytes]
    si = struct.pack('>HH', bmin, bmax) + struct.pack('>I', min(flen))[1:] + struct.pack('>I', max(flen))[1:]
    packed = (rate << 44) | ((C - 1) << 41) | ((bps - 1) << 36) | (n if write_total else 0)
    si += struct.pack('>Q', packed) + md5_of(x, bps)
    blocks = [(0, si)]
    if extra_blocks:
        blocks.append((3, struct.pack('>QQH', 0, 0, sizes[0]) + b'\xff' * 8 + b'\0' * 10))   # a point + a placeholder
        vendor = b'flac_oracle'
        comments = [b'TITLE=coverage', b'ARTIST=\xff\xf8 sync bytes in a comment']
        vc = struct.pack('<I', len(vendor)) + vendor + struct.pack('<I', len(comments))
        for cmt in comments:
            vc += struct.pack('<I', len(cmt)) + cmt
        blocks.append((4, vc))
        mime, desc, img = b'image/png', b'cover', b'\x89PNG\r\n\x1a\n\xff\xf8\xff\xf9'
        blocks.append((6, struct.pack('>II', 3, len(mime)) + mime + struct.pack('>I', len(desc)) + desc
                       + struct.pack('>IIIII', 1, 1, 24, 0, len(img)) + img))
        blocks.append((1, b'\0' * 37))
    out = b'fLaC'
    for i, (t, p) in enumerate(blocks):
        out += _block(t, p, i == len(blocks) - 1)
    return out


def id3v2(footer=False, payload=b'TIT2\x00\x00\x00\x05\x00\x00\x03abcd'):
    size = len(payload)
    ss = bytes([(size >> 21) & 0x7F, (size >> 14) & 0x7F, (size >> 7) & 0x7F, size & 0x7F])
    head = b'ID3' + bytes([4, 0, 0x10 if footer else 0]) + ss
    return head + payload + ((b'3DI' + bytes([4, 0, 0x10]) + ss) if footer else b'')


def encode(x, bps, rate, frames, variable=False, id3=None, extra_blocks=True, write_total=True):
    """A whole stream: [ID3v2] fLaC, STREAMINFO (+ SEEKTABLE, VORBIS_COMMENT, PICTURE, PADDING), frames.
    Returns (bytes, info) with info['frame_offsets'] (byte offset of every frame) and info['stats']."""
    fb, stats = encode_frames(x, bps, rate, frames, variable)
    head = (id3v2(footer=id3 == 'footer') if id3 else b'') + metadata(x, bps, rate, frames, fb, extra_blocks,
                                                                      write_total)
    offs = np.cumsum([len(head)] + [len(b) for b in fb])[:-1]
    return head + b''.join(fb), dict(frame_offsets=[int(o) for o in offs], stats=stats, audio_start=len(head))


# ----------------------------------------------------------------------------------------------- coverage schedule

# (channels, bps, rate, variable, [(block size, block-size code), ...], header rate codes to cycle, id3)
MATRIX = [
    (1, 8, 8000, False, [(192, 1)] * 6 + [(100, 6)], [0, 4, 12, 13, 14], 'plain'),
    (2, 16, 44100, False, [(576, 2)] * 7 + [(500, 7)], [0, 9, 13, 14], 'footer'),
    (2, 24, 48000, True, [(1152, 3), (2304, 4), (256, 8), (512, 9), (1024, 10), (37, 6), (300, 7), (1, 6), (2, 7),
                          (64, 6)], [0, 10, 13, 14], 'plain'),
    (2, 12, 22050, True, [(4608, 5), (2048, 11), (4096, 12), (96, 6)], [0, 6, 13, 14], None),
    (1, 20, 96000, True, [(8192, 13), (16384, 14)], [0, 11, 12, 14], 'plain'),
    (1, 16, 88200, True, [(32768, 15), (65535, 7)], [0, 1, 14], None),
    (3, 16, 176400, False, [(256, 8)] * 2, [0, 2], 'plain'),
    (4, 20, 192000, False, [(256, 8)] * 2, [0, 3], None),
    (5, 8, 16000, False, [(128, 6)] * 3, [0, 5, 12], 'plain'),
    (6, 12, 24000, False, [(256, 8)] * 2, [0, 7], None),
    (7, 16, 32000, False, [(192, 1)] * 2, [0, 8], 'plain'),
    (8, 24, 44100, False, [(288, 7)] * 2, [0, 9], None),
]

_BPS_CODE = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6}
_KINDS = [('constant', 0), ('verbatim', 0)] + [('fixed', o) for o in range(5)] + [('lpc', o) for o in range(1, 33)]


def _base_signal(rng, n, amp, ramp):
    if ramp:
        return (-(amp // 2) + (amp // max(n, 1)) * np.arange(n)).astype(np.int64)
    t = np.arange(n)
    f = rng.uniform(0.001, 0.05)
    s = 0.6 * amp * np.sin(2 * np.pi * f * t + rng.uniform(0, 6)) + rng.integers(-4, 5, n)
    return np.clip(np.round(s), -amp, amp).astype(np.int64)


def _lpc_coefs(rng, order, prec, shift):
    lo, hi = -(1 << (prec - 1)), (1 << (prec - 1)) - 1
    c = rng.integers(lo, hi + 1, order).astype(np.int64)
    tot = int(np.abs(c).sum())
    if tot > (1 << shift):                              # keeps |prediction| <= max|s| so residuals stay in 32 bits
        c = np.fix(c * (1 << shift) / tot).astype(np.int64)
    return c


def matrix_streams(seed=0):
    """The coverage streams: list of (bytes, ints (channels, n), bps, rate, info).  Together they use every subframe
    type and FIXED / LPC order, LPC precisions 1-15 and shifts 0-15, wasted bits, both Rice parameter widths, escaped
    partitions (also with 0 raw bits), partition orders 0-15, every channel assignment, bit depths 8/12/16/20/24, every
    block-size and sample-rate header code, both block strategies, ID3v2 prefixes with and without a footer and the
    PADDING / VORBIS_COMMENT / SEEKTABLE / PICTURE blocks."""
    rng = np.random.default_rng(seed)
    kind_i = prec_i = shift_i = sub_i = 0
    out = []
    stereo_modes = [CH_INDEPENDENT, CH_LEFT_SIDE, CH_SIDE_RIGHT, CH_MID_SIDE]
    mode_i = 0
    for C, bps, rate, variable, sizes, rate_codes, id3 in MATRIX:
        frames, blocks = [], []
        for fi, (bs, bs_code) in enumerate(sizes):
            mode = CH_INDEPENDENT
            if C == 2:
                mode = stereo_modes[mode_i % 4]
                mode_i += 1
            subs, sigs = [], []
            for c in range(C):
                extra = 1 if (mode == CH_LEFT_SIDE and c == 1) or (mode == CH_SIDE_RIGHT and c == 0) or \
                    (mode == CH_MID_SIDE and c == 1) else 0
                amp = 1 << (bps - 3)
                kind, order = _KINDS[kind_i % len(_KINDS)]
                if bs >= 8192 or (bs >= 1024 and c == 0):
                    kind, order = 'fixed', 1                # the large blocks cover partition orders 10-15
                elif order > bs or (kind == 'lpc' and bs < 2 * order):
                    kind, order = 'fixed', min(bs, 1)
                else:
                    kind_i += 1
                w = [0, 1, 0, 2, 0, 3][sub_i % 6] if bps + extra - 3 > 4 else 0
                ramp = sub_i % 5 == 2
                s = _base_signal(rng, bs, amp, ramp) if kind != 'constant' else np.full(bs, rng.integers(-amp, amp))
                s = (s >> w) << w
                sub = dict(type=kind, order=order, wasted=w, rice5=sub_i % 2 == 1,
                           escape=['none', 'some', 'none', 'all'][sub_i % 4] if not ramp else 'all')
                maxp = 0
                while maxp < 15 and bs % (2 << maxp) == 0 and (bs >> (maxp + 1)) >= max(order, 1):
                    maxp += 1
                sub['porder'] = maxp if bs >= 1024 else min(maxp, sub_i % 10)
                if kind == 'lpc':
                    sub['precision'] = 1 + prec_i % 15
                    sub['shift'] = shift_i % 16
                    prec_i += 1
                    shift_i += 1
                    sub['coefs'] = _lpc_coefs(rng, order, sub['precision'], sub['shift'])
                subs.append(sub)
                sigs.append(s)
                sub_i += 1
            # the subframe signals come first; the channels are what decorrelation turns them into
            if mode == CH_LEFT_SIDE:
                L, S = sigs
                blk = [L, L - S]
            elif mode == CH_SIDE_RIGHT:
                S, R = sigs
                blk = [S + R, R]
            elif mode == CH_MID_SIDE:
                M, S = sigs
                m = (M << 1) | (S & 1)
                blk = [(m + S) >> 1, (m - S) >> 1]
            else:
                blk = sigs
            blocks.append(np.stack(blk))
            frames.append(dict(bs=bs, bs_code=bs_code, rate_code=rate_codes[fi % len(rate_codes)],
                               bps_code=_BPS_CODE[bps] if fi % 2 else 0, mode=mode, subs=subs))
        x = np.concatenate(blocks, axis=1)
        assert np.abs(x).max() < (1 << (bps - 1))
        data, info = encode(x, bps, rate, frames, variable=variable, id3=id3)
        out.append((data, x, bps, rate, info))
    return out


def merged_stats(streams):
    st = {}
    for *_, info in streams:
        for k, v in info['stats'].items():
            if isinstance(v, set):
                st.setdefault(k, set()).update(v)
            else:
                st[k] = st.get(k, 0) + v
    return st


# ------------------------------------------------------------------------------------- long stream for the measurement


def _levinson(r, order):
    a = np.zeros(order + 1)
    a[0] = 1.0
    err = r[0]
    for i in range(1, order + 1):
        if err <= 0:
            break
        k = -(r[i] + np.dot(a[1:i], r[i - 1:0:-1])) / err
        a[1:i + 1] = a[1:i + 1] + k * np.concatenate([a[i - 1:0:-1], [1.0]])
        err *= 1 - k * k
    return -a[1:]


def _rice_bits(r):
    u = _zigzag(r)
    k = _rice_param(u, 14)
    return int((u >> k).sum()) + u.size * (k + 1)


def encode_long(x, bps=16, rate=44100, bs=4096, lpc_order=8, precision=14):
    """A fast encoder for long tracks: fixed block size, per frame and channel the cheaper of FIXED orders 0-4 and one
    quantised LPC (Levinson on the block's autocorrelation), stereo coded as left/right.  Returns (bytes, info)."""
    x = np.asarray(x, np.int64)
    C, n = x.shape
    frames = []
    for pos in range(0, n, bs):
        b = min(bs, n - pos)
        subs = []
        for c in range(C):
            s = x[c, pos:pos + b]
            best = ('fixed', 0, _rice_bits(s), None, 0)
            for o in range(1, 5):
                if o < b:
                    bits = _rice_bits(fixed_residual(s, o))
                    if bits < best[2]:
                        best = ('fixed', o, bits, None, 0)
            if b > 4 * lpc_order:
                f = s.astype(np.float64)
                r = np.array([np.dot(f[:b - i], f[i:]) for i in range(lpc_order + 1)])
                if r[0] > 0:
                    r[0] *= 1.0 + 1e-9
                    a = _levinson(r, lpc_order)
                    amax = np.abs(a).max()
                    if amax > 0:
                        shift = int(np.clip(precision - 1 - math.ceil(math.log2(amax + 1e-12)), 0, 15))
                        q = np.clip(np.round(a * (1 << shift)), -(1 << (precision - 1)),
                                    (1 << (precision - 1)) - 1).astype(np.int64)
                        bits = _rice_bits(lpc_residual(s, q, shift)) + lpc_order * precision
                        if bits < best[2]:
                            best = ('lpc', lpc_order, bits, q, shift)
            kind, o, _, q, shift = best
            sub = dict(type=kind, order=o, porder=0, rice5=False)
            if kind == 'lpc':
                sub.update(precision=precision, shift=shift, coefs=q)
            subs.append(sub)
        bs_code = 12 if b == 4096 and bs == 4096 else 7
        frames.append(dict(bs=b, bs_code=bs_code, rate_code=9 if rate == 44100 else 0, bps_code=_BPS_CODE[bps],
                           mode=CH_INDEPENDENT, subs=subs))
    return encode(x, bps, rate, frames)


# ------------------------------------------------------------------------------------------------------------ decoder


def parse_frame_header(d, i):
    """Frame header at byte i, restating RFC 9639 section 9.1: dict, or None when there is no sync, the coded number
    is malformed, the header runs past the data or its CRC-8 does not match.  Reserved codes are returned, not
    judged."""
    n = len(d)
    if i + 5 > n or d[i] != 0xFF or (d[i + 1] & 0xFE) != 0xF8:
        return None
    b2, b3 = d[i + 2], d[i + 3]
    p = i + 4
    lead = d[p]
    if lead < 0x80:
        cont, v = 0, lead
    else:
        for cont, mask, pat in ((1, 0x1F, 0xC0), (2, 0x0F, 0xE0), (3, 0x07, 0xF0), (4, 0x03, 0xF8), (5, 0x01, 0xFC),
                                (6, 0x00, 0xFE)):
            if lead & ~mask & 0xFF == pat:
                v = lead & mask
                break
        else:
            return None
    p += 1
    for _ in range(cont):
        if p >= n or d[p] & 0xC0 != 0x80:
            return None
        v = (v << 6) | (d[p] & 0x3F)
        p += 1
    bs_code, rate_code = b2 >> 4, b2 & 15
    extra_bs = None
    if bs_code in (6, 7):
        k = bs_code - 5
        if p + k > n:
            return None
        extra_bs = int.from_bytes(bytes(d[p:p + k]), 'big')
        p += k
    rate_val = 0
    if rate_code in (12, 13, 14):
        k = 1 if rate_code == 12 else 2
        if p + k > n:
            return None
        rate_val = int.from_bytes(bytes(d[p:p + k]), 'big')
        p += k
    if p >= n or crc8(d[i:p]) != d[p]:
        return None
    return dict(offset=i, variable=d[i + 1] & 1, number=v, bs_code=bs_code, rate_code=rate_code, rate_val=rate_val,
                ch_code=b3 >> 4, bps_code=(b3 >> 1) & 7, reserved=b3 & 1,
                bs=block_size_of_code(bs_code, extra_bs) or 0, header_len=p + 1 - i)


def scan_candidates(d):
    """Every byte offset that holds a frame header (parse_frame_header is not None), in the candidate-table layout of
    lib/flac.py: int64 rows (offset, coded number, block size | header length << 17 | strategy << 22,
    byte 2 | byte 3 << 8 | coded rate value << 16)."""
    d = bytes(d)
    rows = []
    i = d.find(b'\xff')
    while 0 <= i:
        h = parse_frame_header(d, i)
        if h is not None:
            rows.append((i, h['number'], h['bs'] | (h['header_len'] << 17) | (h['variable'] << 22),
                         d[i + 2] | (d[i + 3] << 8) | (h['rate_val'] << 16)))
        i = d.find(b'\xff', i + 1)
    return np.array(rows, np.int64).reshape(-1, 4)


def read_streaminfo(d):
    """(audio start offset, dict of STREAMINFO fields)."""
    p = 0
    if d[:3] == b'ID3':
        size = (d[6] << 21) | (d[7] << 14) | (d[8] << 7) | d[9]
        p = 10 + size + (10 if d[5] & 0x10 else 0)
    if d[p:p + 4] != b'fLaC':
        raise ValueError('not a FLAC stream')
    p += 4
    info = None
    while True:
        hdr = d[p]
        ln = int.from_bytes(d[p + 1:p + 4], 'big')
        if hdr & 0x7F == 0:
            b = d[p + 4:p + 4 + 34]
            packed = int.from_bytes(b[10:18], 'big')
            info = dict(rate=packed >> 44, channels=((packed >> 41) & 7) + 1, bps=((packed >> 36) & 31) + 1,
                        total=packed & ((1 << 36) - 1), md5=bytes(b[18:34]))
        p += 4 + ln
        if hdr & 0x80:
            return p, info


def _decode_subframe(br, bs, bps):
    if br.read(1):
        raise ValueError('subframe padding bit set')
    t = br.read(6)
    w = 0
    if br.read(1):
        w = br.unary() + 1
    eb = bps - w
    if t == 0:
        s = [br.read_signed(eb)] * bs
    elif t == 1:
        s = [br.read_signed(eb) for _ in range(bs)]
    elif 8 <= t <= 12 or t >= 32:
        order = t - 8 if t < 32 else t - 31
        s = [br.read_signed(eb) for _ in range(order)]
        if t >= 32:
            prec = br.read(4) + 1
            if prec == 16:
                raise ValueError('LPC precision code 1111')
            shift = br.read_signed(5)
            if shift < 0:
                raise ValueError('negative LPC shift')
            coefs = [br.read_signed(prec) for _ in range(order)]
        res = _decode_residual(br, bs, order)
        if t < 32:
            fixed = [[], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1]][order]
            for r in res:
                s.append(r + sum(c * s[-1 - j] for j, c in enumerate(fixed)))
        else:
            for r in res:
                s.append(r + (sum(c * s[-1 - j] for j, c in enumerate(coefs)) >> shift))
    else:
        raise ValueError('reserved subframe type %d' % t)
    return [v << w for v in s]


def _decode_residual(br, bs, order):
    method = br.read(2)
    if method > 1:
        raise ValueError('reserved residual coding method')
    pbits, esc = (5, 31) if method else (4, 15)
    porder = br.read(4)
    res = []
    for p in range(1 << porder):
        n = (bs >> porder) - (order if p == 0 else 0)
        k = br.read(pbits)
        if k == esc:
            raw = br.read(5)
            res += [br.read_signed(raw) for _ in range(n)]
        else:
            for _ in range(n):
                u = (br.unary() << k) | br.read(k)
                res.append((u >> 1) ^ -(u & 1))
    return res


def decode(d):
    """bytes -> (int64 (channels, n), rate, bps), decoding frame after frame from the end of the metadata and
    checking each frame's CRC-8 and CRC-16, the frame numbers and the STREAMINFO total."""
    d = bytes(d)
    p, si = read_streaminfo(d)
    if si['bps'] == 32:
        raise ValueError('32-bit FLAC is not supported')
    C, bps = si['channels'], si['bps']
    chans = [[] for _ in range(C)]
    k = n = 0
    while p < len(d):
        h = parse_frame_header(d, p)
        if h is None:
            raise ValueError('frame %d: no valid frame header at byte %d' % (k, p))
        if h['number'] != (n if h['variable'] else k):
            raise ValueError('frame %d: coded number %d' % (k, h['number']))
        if h['bs_code'] == 0 or h['rate_code'] == 15 or h['ch_code'] > 10 or h['bps_code'] in (3, 7) or h['reserved']:
            raise ValueError('frame %d: reserved header code' % k)
        fbps = BPS_CODES.get(h['bps_code'], bps)
        bs, ch = h['bs'], h['ch_code']
        nch = ch + 1 if ch < 8 else 2
        if nch != C or fbps != bps:
            raise ValueError('frame %d: header disagrees with STREAMINFO' % k)
        br = BitReader(d, 8 * (p + h['header_len']))
        extra = {8: [0, 1], 9: [1, 0], 10: [0, 1]}.get(ch, [0] * C)
        sub = [_decode_subframe(br, bs, bps + extra[c]) for c in range(C)]
        br.align()
        e = br.pos // 8
        if crc16(d[p:e]) != int.from_bytes(d[e:e + 2], 'big'):
            raise ValueError('frame %d: CRC-16 mismatch' % k)
        if ch == 8:
            sub[1] = [a - b for a, b in zip(sub[0], sub[1])]
        elif ch == 9:
            sub[0] = [a + b for a, b in zip(sub[0], sub[1])]
        elif ch == 10:
            mid, side = sub
            ms = [((m << 1) | (s & 1), s) for m, s in zip(mid, side)]
            sub = [[(m + s) >> 1 for m, s in ms], [(m - s) >> 1 for m, s in ms]]
        for c in range(C):
            chans[c] += sub[c]
        p = e + 2
        k += 1
        n += bs
    if si['total'] and si['total'] != n:
        raise ValueError('STREAMINFO gives %d samples, the frames %d' % (si['total'], n))
    return np.array(chans, np.int64).reshape(C, n), si['rate'], bps
