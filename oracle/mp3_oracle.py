"""MPEG-1 Audio Layer III (ISO/IEC 11172-3) test infrastructure: a float64 decoder restating the standard, a seeded
encoder with a real analysis (polyphase analysis filterbank, MDCT, quantisation, Huffman coding, bit reservoir), and a
``matrix()`` of short streams whose schedule covers the format lib/mp3.py accepts.  CPU only; the product (lib/mp3.py,
csrc/mp3.cu) never imports it.  The tables live in oracle/mp3_tables.py and are pinned by decoding ``matrix()`` with
FFmpeg's ``mp3float`` (oracle/ffmpeg_mp3.py).

Decoder contract (what lib/mp3.py reproduces on the GPU):
- an ID3v2 tag at the start is skipped; ID3v1 (``TAG``, 128 bytes) and APEv2 (``APETAGEX``) at the end are dropped;
- the chain starts at the first MPEG-1 Layer III header followed by a consistent one (same rate and mode) at the
  distance its frame length gives, and continues frame by frame to the end of the audio; a last frame cut short is
  dropped (``info['dropped']``);
- a first frame carrying ``Xing``, ``Info`` or ``VBRI`` produces no samples; with a LAME extension, the first
  ``delay + 529`` and the last ``max(padding - 529, 0)`` samples are dropped;
- a frame whose main data starts before the first byte of the stream decodes as an all-zero spectrum
  (``info['zeroed']``); the synthesis carries on through it;
- MPEG-1 intensity stereo uses the right channel's zero part; is_pos 7 is "not intensity" (that band takes MS when MS
  is on); the last band (long 21, short 12) takes the is_pos of the band below it, as FFmpeg and mpg123 do;
- a count1 quadruple that crosses the end of part2_3_length is dropped; tables 0, 4 and 14 code no bits.

The round trip ``decode(encode(x))`` reproduces ``x`` after ``LAG`` samples (analysis + synthesis polyphase delay 481,
plus one granule of the hybrid filterbank, 576); ``encode`` writes a LAME tag whose delay + 529 is that lag, so the
gapless trim gives back exactly the input's span.
"""
import bisect
import math

import numpy as np

from . import mp3_tables as T

LAG = 1057
GRANULE = 576
FRAME = 1152

# ------------------------------------------------------------------------------------------------------------- tables

_CODES = T.huffman_codes()
_DEC = []        # code table -> (left-aligned codes, lengths, symbols)
_ENC = []        # code table -> (lens[16][16], codes[16][16]) by (x, y)
for _rows in _CODES:
    _DEC.append(([c << (32 - ln) for _, ln, c in _rows], [ln for _, ln, _ in _rows], [s for s, _, _ in _rows]))
    _l, _c = np.zeros((16, 16), np.int64), np.zeros((16, 16), np.int64)
    for _s, _ln, _cd in _rows:
        _l[_s >> 4, _s & 15], _c[_s >> 4, _s & 15] = _ln, _cd
    _ENC.append((_l, _c))
_QA = sorted((c << (32 - ln), ln, v) for v, (c, ln) in enumerate(zip(T.QUAD_A_CODES, T.QUAD_A_LENGTHS)))
_QA_LEFT, _QA_LEN, _QA_VAL = [r[0] for r in _QA], [r[1] for r in _QA], [r[2] for r in _QA]
_D = np.asarray(T.synth_window())
_C = _D / 32.0


def _band_starts(widths):
    return np.concatenate([[0], np.cumsum(widths)]).astype(np.int64)


def _sin_window(n, i):
    return np.sin(np.pi / n * (np.asarray(i, np.float64) + 0.5))


def imdct_windows():
    """[block type 0, 1, 3] -> 36 taps; [2] -> the 12 taps of a short window."""
    i = np.arange(36)
    w0 = _sin_window(36, i)
    w1 = np.concatenate([w0[:18], np.ones(6), _sin_window(12, np.arange(6, 12)), np.zeros(6)])
    w3 = np.concatenate([np.zeros(6), _sin_window(12, np.arange(6)), np.ones(6), w0[18:]])
    return {0: w0, 1: w1, 2: _sin_window(12, np.arange(12)), 3: w3}


_WIN = imdct_windows()
_COS36 = np.cos(np.pi / 72 * np.outer(2 * np.arange(36) + 1 + 18, 2 * np.arange(18) + 1))   # [i][k]
_COS12 = np.cos(np.pi / 24 * np.outer(2 * np.arange(12) + 1 + 6, 2 * np.arange(6) + 1))
_N = np.cos(np.outer(16 + np.arange(64), 2 * np.arange(32) + 1) * np.pi / 64)               # V = N @ S
_M = np.cos(np.outer(2 * np.arange(32) + 1, np.arange(64) - 16) * np.pi / 64)               # S = M @ Y
_CI = np.array([-0.6, -0.535, -0.33, -0.185, -0.095, -0.041, -0.0142, -0.0037])
_CS, _CA = 1 / np.sqrt(1 + _CI ** 2), _CI / np.sqrt(1 + _CI ** 2)


def is_ratio(pos):
    """(left, right) gains of MPEG-1 intensity position 0..6."""
    if pos == 6:
        return 1.0, 0.0
    t = math.tan(pos * math.pi / 12)
    return t / (1 + t), 1 / (1 + t)


# ------------------------------------------------------------------------------------------------------------ headers


def parse_header(d, i):
    """Fields of the 4 bytes at ``i`` if they start with the 11-bit sync, else None."""
    if i + 4 > len(d) or d[i] != 0xFF or (d[i + 1] & 0xE0) != 0xE0:
        return None
    h = int.from_bytes(bytes(d[i:i + 4]), 'big')
    return dict(version=(h >> 19) & 3, layer=(h >> 17) & 3, crc=((h >> 16) & 1) == 0, br=(h >> 12) & 15,
                sr=(h >> 10) & 3, pad=(h >> 9) & 1, mode=(h >> 6) & 3, modex=(h >> 4) & 3, emph=h & 3, word=h)


def header_problem(h):
    """None for an MPEG-1 Layer III header this decoder takes, else why not."""
    if h['version'] == 1:
        return 'reserved MPEG version'
    if h['version'] != 3:
        return 'MPEG-2 / MPEG-2.5 (LSF, 8 to 24 kHz) is not supported'
    if h['layer'] == 0:
        return 'reserved layer'
    if h['layer'] != 1:
        return 'Layer %s is not supported (Layer III only)' % ('I' if h['layer'] == 3 else 'II')
    if h['br'] == 0:
        return 'free-format bitrate is not supported'
    if h['br'] == 15:
        return 'reserved bitrate index 15'
    if h['sr'] == 3:
        return 'reserved sampling frequency'
    if h['emph'] == 2:
        return 'reserved emphasis'
    return None


def frame_length(h):
    return 144000 * T.BITRATES[h['br']] // T.RATES[h['sr']] + h['pad']


def side_info_length(h):
    return 17 if h['mode'] == 3 else 32


class _Bits(object):
    """MSB-first reader over bytes [start bit, ...); bits past the data read as zero."""

    def __init__(self, buf, start, length):
        b0 = start // 8
        raw = bytes(buf[b0:(start + length + 7) // 8]) + bytes(8)
        self.v, self.n = int.from_bytes(raw, 'big'), 8 * len(raw)
        self.pos = start - 8 * b0
        self.end = self.pos + length

    def read(self, k):
        if k == 0:
            return 0
        self.pos += k
        return (self.v >> (self.n - self.pos)) & ((1 << k) - 1)

    def peek32(self):
        return (self.v >> (self.n - self.pos - 32)) & 0xFFFFFFFF


def parse_side_info(d, i, h):
    """Side info of the frame at byte ``i``: dict(main_data_begin, scfsi[ch], gr[gr][ch] dicts)."""
    C = 1 if h['mode'] == 3 else 2
    br = _Bits(d, 8 * (i + 4 + (2 if h['crc'] else 0)), 8 * side_info_length(h))
    si = dict(main_data_begin=br.read(9))
    br.read(5 if C == 1 else 3)
    si['scfsi'] = [br.read(4) for _ in range(C)]
    grs = []
    for gr in range(2):
        row = []
        for ch in range(C):
            g = dict(part2_3_length=br.read(12), big_values=br.read(9), global_gain=br.read(8),
                     scalefac_compress=br.read(4), window_switching=br.read(1))
            if g['window_switching']:
                g['block_type'], g['mixed'] = br.read(2), br.read(1)
                g['table_select'] = [br.read(5), br.read(5), 0]
                g['subblock_gain'] = [br.read(3) for _ in range(3)]
                g['region0_count'], g['region1_count'] = None, None
            else:
                g['block_type'], g['mixed'] = 0, 0
                g['table_select'] = [br.read(5) for _ in range(3)]
                g['subblock_gain'] = [0, 0, 0]
                g['region0_count'], g['region1_count'] = br.read(4), br.read(3)
            g['preflag'], g['scalefac_scale'], g['count1table'] = br.read(1), br.read(1), br.read(1)
            row.append(g)
        grs.append(row)
    si['gr'] = grs
    return si


# ------------------------------------------------------------------------------------------------ granule decoding


def _regions(g, sr):
    """(region1 start, region2 start, big-values end) in lines."""
    big = 2 * g['big_values']
    if g['window_switching']:
        r1, r2 = 36, 576
    else:
        bl = _band_starts(T.BAND_LONG[sr])
        r1 = int(bl[g['region0_count'] + 1])
        r2 = int(bl[min(g['region0_count'] + g['region1_count'] + 2, 22)])
    return min(r1, big), min(r2, big), big


def _read_scalefactors(br, g, gr, scfsi, prev):
    """Scale factors as dict(long=[22], short=[13][3]); ``prev``: granule 0's (for scfsi)."""
    s1, s2 = T.SLEN[g['scalefac_compress']]
    lo, sh = [0] * 22, [[0, 0, 0] for _ in range(13)]
    if g['block_type'] == 2 and g['window_switching']:
        if g['mixed']:
            for b in range(8):
                lo[b] = br.read(s1)
            first = 3
        else:
            first = 0
        for b in range(first, 12):
            for w in range(3):
                sh[b][w] = br.read(s1 if b < 6 else s2)
    else:
        groups = ((0, 6, s1), (6, 11, s1), (11, 16, s2), (16, 21, s2))
        for k, (a, b, s) in enumerate(groups):
            if gr == 1 and scfsi & (8 >> k):
                # granule 0's long scale factors; a short granule 0 has them only in a mixed block's bands 0-7, the
                # rest are 0 (FFmpeg copies its short-block values there instead; valid encoders never do this)
                lo[a:b] = prev['long'][a:b]
            else:
                for j in range(a, b):
                    lo[j] = br.read(s)
    return dict(long=lo, short=sh)


def line_layout(g, sr):
    """Per line of the granule in bitstream order: (sfb, window or -1 for long lines)."""
    sfb, win = np.zeros(576, np.int64), np.full(576, -1, np.int64)
    if g['block_type'] == 2 and g['window_switching']:
        p = 0
        if g['mixed']:
            bl = T.BAND_LONG[sr]
            for b in range(8):
                sfb[p:p + bl[b]] = b
                p += bl[b]
        bs = T.BAND_SHORT[sr]
        for b in range(3 if g['mixed'] else 0, 13):
            for w in range(3):
                sfb[p:p + bs[b]] = b
                win[p:p + bs[b]] = w
                p += bs[b]
    else:
        sfb = np.repeat(np.arange(22), T.BAND_LONG[sr])
    return sfb, win


def decode_granule(md, start, g, gr, scfsi, prev_sf, sr, stats=None):
    """(integer values [576], scale factors) of one granule-channel whose part2_3 data starts at bit ``start``."""
    br = _Bits(md, start, g['part2_3_length'])
    sf = _read_scalefactors(br, g, gr, scfsi, prev_sf)
    r1, r2, big = _regions(g, sr)
    ix = np.zeros(576, np.int64)
    k = 0
    for reg, stop in enumerate((r1, r2, big)):
        ts = g['table_select'][reg]
        tab = T.HUFF_TABLE[ts]
        if stats is not None and k < stop:
            stats['table_select'].add(ts)
        if tab is None:
            k = max(k, stop)
            continue
        lefts, lens, syms = _DEC[tab[0]]
        linbits = tab[1]
        while k < stop:
            i = bisect.bisect_right(lefts, br.peek32()) - 1
            br.pos += lens[i]
            x, y = syms[i] >> 4, syms[i] & 15
            if linbits and x == 15:
                x += br.read(linbits)
            if x and br.read(1):
                x = -x
            if linbits and y == 15:
                y += br.read(linbits)
            if y and br.read(1):
                y = -y
            ix[k], ix[k + 1] = x, y
            k += 2
    while k <= 572:
        if br.pos >= br.end:
            break
        if g['count1table']:
            v = 15 - br.read(4)
        else:
            i = bisect.bisect_right(_QA_LEFT, br.peek32()) - 1
            br.pos += _QA_LEN[i]
            v = _QA_VAL[i]
        q = [(v >> 3) & 1, (v >> 2) & 1, (v >> 1) & 1, v & 1]
        for j in range(4):
            if q[j] and br.read(1):
                q[j] = -1
        if br.pos > br.end:
            if stats is not None:
                stats['quad_dropped'] += 1
            break
        ix[k:k + 4] = q
        k += 4
    if stats is not None:
        stats['count1table'].add(g['count1table'])
        stats['count1_lines'] += k - big
    return ix, sf


def requantise(ix, g, sf, sr):
    sfb, win = line_layout(g, sr)
    mult = 1.0 if g['scalefac_scale'] else 0.5
    lo, sh = np.asarray(sf['long'], np.float64), np.asarray(sf['short'], np.float64)
    pre = np.asarray(T.PRETAB, np.float64) * g['preflag']
    e = np.where(win < 0, 0.25 * (g['global_gain'] - 210) - mult * (lo[sfb % 22] + pre[sfb % 22]),
                 0.25 * (g['global_gain'] - 210 - 8 * np.asarray(g['subblock_gain'])[np.maximum(win, 0)])
                 - mult * sh[np.minimum(sfb, 12), np.maximum(win, 0)])
    a = np.abs(ix).astype(np.float64)
    return np.sign(ix) * a ** (4.0 / 3.0) * np.exp2(e)


def stereo(xr, g, sf_r, modex, sr):
    """MS and MPEG-1 intensity stereo in place on xr[2][576] (bitstream order), after FFmpeg's compute_stereo."""
    ms, inten = modex & 2, modex & 1
    if not inten:
        if ms:
            a, b = xr[0].copy(), xr[1].copy()
            xr[0], xr[1] = (a + b) / math.sqrt(2), (a - b) / math.sqrt(2)
        return
    g1 = g[1]
    short = g1['block_type'] == 2 and g1['window_switching']
    long_end = (8 if g1['mixed'] else 0) if short else 22
    bl, bs = T.BAND_LONG[sr], T.BAND_SHORT[sr]
    p = 576
    found = {}

    def apply(a, n, pos):
        seg0, seg1 = xr[0, a:a + n], xr[1, a:a + n]
        if pos is None:
            if ms:
                s0, s1 = seg0.copy(), seg1.copy()
                xr[0, a:a + n], xr[1, a:a + n] = (s0 + s1) / math.sqrt(2), (s0 - s1) / math.sqrt(2)
            return
        lg, rg = is_ratio(pos)
        s0 = seg0.copy()
        xr[0, a:a + n], xr[1, a:a + n] = s0 * lg, s0 * rg

    if short:
        for b in range(12, (3 if g1['mixed'] else 0) - 1, -1):
            n = bs[b]
            for w in (2, 1, 0):
                p -= n
                if not found.get(w) and np.any(xr[1, p:p + n] != 0):
                    found[w] = True
                if found.get(w):
                    apply(p, n, None)
                    continue
                pos = sf_r['short'][11 if b == 12 else b][w]
                apply(p, n, None if pos >= 7 else pos)
        nz = any(found.values())
    else:
        nz = False
    for b in range(long_end - 1, -1, -1):
        n = bl[b]
        p -= n
        if not nz and np.any(xr[1, p:p + n] != 0):
            nz = True
        if nz:
            apply(p, n, None)
            continue
        pos = sf_r['long'][20 if b == 21 else b]
        apply(p, n, None if pos >= 7 else pos)


def reorder(xr, g, sr):
    """Short-block lines from bitstream order (sfb, window, line) to (subband, 3 * k + window)."""
    if not (g['block_type'] == 2 and g['window_switching']):
        return xr
    out = xr.copy()
    p = 36 if g['mixed'] else 0
    bs = T.BAND_SHORT[sr]
    for b in range(3 if g['mixed'] else 0, 13):
        n = bs[b]
        blk = xr[p:p + 3 * n].reshape(3, n)
        out[p:p + 3 * n] = blk.T.reshape(-1)
        p += 3 * n
    return out


def antialias(xr, g):
    short = g['block_type'] == 2 and g['window_switching']
    if short and not g['mixed']:
        return xr
    xr = xr.copy()
    for sb in range(1 if short else 31):
        a = xr[18 * sb + 17 - np.arange(8)].copy()
        b = xr[18 * (sb + 1) + np.arange(8)].copy()
        xr[18 * sb + 17 - np.arange(8)] = a * _CS - b * _CA
        xr[18 * (sb + 1) + np.arange(8)] = b * _CS + a * _CA
    return xr


def imdct(xr, g):
    """[32][36] windowed IMDCT outputs of a granule (after reorder and antialias)."""
    short = g['block_type'] == 2 and g['window_switching']
    x = xr.reshape(32, 18)
    out = np.zeros((32, 36))
    for sb in range(32):
        if short and not (g['mixed'] and sb < 2):
            for w in range(3):
                y = _COS12 @ x[sb, w::3] * _WIN[2]
                out[sb, 6 + 6 * w:18 + 6 * w] += y
        else:
            bt = 0 if short else g['block_type']
            out[sb] = _COS36 @ x[sb] * _WIN[bt]
    return out


def synthesise(S):
    """Polyphase synthesis of subband samples S[slot][32] (float64) -> samples (32 * slots,), zero state before."""
    T_ = S.shape[0]
    V = np.concatenate([np.zeros((16, 64)), S @ _N.T])       # V[t + 16] is slot t's vector
    out = np.zeros((T_, 32))
    for i in range(8):
        out += V[16 - 2 * i:16 - 2 * i + T_, :32] * _D[64 * i:64 * i + 32]
        out += V[15 - 2 * i:15 - 2 * i + T_, 32:] * _D[64 * i + 32:64 * i + 64]
    return out.reshape(-1)


# ---------------------------------------------------------------------------------------------------------- streams


def id3v2_size(d):
    if len(d) < 10 or d[:3] != b'ID3':
        return 0
    return 10 + ((d[6] & 0x7F) << 21 | (d[7] & 0x7F) << 14 | (d[8] & 0x7F) << 7 | (d[9] & 0x7F)) + \
        (10 if d[5] & 0x10 else 0)


def audio_end(d, start):
    """End of the frames: the file's end less an ID3v1 tag and an APEv2 tag (in either order of the two checks)."""
    end = len(d)
    for _ in range(2):
        if end - 128 >= start and d[end - 128:end - 125] == b'TAG':
            end -= 128
            continue
        if end - 32 >= start and d[end - 32:end - 24] == b'APETAGEX':
            size = int.from_bytes(d[end - 20:end - 16], 'little')
            flags = int.from_bytes(d[end - 12:end - 8], 'little')
            end -= size + (32 if flags & 0x80000000 else 0)
            end = max(end, start)
            continue
        break
    return end


def xing_info(d, i, h):
    """None, or dict(delay, padding, lame) of a Xing / Info / VBRI header in the frame at ``i``."""
    o = i + 4 + (2 if h['crc'] else 0) + side_info_length(h)
    if d[i + 36:i + 40] == b'VBRI':
        return dict(delay=0, padding=0, lame=False)
    if d[o:o + 4] not in (b'Xing', b'Info'):
        return None
    flags = int.from_bytes(d[o + 4:o + 8], 'big')
    p = o + 8 + (4 if flags & 1 else 0) + (4 if flags & 2 else 0) + (100 if flags & 4 else 0) + \
        (4 if flags & 8 else 0)
    if d[p:p + 4] in (b'LAME', b'Lavf', b'Lavc') and p + 24 <= i + frame_length(h):
        v = int.from_bytes(d[p + 21:p + 24], 'big')
        return dict(delay=v >> 12, padding=v & 0xFFF, lame=True)
    return dict(delay=0, padding=0, lame=False)


def find_frames(d, name='<bytes>'):
    """(frame byte offsets, headers, info) by the chain rules in the module docstring."""
    start = id3v2_size(d)
    end = audio_end(d, start)
    first = None
    i = start
    while i + 4 <= end:
        h = parse_header(d, i)
        if h is not None and header_problem(h) is None:
            j = i + frame_length(h)
            h2 = parse_header(d, j) if j + 4 <= end else None
            if j == end or (h2 is not None and header_problem(h2) is None and h2['sr'] == h['sr'] and
                            h2['mode'] == h['mode']):
                first = i
                break
        i += 1
    if first is None:
        raise ValueError('%s: no MPEG-1 Layer III frame found' % name)
    offs, hdrs, dropped = [], [], 0
    i = first
    while i < end:
        h = parse_header(d, i) if i + 4 <= end else None
        if h is None:
            raise ValueError('%s: frame %d (byte %d): the frame chain breaks' % (name, len(offs), i))
        why = header_problem(h)
        if why:
            raise ValueError('%s: frame %d (byte %d): %s' % (name, len(offs), i, why))
        if hdrs and (h['sr'] != hdrs[0]['sr'] or h['mode'] != hdrs[0]['mode']):
            raise ValueError('%s: frame %d (byte %d): the sample rate or channel mode changes' % (name, len(offs), i))
        n = frame_length(h)
        if i + n > end:
            dropped += 1
            break
        offs.append(i)
        hdrs.append(h)
        i += n
    return offs, hdrs, dict(start=start, end=end, dropped=dropped)


def decode_frames(d, offs, hdrs, stats=None):
    """float64 (channels, 1152 * frames) of the given frames, decoded in order, no trim; also the zeroed count."""
    C = 1 if hdrs[0]['mode'] == 3 else 2
    sr = hdrs[0]['sr']
    md, md_off, sis = bytearray(), [], []
    for i, h in zip(offs, hdrs):
        s = i + 4 + (2 if h['crc'] else 0) + side_info_length(h)
        md_off.append(len(md))
        md += d[s:i + frame_length(h)]
        sis.append(parse_side_info(d, i, h))
    md = bytes(md)
    F = len(offs)
    S = np.zeros((C, 36 * F, 32))
    prev_tail = np.zeros((C, 32, 18))
    zeroed = 0
    for f, (h, si) in enumerate(zip(hdrs, sis)):
        begin = md_off[f] - si['main_data_begin']
        bit = 8 * begin
        zero = begin < 0
        zeroed += zero
        sf_prev = [None] * C
        if stats is not None:
            stats['modes'].add((h['mode'], h['modex'] if h['mode'] == 1 else 0))
            stats['bitrates'].add(h['br'])
            stats['rates'].add(h['sr'])
            stats['crc'].add(h['crc'])
            stats['padding'].add(h['pad'])
            stats['main_data_begin'] = max(stats['main_data_begin'], si['main_data_begin'])
        for gr in range(2):
            gs = si['gr'][gr]
            xr = np.zeros((C, 576))
            sfs = []
            for ch in range(C):
                g = gs[ch]
                if zero:
                    sfs.append(dict(long=[0] * 22, short=[[0] * 3 for _ in range(13)]))
                    continue
                if stats is not None:
                    blk = (g['block_type'], g['mixed']) if g['window_switching'] else (0, 0)
                    stats['blocks'].add(blk)
                    stats['rate_blocks'].add((h['sr'],) + blk)
                    if C == 2 and h['mode'] == 1 and h['modex'] & 1:
                        stats['rate_is'].add(h['sr'])
                    for key in ('preflag', 'scalefac_scale'):
                        stats[key].add(g[key])
                    stats['subblock_gain'].add(max(g['subblock_gain']))
                    if gr == 1 and si['scfsi'][ch]:
                        stats['scfsi'].add(si['scfsi'][ch])
                    e = bit + g['part2_3_length']
                    if e > 8 * (md_off[f] + 1) and bit < 8 * md_off[f]:
                        stats['spanning'] += 1
                ix, sf = decode_granule(md, bit, g, gr, si['scfsi'][ch], sf_prev[ch], sr, stats)
                bit += g['part2_3_length']
                sf_prev[ch] = sf
                sfs.append(sf)
                xr[ch] = requantise(ix, g, sf, sr)
            if not zero and C == 2 and h['mode'] == 1:
                stereo(xr, gs, sfs[1], h['modex'], sr)
            for ch in range(C):
                g = gs[ch]
                y = imdct(antialias(reorder(xr[ch], g, sr), g), g) if not zero else np.zeros((32, 36))
                out = y[:, :18] + prev_tail[ch]
                prev_tail[ch] = y[:, 18:]
                out[1::2, 1::2] *= -1
                S[ch, 36 * f + 18 * gr:36 * f + 18 * gr + 18] = out.T
    return np.stack([synthesise(S[c]) for c in range(C)]), zeroed


def decode(d, name='<bytes>', stats=None):
    """(float64 (channels, n), rate, info) of a whole file's bytes, by the contract in the module docstring."""
    d = bytes(d)
    offs, hdrs, info = find_frames(d, name)
    x = xing_info(d, offs[0], hdrs[0])
    delay = padding = 0
    if x is not None:
        offs, hdrs = offs[1:], hdrs[1:]
        if x['lame']:
            delay, padding = x['delay'], x['padding']
    if not offs:
        raise ValueError('%s: no audio frame after the Xing / Info header' % name)
    y, zeroed = decode_frames(d, offs, hdrs, stats)
    n = y.shape[1]
    a = min(delay + 529, n) if x is not None and x['lame'] else 0
    b = n - max(padding - 529, 0) if x is not None and x['lame'] else n
    info.update(frames=len(offs), delay=delay, padding=padding, zeroed=zeroed, xing=x is not None,
                lame=bool(x and x['lame']))
    return y[:, a:max(a, b)], T.RATES[hdrs[0]['sr']], info


def new_stats():
    return dict(table_select=set(), count1table=set(), blocks=set(), rate_blocks=set(), rate_is=set(), preflag=set(), scalefac_scale=set(),
                subblock_gain=set(), scfsi=set(), modes=set(), bitrates=set(), rates=set(), crc=set(), padding=set(),
                main_data_begin=0, spanning=0, quad_dropped=0, count1_lines=0)


# ------------------------------------------------------------------------------------------------------------ encoder


def analyse(x):
    """Polyphase analysis of (n,) samples -> subband samples [slot][32] (slots = ceil(n / 32)), zero state before."""
    n = len(x)
    T_ = (n + 31) // 32
    xp = np.concatenate([np.zeros(512), np.asarray(x, np.float64), np.zeros(32 * T_ - n)])
    out = np.zeros((T_, 32))
    step = 4096
    for a in range(0, T_, step):
        t = np.arange(a, min(T_, a + step))
        idx = 512 + 32 * t[:, None] + 31 - np.arange(512)[None, :]      # X[i] = x[32 t + 31 - i]
        Z = xp[idx] * _C
        Y = Z.reshape(len(t), 8, 64).sum(1)
        out[t] = Y @ _M.T
    return out


def _mdct_granule(blk, bt, mixed):
    """blk: [32][36] subband samples (previous granule's 18 then this one's) -> aliased spectrum [576] as the decoder
    reads it after its antialias butterflies (hybrid order: subband, then 3 * k + window for short blocks)."""
    out = np.zeros((32, 18))
    for sb in range(32):
        if bt == 2 and not (mixed and sb < 2):
            for w in range(3):
                z = blk[sb, 6 + 6 * w:18 + 6 * w] * _WIN[2]
                out[sb, w::3] = (z @ _COS12) / 3.0
        else:
            z = blk[sb] * _WIN[0 if bt == 2 else bt]
            out[sb] = (z @ _COS36) / 9.0
    return out.reshape(-1)


def _inverse_antialias(xr, bt, mixed):
    if bt == 2 and not mixed:
        return xr
    xr = xr.copy()
    for sb in range(1 if bt == 2 else 31):
        a = xr[18 * sb + 17 - np.arange(8)].copy()
        b = xr[18 * (sb + 1) + np.arange(8)].copy()
        xr[18 * sb + 17 - np.arange(8)] = a * _CS + b * _CA
        xr[18 * (sb + 1) + np.arange(8)] = b * _CS - a * _CA
    return xr


def _to_bitstream_order(xr, bt, mixed, sr):
    if bt != 2:
        return xr
    out = xr.copy()
    p = 36 if mixed else 0
    for b in range(3 if mixed else 0, 13):
        n = T.BAND_SHORT[sr][b]
        out[p:p + 3 * n] = xr[p:p + 3 * n].reshape(n, 3).T.reshape(-1)
        p += 3 * n
    return out


class _Writer(object):
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, val, k):
        k = int(k)
        if k:
            self.v = (self.v << k) | (int(val) & ((1 << k) - 1))
            self.n += k

    def bytes(self):
        pad = (-self.n) % 8
        return (self.v << pad).to_bytes((self.n + pad) // 8, 'big')


def _pair_bits(a, ts):
    """Bits of the pairs a[::2], a[1::2] (absolute values) with table_select ts, or None if it cannot code them."""
    tab = T.HUFF_TABLE[ts]
    if tab is None:
        return 0 if not a.any() else None
    ct, lb = tab
    size = T.HUFF_SIZES[ct]
    mx = int(a.max()) if a.size else 0
    if (lb == 0 and mx >= size) or (lb and mx > 15 + (1 << lb) - 1):
        return None
    lens = _ENC[ct][0]
    x, y = np.minimum(a[0::2], 15), np.minimum(a[1::2], 15)
    return int(lens[x, y].sum() + (a > 0).sum() + (lb * ((a >= 15).sum()) if lb else 0))


def _capacity(ts):
    """Largest value table_select ts codes."""
    tab = T.HUFF_TABLE[ts]
    if tab is None:
        return 0
    return T.HUFF_SIZES[tab[0]] - 1 + ((1 << tab[1]) - 1 if tab[1] else 0)


def _quad_bits(a, table):
    q = a.reshape(-1, 4)
    v = q[:, 0] * 8 + q[:, 1] * 4 + q[:, 2] * 2 + q[:, 3]
    if table:
        return int(4 * len(v) + q.sum())
    return int(np.asarray(T.QUAD_A_LENGTHS)[v].sum() + q.sum())


class _Plan(object):
    """Everything the encoder decides for one granule-channel."""


def _layout(bt, mixed, sr):
    g = dict(block_type=bt, mixed=mixed, window_switching=1 if bt else 0)
    return line_layout(g, sr)


def _code_granule(ix, p, sr, opts, q):
    """Choose regions, tables and count1 for integer values ix (bitstream order); returns part2_3 bits and fills p."""
    a = np.abs(ix)
    nz = np.flatnonzero(a)
    last = int(nz[-1]) + 1 if nz.size else 0
    big_end = int(np.flatnonzero(a > 1)[-1]) + 1 if (a > 1).any() else 0
    big_end += big_end & 1
    c1_end = big_end
    while c1_end < last:
        c1_end += 4
    if c1_end > 576:                 # the quads do not fit: widen the big-values region
        big_end = last + (last & 1)
        c1_end = big_end
    p.big_values = big_end // 2
    if p.window_switching:
        r1 = min(36, big_end)
        r2 = big_end
        p.region0_count = p.region1_count = None
    else:
        bl = _band_starts(T.BAND_LONG[sr])
        best = None
        for r0 in range(16):
            for rr in range(8):
                if r0 + rr + 2 > 22:
                    continue
                a1, a2 = int(bl[r0 + 1]), int(bl[r0 + rr + 2])
                score = abs(a1 - big_end // 3) + abs(a2 - 2 * big_end // 3)
                if best is None or score < best[0]:
                    best = (score, r0, rr)
        p.region0_count, p.region1_count = best[1], best[2]
        r1 = min(int(bl[p.region0_count + 1]), big_end)
        r2 = min(int(bl[min(p.region0_count + p.region1_count + 2, 22)]), big_end)
    bits = 0
    p.table_select = [0, 0, 0]
    for reg, (s, e) in enumerate(((0, r1), (r1, r2), (r2, big_end))):
        if p.window_switching and reg == 2:
            continue
        seg = a[s:e]
        cands = [(b, ts) for ts in range(32) if (b := _pair_bits(seg, ts)) is not None and T.HUFF_TABLE[ts]]
        if not seg.any():
            cands.append((0, 0))
        if opts.get('cycle_tables') and seg.size:
            cands.sort(key=lambda c: (_capacity(c[1]), c[1]))       # the narrowest tables first
            used = opts.setdefault('_used', set())
            fresh = [c for c in cands if c[1] not in used]
            opts['_turn'] = opts.get('_turn', -1) + 1
            b, ts = fresh[0] if fresh else cands[opts['_turn'] % len(cands)]
            if opts.get('_commit'):                                    # the choice that gets written
                used.add(ts)
        else:
            b, ts = min(cands)
        p.table_select[reg] = ts
        bits += b
    qa = a[big_end:c1_end]
    if opts.get('count1') is not None:
        p.count1table = opts['count1'] if not callable(opts['count1']) else opts['count1'](q)
    else:
        p.count1table = int(_quad_bits(qa, 1) < _quad_bits(qa, 0))
    bits += _quad_bits(qa, p.count1table)
    p.regions = (r1, r2, big_end, c1_end)
    return bits


def _write_granule(w, ix, p):
    r1, r2, big_end, c1_end = p.regions
    for reg, (s, e) in enumerate(((0, r1), (r1, r2), (r2, big_end))):
        tab = T.HUFF_TABLE[p.table_select[reg]]
        if tab is None:
            continue
        lens, codes = _ENC[tab[0]]
        lb = tab[1]
        for k in range(s, e, 2):
            vals = (int(ix[k]), int(ix[k + 1]))
            ax, ay = abs(vals[0]), abs(vals[1])
            cx, cy = min(ax, 15), min(ay, 15)
            w.put(codes[cx, cy], lens[cx, cy])
            for v, av in ((vals[0], ax), (vals[1], ay)):
                if lb and av >= 15:
                    w.put(av - 15, lb)
                if av:
                    w.put(1 if v < 0 else 0, 1)
    for k in range(big_end, c1_end, 4):
        q = [int(v) for v in ix[k:k + 4]]
        v = (abs(q[0]) << 3) | (abs(q[1]) << 2) | (abs(q[2]) << 1) | abs(q[3])
        if p.count1table:
            w.put(15 - v, 4)
        else:
            w.put(T.QUAD_A_CODES[v], T.QUAD_A_LENGTHS[v])
        for val in q:
            if val:
                w.put(1 if val < 0 else 0, 1)


def _quantise(xr, p, sr):
    """Integer values of xr (bitstream order) for the plan's gains and scale factors (nearest integer of |x|^(3/4))."""
    sfb, win = _layout(p.block_type, p.mixed, sr)
    mult = 1.0 if p.scalefac_scale else 0.5
    lo, sh = np.asarray(p.sf_long, np.float64), np.asarray(p.sf_short, np.float64)
    pre = np.asarray(T.PRETAB, np.float64) * p.preflag
    e = np.where(win < 0, 0.25 * (p.global_gain - 210) - mult * (lo[sfb % 22] + pre[sfb % 22]),
                 0.25 * (p.global_gain - 210 - 8 * np.asarray(p.subblock_gain)[np.maximum(win, 0)])
                 - mult * sh[np.minimum(sfb, 12), np.maximum(win, 0)])
    v = np.floor((np.abs(xr) * np.exp2(-e)) ** 0.75 + 0.5)
    return (np.sign(xr) * np.minimum(v, 8206)).astype(np.int64), bool((v > 8206).any())


def _sf_bits(p, gr, scfsi):
    s1, s2 = T.SLEN[p.scalefac_compress]
    if p.block_type == 2:
        return (8 * s1 + 9 * s1 + 18 * s2) if p.mixed else (18 * s1 + 18 * s2)
    n = 0
    for k, (cnt, s) in enumerate(((6, s1), (5, s1), (5, s2), (5, s2))):
        if not (gr == 1 and scfsi & (8 >> k)):
            n += cnt * s
    return n


def _write_sf(w, p, gr, scfsi):
    s1, s2 = T.SLEN[p.scalefac_compress]
    if p.block_type == 2:
        if p.mixed:
            for b in range(8):
                w.put(p.sf_long[b], s1)
        for b in range(3 if p.mixed else 0, 12):
            for win in range(3):
                w.put(p.sf_short[b][win], s1 if b < 6 else s2)
        return
    groups = ((0, 6, s1), (6, 11, s1), (11, 16, s2), (16, 21, s2))
    for k, (a, b, s) in enumerate(groups):
        if not (gr == 1 and scfsi & (8 >> k)):
            for j in range(a, b):
                w.put(p.sf_long[j], s)


def _crc16(data):
    c = 0xFFFF
    for b in data:
        for k in range(7, -1, -1):
            bit = ((b >> k) & 1) ^ ((c >> 15) & 1)
            c = (c << 1) & 0xFFFF
            if bit:
                c ^= 0x8005
    return c


def _header_bytes(br, sr, pad, mode, modex, crc):
    h = (0x7FF << 21) | (3 << 19) | (1 << 17) | ((0 if crc else 1) << 16) | (br << 12) | (sr << 10) | (pad << 9) | \
        (mode << 6) | (modex << 4)
    return h.to_bytes(4, 'big')


def _side_info_bytes(C, mdb, scfsi, plans):
    w = _Writer()
    w.put(mdb, 9)
    w.put(0, 5 if C == 1 else 3)
    for ch in range(C):
        w.put(scfsi[ch], 4)
    for gr in range(2):
        for ch in range(C):
            p = plans[gr][ch]
            w.put(p.part2_3_length, 12)
            w.put(p.big_values, 9)
            w.put(p.global_gain, 8)
            w.put(p.scalefac_compress, 4)
            w.put(p.window_switching, 1)
            if p.window_switching:
                w.put(p.block_type, 2)
                w.put(p.mixed, 1)
                w.put(p.table_select[0], 5)
                w.put(p.table_select[1], 5)
                for s in p.subblock_gain:
                    w.put(s, 3)
            else:
                for t in p.table_select:
                    w.put(t, 5)
                w.put(p.region0_count, 4)
                w.put(p.region1_count, 3)
            w.put(p.preflag, 1)
            w.put(p.scalefac_scale, 1)
            w.put(p.count1table, 1)
    return w.bytes()


MODES = {'stereo': 0, 'joint': 1, 'dual': 2, 'mono': 3}


def encode(x, rate, bitrate=128, mode=None, crc=False, blocks=None, mixed=False, modex=None, seed=0, opts=None,
           xing=None, id3v2=False, id3v1=False, ape=False, max_begin=511, min_gain=0):
    """float (channels, n) in [-1, 1] -> MPEG-1 Layer III bytes.

    bitrate: kbit/s, or a callable frame -> bitrate index (VBR).  mode: 'mono' / 'stereo' / 'joint' / 'dual'.
    blocks: callable granule -> block type (default: all long).  mixed: callable granule -> bool (for block type 2).
    modex: callable frame -> joint-stereo mode extension (bit 1 MS, bit 0 intensity).  opts: seeded choices:
    'scalefactors' ('zero' / 'random'), 'scfsi', 'preflag', 'scalefac_scale', 'subblock_gain' (bools),
    'cycle_tables' (rotate table_select through every table that can code a region), 'count1' (0, 1 or callable),
    'budget' (callable frame -> fraction of the frame's bits to spend; the rest goes to the reservoir).
    xing: None, 'Xing', 'Info' (with a LAME tag giving the gapless trim) or 'VBRI'.  min_gain: the smallest
    global_gain tried (the finest quantisation)."""
    rng = np.random.default_rng(seed)
    opts = dict(opts or {})
    x = np.asarray(x, np.float64)
    if x.ndim == 1:
        x = x[None]
    C = x.shape[0]
    mode = mode or ('mono' if C == 1 else 'joint')
    mcode = MODES[mode]
    sr = T.RATES.index(rate)
    n = x.shape[1]
    delay = LAG - 529
    F = (n + LAG + FRAME - 1) // FRAME
    G = 2 * F
    sub = np.stack([analyse(np.concatenate([x[c], np.zeros(F * FRAME - n)])) for c in range(C)])   # [C][slots][32]
    sub[:, :, 1::2] *= np.where(np.arange(sub.shape[1]) % 2 == 1, -1.0, 1.0)[None, :, None]
    sub = np.concatenate([np.zeros((C, 18, 32)), sub], axis=1)
    bt_of = blocks or (lambda g: 0)
    mixed_of = mixed if callable(mixed) else (lambda g: bool(mixed))
    modex_of = modex if callable(modex) else (lambda f: (2 if modex is None else modex) if mcode == 1 else 0)
    br_of = bitrate if callable(bitrate) else (lambda f, b=T.BITRATES.index(bitrate): b)
    budget_of = opts.get('budget', lambda f: 1.0)
    frames = []
    md_bytes = bytearray()
    cap_total, written = 0, 0
    rem = 0
    q = 0
    for f in range(F):
        br = br_of(f)
        rem += 144000 * T.BITRATES[br] % rate
        pad = 0
        if rem >= rate:
            rem -= rate
            pad = 1
        flen = 144000 * T.BITRATES[br] // rate + pad
        sil = 17 if C == 1 else 32
        cap = flen - 4 - (2 if crc else 0) - sil
        begin = cap_total - written
        if begin > max_begin:
            md_bytes += bytes(begin - max_begin)
            written += begin - max_begin
            begin = max_begin
        avail = 8 * (begin + cap)
        mx = modex_of(f) if mcode == 1 else 0
        plans = [[None] * C for _ in range(2)]
        scfsi = [0] * C
        w = _Writer()
        spend = int(8 * cap * budget_of(f)) + 8 * begin
        for gr in range(2):
            g = 2 * f + gr
            bt = bt_of(g)
            mx_blk = bool(mixed_of(g)) and bt == 2
            spec = []
            for c in range(C):
                blk = sub[c, 18 * g:18 * g + 36].T
                spec.append(_inverse_antialias(_mdct_granule(blk, bt, mx_blk), bt, mx_blk))
            spec = [_to_bitstream_order(s, bt, mx_blk, sr) for s in spec]
            if mcode == 1 and C == 2:
                if mx & 2:
                    a, b = spec
                    spec = [(a + b) / math.sqrt(2), (a - b) / math.sqrt(2)]
                if mx & 1:   # intensity: the right channel is zero from the upper half of its lines on
                    cut = 288 if bt != 2 else 300
                    spec[0][cut:] = spec[0][cut:] + spec[1][cut:]
                    spec[1][cut:] = 0.0
            for c in range(C):
                p = _Plan()
                p.block_type, p.mixed, p.window_switching = bt, int(mx_blk), 1 if bt else 0
                p.scalefac_scale = int(opts.get('scalefac_scale', False) and rng.random() < 0.5)
                p.preflag = int(opts.get('preflag', False) and bt != 2 and rng.random() < 0.5)
                p.subblock_gain = [int(v) for v in rng.integers(0, 8, 3)] if (opts.get('subblock_gain') and
                                                                               bt == 2) else [0, 0, 0]
                is_right = mcode == 1 and C == 2 and (mx & 1) and c == 1
                if is_right:
                    p.scalefac_compress = 13
                elif opts.get('scalefactors') == 'random':
                    p.scalefac_compress = int(rng.integers(0, 16))
                else:
                    p.scalefac_compress = 0
                s1, s2 = T.SLEN[p.scalefac_compress]
                p.sf_long = [int(rng.integers(0, 1 << (s1 if b < 11 else s2))) if b < 21 else 0 for b in range(22)] \
                    if p.scalefac_compress else [0] * 22
                p.sf_short = [[int(rng.integers(0, 1 << (s1 if b < 6 else s2))) if b < 12 else 0 for _ in range(3)]
                              for b in range(13)] if p.scalefac_compress else [[0] * 3 for _ in range(13)]
                if is_right:
                    p.sf_long = [int(v) for v in rng.integers(0, 8, 22)]
                    p.sf_short = [[int(v) for v in rng.integers(0, 8, 3)] for _ in range(13)]
                    p.sf_long[21], p.sf_short[12] = 0, [0, 0, 0]
                after_short = gr == 1 and opts.get('scfsi_after_short') and bt in (1, 3) and \
                    plans[0][c].block_type == 2
                if gr == 1 and opts.get('scfsi') and ((bt == 0 and plans[0][c].block_type == 0) or after_short):
                    prev = plans[0][c]
                    if prev.scalefac_compress == p.scalefac_compress or after_short:
                        scfsi[c] = int(rng.integers(1, 16))
                        # what the decoder takes for granule 0's long scale factors (_read_scalefactors)
                        shared = [prev.sf_long[b] if prev.block_type != 2 or (prev.mixed and b < 8) else 0
                                  for b in range(22)]
                        for k, (a, b) in enumerate(((0, 6), (6, 11), (11, 16), (16, 21))):
                            if scfsi[c] & (8 >> k):
                                p.sf_long[a:b] = shared[a:b]
                remaining = spend - w.n
                left = (2 - gr) * C - c
                target = min(4095, max(0, remaining // left))
                lo_g, hi_g = min_gain, 255
                best = None
                while lo_g <= hi_g:
                    mid = (lo_g + hi_g) // 2
                    p.global_gain = mid
                    ix, over = _quantise(spec[c], p, sr)
                    bits = _code_granule(ix, p, sr, opts, q) + _sf_bits(p, gr, scfsi[c])
                    if not over and bits <= target:
                        best = mid
                        hi_g = mid - 1
                    else:
                        lo_g = mid + 1
                if best is None:
                    best = 255
                    p.global_gain = 255
                    p.sf_long, p.sf_short = [0] * 22, [[0] * 3 for _ in range(13)]
                    p.preflag, p.subblock_gain, p.scalefac_compress = 0, [0, 0, 0], 0
                    scfsi[c] = 0
                p.global_gain = best
                ix, _ = _quantise(spec[c], p, sr)
                opts['_commit'] = True
                if _code_granule(ix, p, sr, opts, q) + _sf_bits(p, gr, scfsi[c]) > target:
                    ix = np.zeros(576, np.int64)
                    _code_granule(ix, p, sr, opts, q)
                opts['_commit'] = False
                start = w.n
                _write_sf(w, p, gr, scfsi[c])
                _write_granule(w, ix, p)
                # (not the quadruple at lines 572..575: FFmpeg's loop ends there without the check and keeps it)
                if opts.get('cut_quad') and p.regions[2] < p.regions[3] < 576 and opts['cut_quad'](q):
                    w.v >>= 1          # the last quadruple loses its last bit: it crosses the granule's end
                    w.n -= 1
                p.part2_3_length = w.n - start
                plans[gr][c] = p
                q += 1
        body = w.bytes()
        assert len(body) <= begin + cap, (len(body), begin, cap)
        hdr = _header_bytes(br, sr, pad, mcode, mx, crc)
        si = _side_info_bytes(C, begin, scfsi, plans)
        frames.append([hdr, si, cap])
        md_bytes += body
        written += len(body)
        cap_total += cap
    out = bytearray()
    pos = 0
    for hdr, si, cap in frames:
        chunk = bytes(md_bytes[pos:pos + cap])
        chunk += bytes(cap - len(chunk))
        pos += cap
        c = (_crc16(hdr[2:4] + si).to_bytes(2, 'big') if hdr[1] & 1 == 0 else b'')
        out += hdr + c + si + chunk
    if xing:
        out = _xing_frame(xing, frames[0][0], C, F, len(out), delay, F * FRAME - delay - n) + out
    if id3v2:
        tag = b'TIT2\x00\x00\x00\x05\x00\x00\x03' + bytes([0xFF, 0xFB]) + b'\x90\x44'   # a false sync in the tag
        size = len(tag)
        out = b'ID3\x04\x00\x00' + bytes([(size >> 21) & 127, (size >> 14) & 127, (size >> 7) & 127, size & 127]) + \
            tag + out
    if ape:
        items = b'\x05\x00\x00\x00\x00\x00\x00\x00Title\x00' + bytes([0xFF, 0xFB, 0x90, 0x44, 0])
        foot = lambda flags: b'APETAGEX' + (2000).to_bytes(4, 'little') + (len(items) + 32).to_bytes(4, 'little') + \
            (1).to_bytes(4, 'little') + flags.to_bytes(4, 'little') + bytes(8)
        out += foot(0xA0000000) + items + foot(0x80000000)
    if id3v1:
        out += b'TAG' + bytes([0xFF, 0xFB, 0x90]) + bytes(122)
    return bytes(out)


def _xing_frame(kind, hdr, C, frames, nbytes, delay, padding):
    """A first frame with a Xing / Info header and a LAME tag (or a VBRI header), same header as the stream's first."""
    h = parse_header(hdr, 0)
    body = bytearray(frame_length(h) - 4)
    sil = 17 if C == 1 else 32
    if kind == 'VBRI':
        body[32:36] = b'VBRI'
    else:
        o = sil
        body[o:o + 4] = kind.encode()
        body[o + 4:o + 8] = (0x0F).to_bytes(4, 'big')
        body[o + 8:o + 12] = frames.to_bytes(4, 'big')
        body[o + 12:o + 16] = nbytes.to_bytes(4, 'big')
        body[o + 16:o + 116] = bytes(range(0, 200, 2))
        body[o + 116:o + 120] = (50).to_bytes(4, 'big')
        lame = o + 120
        body[lame:lame + 9] = b'LAME3.100'
        body[lame + 21:lame + 24] = ((delay << 12) | padding).to_bytes(3, 'big')
    return _header_bytes(h['br'], h['sr'], h['pad'], h['mode'], h['modex'], False) + bytes(body)


# ------------------------------------------------------------------------------------------------------------- matrix


def sine_mix(n, rate, channels=2, seed=0, amp=0.3):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    out = []
    for c in range(channels):
        f = rng.uniform(80, 5000, 4)
        out.append(sum(amp / 4 * np.sin(2 * np.pi * fi * t + rng.uniform(0, 6.28)) for fi in f))
    return np.stack(out)


def matrix(seed=0):
    """[(name, bytes)] of short streams that together cover the format (tests/test_mp3.py asserts the coverage)."""
    out = []
    x2 = lambda rate, n=FRAME * 6, s=0, amp=0.3: sine_mix(n, rate, 2, seed + s, amp)
    # block types: every transition the standard allows (0 / 3 -> 0 / 1, 1 -> 2, 2 -> 2 / 3)
    cyc = [0, 1, 2, 3, 0, 0, 1, 2, 2, 3, 1, 2, 3, 0]
    out.append(('long_short_mixed_44k_joint_ms_is', encode(x2(44100), 44100, 128, mode='joint',
                                                          blocks=lambda g: cyc[g % len(cyc)],
                                                          mixed=lambda g: g % 2 == 0, modex=lambda f: f % 4,
                                                          opts=dict(scalefactors='random', subblock_gain=True,
                                                                    scalefac_scale=True, preflag=True), seed=seed)))
    out.append(('tables_48k_stereo_crc', encode(x2(48000, s=1, amp=0.02), 48000, 320, mode='stereo', crc=True,
                                                opts=dict(cycle_tables=True, count1=lambda q: q & 1,
                                                          cut_quad=lambda q: q % 3 == 0), seed=seed + 1)))
    out.append(('linbits_32k_dual', encode(x2(32000, s=2, amp=0.9), 32000, 320, mode='dual', seed=seed + 2,
                                           blocks=lambda g: cyc[(g + 5) % len(cyc)], mixed=lambda g: g % 2 == 1,
                                           opts=dict(cycle_tables=True))))
    out.append(('short_mixed_32k_joint_ms_is', encode(x2(32000, s=7), 32000, 96, mode='joint',
                                                     blocks=lambda g: cyc[g % len(cyc)],
                                                     mixed=lambda g: g % 2 == 0, modex=lambda f: 3 - f % 4,
                                                     opts=dict(scalefactors='random', subblock_gain=True),
                                                     seed=seed + 7)))
    out.append(('bitrates_vbr_mono_44k', encode(sine_mix(FRAME * 16, 44100, 1, seed + 3), 44100,
                                                lambda f: 1 + f % 14, mode='mono', seed=seed + 3,
                                                opts=dict(scfsi=True, scalefactors='random'))))
    out.append(('reservoir_44k_stereo', encode(x2(44100, n=FRAME * 12, s=4), 44100, 64, mode='stereo', seed=seed + 4,
                                               opts=dict(budget=lambda f: 0.2 if f % 6 < 4 else 1.0))))
    out.append(('tags_info_lame', encode(x2(44100, s=5), 44100, 128, xing='Info', id3v2=True, id3v1=True, ape=True,
                                         seed=seed + 5)))
    out.append(('xing_vbr_crc_48k', encode(x2(48000, s=6), 48000, lambda f: 9 + f % 3, xing='Xing', crc=True,
                                           blocks=lambda g: cyc[(g + 1) % len(cyc)], mixed=lambda g: g % 2 == 1,
                                           modex=lambda f: f % 4, seed=seed + 6)))
    return out


def scfsi_after_short_stream(seed=0):
    """A stream whose granule 1 shares scale factors by scfsi after a short (and a mixed) granule 0: outside what valid
    encoders write, and decoded by the rule in _read_scalefactors."""
    cyc = [1, 2, 3]
    return encode(sine_mix(FRAME * 12, 44100, 2, seed + 8), 44100, 192, mode='stereo', blocks=lambda g: cyc[g % 3],
                  mixed=lambda g: g % 12 == 4, seed=seed + 8,
                  opts=dict(scfsi=True, scfsi_after_short=True, scalefactors='random'))


def frames_of(d):
    """(frames as bytes list, channels) of a stream by the chain rules, Xing frame included (for FFmpeg)."""
    offs, hdrs, _ = find_frames(d)
    C = 1 if hdrs[0]['mode'] == 3 else 2
    return [d[o:o + frame_length(h)] for o, h in zip(offs, hdrs)], C
