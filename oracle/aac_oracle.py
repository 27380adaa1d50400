"""MPEG-4 AAC-LC in ISO BMFF (.m4a / .mp4) for the tests: a float64 decoder restating ISO/IEC 14496-3 (subpart 4) for
the scope of DESIGN.md §14, a seeded syntax-level encoder, an MP4 writer, and ``matrix()``, the streams that cover it.

Decoder: ``decode(data) -> (float64 (channels, n), rate, info)`` reads the container with lib/aac.py's ``parse`` (the
container tests check that against what ``mp4`` wrote) and ``decode_packets`` does the rest, with the tools in the
standard's order: dequantisation and PNS, M/S on bands where both channels are neither noise nor intensity, intensity,
TNS, then the filterbank (IMDCT, the previous frame's window shape on the left half, overlap-add).  The output is the
standard's, over 32768 (full scale 1), as FFmpeg's float decoder gives it.

PNS noise is a counter-based hash of (packet, channel, window, bin) (``noise``), scaled per window to the energy
``noise_energy`` codes; where both channels of an M/S band are noise, the right channel uses the left's vector.

Encoder: ``encode(x, rate, kbps, plan, seed)`` -> (packets, AudioSpecificConfig).  MDCT analysis with the windows the
frame's plan names, TNS as the FIR inverse of the decoder's filter, M/S, intensity and PNS by band, quantisation
against a bit budget (a binary search on the global scale factor), then section and codebook choice (the cheapest
codebook, or a seeded choice among those that can code the band).
"""
import bisect
import struct

import numpy as np

from . import aac_tables as T

FRAME = 1024
OUT_SCALE = 1.0 / 32768.0
ONLY_LONG, LONG_START, EIGHT_SHORT, LONG_STOP = 0, 1, 2, 3
SCE, CPE, CCE, LFE, DSE, PCE, FIL, END = range(8)
# the standard leaves noise_energy and is_position unbounded; each is clipped to this range before it scales a band, as
# FFmpeg does, so that an extreme but valid value cannot overflow
NOISE_RANGE, IS_RANGE = (-100, 155), (-155, 100)


class Malformed(ValueError):
    pass


# ------------------------------------------------------------------------------------------------------------ tables

def _codebook(b):
    a, e = T.HUFF_START[b], T.HUFF_START[b + 1]
    lens = list(T.HUFF_LENGTHS[a:e])
    starts, code = [], 0
    for ln in lens:
        starts.append(code)
        code += 1 << (32 - ln)
    natural = np.zeros(e - a, np.int64)
    natural[list(T.HUFF_SYMBOLS[a:e])] = lens
    codes = np.zeros(e - a, np.int64)
    codes[list(T.HUFF_SYMBOLS[a:e])] = [s >> (32 - ln) for s, ln in zip(starts, lens)]
    return dict(starts=starts, lens=lens, syms=list(T.HUFF_SYMBOLS[a:e]), len_of=natural, code_of=codes)


BOOKS = [_codebook(b) for b in range(12)]


def noise(packet, channel, window, bins):
    """PNS source: uniform in [-1, 1) from a 32-bit hash of (packet, channel, window, bin); bins: int array."""
    m = 0xFFFFFFFF
    h = ((packet * 0x9E3779B1) ^ ((channel * 8 + window) * 0x85EBCA77)) & m
    x = (np.asarray(bins, np.uint64) * np.uint64(0xC2B2AE3D) ^ np.uint64(h)) & np.uint64(m)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x85EBCA6B)) & np.uint64(m)
    x ^= x >> np.uint64(13)
    x = (x * np.uint64(0xC2B2AE35)) & np.uint64(m)
    x ^= x >> np.uint64(16)
    return x.astype(np.uint32).view(np.int32).astype(np.float64) / 2.0 ** 31


def tns_lpc(parcor):
    """The standard's step-up from reflection to direct-form coefficients a[1..order]."""
    a = np.zeros(len(parcor) + 1)
    a[0] = 1.0
    for m in range(1, len(parcor) + 1):
        b = a.copy()
        for i in range(1, m):
            b[i] = a[i] + parcor[m - 1] * a[m - i]
        a = b
        a[m] = parcor[m - 1]
    return a[1:]


def tns_coef_value(raw, res_bits, compress):
    w = res_bits - compress
    v = raw - (1 << w) if raw >= (1 << (w - 1)) else raw
    return (T.TNS_COEF_3 if res_bits == 3 else T.TNS_COEF_4)[v + (1 << (res_bits - 1))]


def tns_range(swb, num_swb, max_sfb, max_bands, top_band, length):
    bottom = max(top_band - length, 0)
    mmm = min(max_bands, max_sfb)
    return swb[min(bottom, mmm)], swb[min(top_band, mmm)], bottom


_COS = {}


def _cos(N):
    if N not in _COS:
        n = np.arange(N)[:, None] + (N / 2 + 1) / 2.0
        k = np.arange(N // 2)[None, :] + 0.5
        _COS[N] = np.cos(2 * np.pi / N * n * k)
    return _COS[N]


def imdct(X):
    N = 2 * len(X)
    return (2.0 / N) * (_cos(N) @ X)


def mdct(z):
    return 2.0 * (_cos(len(z)).T @ z)


def frame_window(ws, shape, prev_shape):
    """The 2048-point window of a long, start or stop frame; for EIGHT_SHORT the (8, 256) windows."""
    L, S = T.WINDOW_LONG, T.WINDOW_SHORT
    if ws == EIGHT_SHORT:
        w = np.empty((8, 256))
        for j in range(8):
            w[j, :128] = S[prev_shape if j == 0 else shape]
            w[j, 128:] = S[shape][::-1]
        return w
    w = np.zeros(2048)
    if ws == LONG_STOP:
        w[448:576] = S[prev_shape]
        w[576:1024] = 1.0
    else:
        w[:1024] = L[prev_shape]
    if ws == LONG_START:
        w[1024:1472] = 1.0
        w[1472:1600] = S[shape][::-1]
    else:
        w[1024:] = L[shape][::-1]
    return w


def synthesis(spec, ws, shape, prev_shape):
    """Windowed IMDCT of one frame's spectrum -> 2048 samples (standard scale)."""
    w = frame_window(ws, shape, prev_shape)
    if ws != EIGHT_SHORT:
        return imdct(spec) * w
    z = np.zeros(2048)
    for j in range(8):
        z[448 + 128 * j:704 + 128 * j] += imdct(spec[128 * j:128 * (j + 1)]) * w[j]
    return z


def analysis(z, ws, shape, prev_shape):
    """Forward MDCT of 2048 samples with the frame's windows -> 1024 coefficients (short: 8 x 128, window-major).
    Inverts ``synthesis`` under overlap-add (time-domain aliasing cancellation)."""
    w = frame_window(ws, shape, prev_shape)
    if ws != EIGHT_SHORT:
        return mdct(z * w)
    return np.concatenate([mdct(z[448 + 128 * j:704 + 128 * j] * w[j]) for j in range(8)])


def frame_spectra(y, frames):
    """The spectrum of each frame but the last recovered from a decoder's output y ((channels, n) at full scale 1,
    untrimmed) by ``analysis`` with that frame's windows: frames is decode_packets' per-frame list."""
    out = []
    for k in range(len(frames) - 1):
        row = []
        for c, f in enumerate(frames[k]['ics']):
            z = y[c, k * FRAME:k * FRAME + 2 * FRAME] / OUT_SCALE
            row.append(analysis(z, f['ws'], f['shape'], f['prev_shape']))
        out.append(row)
    return out


# ------------------------------------------------------------------------------------------------------------ decoder

class BitReader(object):
    def __init__(self, data, packet=0, offset=0):
        self.v = int.from_bytes(bytes(data) + b'\0\0\0\0', 'big')
        self.n = 8 * len(data)
        self.total = 8 * len(data) + 32
        self.pos = 0
        self.packet, self.offset = packet, offset

    def fail(self, why, bit=None):
        raise Malformed('packet %d (byte %d): %s (bit %d)' % (self.packet, self.offset, why,
                                                              self.pos if bit is None else bit))

    def peek32(self):
        return (self.v >> (self.total - self.pos - 32)) & 0xFFFFFFFF

    def read(self, k):
        if k == 0:
            return 0
        if self.pos + k > self.n:
            self.fail('the bits run past the end of the packet')
        v = (self.v >> (self.total - self.pos - k)) & ((1 << k) - 1)
        self.pos += k
        return v

    def huff(self, b):
        bk = BOOKS[b]
        i = bisect.bisect_right(bk['starts'], self.peek32()) - 1
        self.read(bk['lens'][i])
        return bk['syms'][i]


def new_stats():
    return dict(rates=set(), channels=set(), codebooks=set(), ws=set(), ws_pairs=set(), shapes=set(), groupings=set(),
                pulse=0, tns=set(), ms=set(), is_cb=set(), is_inverted=0, pns=0, pns_ms=0, esc_long=0, fil=0, dse=0,
                common_window=set())


def read_ics_info(br, sfi):
    if br.read(1):
        br.fail('ics_reserved_bit is set', br.pos - 1)
    info = dict(ws=br.read(2), shape=br.read(1))
    if info['ws'] == EIGHT_SHORT:
        info['max_sfb'] = br.read(4)
        grouping = br.read(7)
        lens = [1]
        for i in range(7):
            if grouping & (1 << (6 - i)):
                lens[-1] += 1
            else:
                lens.append(1)
        info['group_len'] = lens
        info['grouping'] = grouping
        swb = T.SWB_SHORT[sfi]
    else:
        info['max_sfb'] = br.read(6)
        if br.read(1):
            br.fail('predictor_data_present is set: Main-profile or LTP prediction is not AAC-LC', br.pos - 1)
        info['group_len'] = [1]
        info['grouping'] = 0
        swb = T.SWB_LONG[sfi]
    info['swb'] = swb
    if info['max_sfb'] > len(swb) - 1:
        br.fail('max_sfb %d is above the %d scale-factor bands' % (info['max_sfb'], len(swb) - 1))
    return info


def read_ics(br, sfi, info, st, ms=None):
    gg = br.read(8)
    if info is None:
        info = read_ics_info(br, sfi)
    info = dict(info)
    short = info['ws'] == EIGHT_SHORT
    swb, max_sfb = info['swb'], info['max_sfb']
    G = len(info['group_len'])
    cb = np.zeros((G, max(max_sfb, 1)), np.int64)
    sbits = 3 if short else 5
    esc = (1 << sbits) - 1
    for g in range(G):
        k = 0
        while k < max_sfb:
            c = br.read(4)
            if c == 12:
                br.fail('reserved section codebook 12', br.pos - 4)
            n = 0
            while True:
                inc = br.read(sbits)
                n += inc
                if inc != esc:
                    break
            if k + n > max_sfb:
                br.fail('a section runs past max_sfb')
            cb[g, k:k + n] = c
            k += n
    sf = np.zeros_like(cb)
    scale, is_pos, nrg, first_noise = gg, 0, gg - 90, True
    for g in range(G):
        for b in range(max_sfb):
            c = cb[g, b]
            if c == 0:
                continue
            if c in (14, 15):
                d = br.huff(0) - 60
                is_pos += d
                sf[g, b] = is_pos
            elif c == 13:
                if first_noise:
                    nrg += br.read(9) - 256
                    first_noise = False
                else:
                    d = br.huff(0) - 60
                    nrg += d
                sf[g, b] = nrg
            else:
                d = br.huff(0) - 60
                scale += d
                if scale < 0 or scale > 255:
                    br.fail('a scale factor leaves [0, 255]')
                sf[g, b] = scale
    pulse = None
    if br.read(1):
        if short:
            br.fail('pulse data in an EIGHT_SHORT frame', br.pos - 1)
        npulse = br.read(2) + 1
        start = br.read(6)
        if start >= len(swb) - 1:
            br.fail('pulse_start_sfb is past the last band', br.pos - 6)
        pos = swb[start]
        pulse = []
        for _ in range(npulse):
            pos += br.read(5)
            amp = br.read(4)
            if pos >= 1024:
                br.fail('a pulse lies past the spectrum')
            pulse.append((pos, amp))
    tns = None
    if br.read(1):
        tns = []
        for w in range(8 if short else 1):
            nf = br.read(1 if short else 2)
            filters = []
            res = br.read(1) + 3 if nf else 3
            for _ in range(nf):
                length = br.read(4 if short else 6)
                order = br.read(3 if short else 5)
                if order > (T.TNS_MAX_ORDER_SHORT if short else T.TNS_MAX_ORDER_LONG):
                    br.fail('TNS order %d above the maximum' % order, br.pos - 5)
                d = comp = 0
                coefs = []
                if order:
                    d = br.read(1)
                    comp = br.read(1)
                    coefs = [tns_coef_value(br.read(res - comp), res, comp) for _ in range(order)]
                    st['tns'].add(('short' if short else 'long', res, comp))
                filters.append(dict(length=length, order=order, direction=d, coefs=coefs))
            tns.append(filters)
    if br.read(1):
        br.fail('gain_control_data_present is set: AAC SSR is not AAC-LC', br.pos - 1)
    q = np.zeros(1024, np.int64)
    g0 = 0
    for g in range(G):
        for b in range(max_sfb):
            c = int(cb[g, b])
            if c == 0 or c >= 13:
                continue
            st['codebooks'].add(c)
            dim, signed, mod = T.SPECTRAL_CODEBOOKS[c]
            for w in range(g0, g0 + info['group_len'][g]):
                k, e = 128 * w + swb[b], 128 * w + swb[b + 1]
                while k < e:
                    s = br.huff(c)
                    vals = []
                    for _ in range(dim):
                        vals.append(s % mod)
                        s //= mod
                    vals = vals[::-1]
                    if signed:
                        vals = [v - mod // 2 for v in vals]
                    else:
                        vals = [-v if v and br.read(1) else v for v in vals]
                        if c == 11:
                            for i, v in enumerate(vals):
                                if abs(v) == 16:
                                    n = 0
                                    while br.read(1):
                                        n += 1
                                    if n > 8:
                                        br.fail('an escape sequence is longer than 13 bits')
                                    vals[i] = (1 if v > 0 else -1) * ((1 << (n + 4)) + br.read(n + 4))
                                    if not short:
                                        st['esc_long'] += 1
                    q[k:k + dim] = vals
                    k += dim
        g0 += info['group_len'][g]
    st['codebooks'].update(int(c) for c in cb[:, :max_sfb].ravel())
    if pulse:
        st['pulse'] += 1
        for pos, amp in pulse:
            q[pos] = q[pos] + amp if q[pos] > 0 else q[pos] - amp
    info.update(cb=cb, sf=sf, q=q, tns=tns, global_gain=gg, pulse=pulse)
    return info


def parse_packet(data, sfi, C, packet=0, offset=0, st=None):
    """One raw_data_block -> (list of per-channel ICS dicts, M/S dict or None)."""
    st = new_stats() if st is None else st
    br = BitReader(data, packet, offset)
    chans, ms = [], None
    while True:
        at = br.pos
        el = br.read(3)
        if el == END:
            break
        if el in (SCE, CPE):
            if chans or (el == SCE) != (C == 1):
                br.fail('%s does not match the channel configuration' % ('an SCE' if el == SCE else 'a CPE'), at)
            br.read(4)
            if el == SCE:
                chans = [read_ics(br, sfi, None, st)]
                continue
            cw = br.read(1)
            st['common_window'].add(cw)
            info, msp, used = None, 0, None
            if cw:
                info = read_ics_info(br, sfi)
                msp = br.read(2)
                if msp == 3:
                    br.fail('reserved ms_mask_present 3', br.pos - 2)
                G = len(info['group_len'])
                used = np.zeros((G, max(info['max_sfb'], 1)), np.int64)
                if msp == 1:
                    for g in range(G):
                        for b in range(info['max_sfb']):
                            used[g, b] = br.read(1)
                elif msp == 2:
                    used[:] = 1
                st['ms'].add(msp)
            chans = [read_ics(br, sfi, info, st), read_ics(br, sfi, info, st)]
            ms = dict(common=cw, present=msp, used=used)
        elif el == DSE:
            br.read(4)
            align = br.read(1)
            n = br.read(8)
            if n == 255:
                n += br.read(8)
            if align and br.pos % 8:
                br.read(8 - br.pos % 8)
            br.read(8 * n) if n else None
            st['dse'] += 1
        elif el == FIL:
            n = br.read(4)
            if n == 15:
                n += br.read(8) - 1
            if n:
                typ = br.read(4)
                if typ in (13, 14):
                    br.fail('an SBR extension payload in a FIL element (HE-AAC, implicit signalling) is not '
                            'supported', br.pos - 4)
                br.read(8 * n - 4)
            st['fil'] += 1
        else:
            br.fail({CCE: 'a CCE element (coupling channel) is not supported',
                     LFE: 'an LFE element is not supported',
                     PCE: 'a PCE element (program config) is not supported'}[el], at)
    if not chans:
        br.fail('no channel element before END')
    return chans, ms


def _windows_of(ics):
    """(window, group, first bin of window) for each of the frame's windows."""
    out, w = [], 0
    for g, n in enumerate(ics['group_len']):
        for _ in range(n):
            out.append((w, g))
            w += 1
    return out


def spectral(chans, ms, sfi, packet, st):
    """Dequantisation, PNS, M/S, intensity, TNS -> (C, 1024) float64 spectra (standard scale)."""
    C = len(chans)
    spec = np.zeros((C, 1024))
    for c, ics in enumerate(chans):
        swb = ics['swb']
        for w, g in _windows_of(ics):
            for b in range(ics['max_sfb']):
                cbv = ics['cb'][g, b]
                a, e = 128 * w + swb[b], 128 * w + swb[b + 1]
                if 1 <= cbv <= 11:
                    q = ics['q'][a:e].astype(np.float64)
                    spec[c, a:e] = np.sign(q) * np.abs(q) ** (4.0 / 3.0) * 2.0 ** (0.25 * (ics['sf'][g, b] - 100))
                elif cbv == 13:
                    src = c
                    if c == 1 and ms and ms['present'] and ms['used'][g, b] and chans[0]['cb'][g, b] == 13:
                        src = 0
                        st['pns_ms'] += 1
                    r = noise(packet, src, w, np.arange(a, e) - 128 * w)
                    nrg = np.clip(ics['sf'][g, b], *NOISE_RANGE)
                    spec[c, a:e] = r * 2.0 ** (0.25 * nrg) / np.sqrt(np.sum(r * r))
                    st['pns'] += 1
    if ms and ms['common']:
        L, R = chans
        for w, g in _windows_of(L):
            for b in range(L['max_sfb']):
                a, e = 128 * w + L['swb'][b], 128 * w + L['swb'][b + 1]
                if ms['present'] and ms['used'][g, b] and L['cb'][g, b] < 13 and R['cb'][g, b] < 13:
                    m, s = spec[0, a:e].copy(), spec[1, a:e].copy()
                    spec[0, a:e], spec[1, a:e] = m + s, m - s
                if R['cb'][g, b] in (14, 15):
                    sign = 1.0 if R['cb'][g, b] == 15 else -1.0
                    st['is_cb'].add(int(R['cb'][g, b]))
                    if ms['present'] == 1 and ms['used'][g, b]:
                        sign = -sign
                        st['is_inverted'] += 1
                    spec[1, a:e] = spec[0, a:e] * sign * 0.5 ** (0.25 * np.clip(R['sf'][g, b], *IS_RANGE))
    for c, ics in enumerate(chans):
        if not ics['tns']:
            continue
        short = ics['ws'] == EIGHT_SHORT
        num_swb = len(ics['swb']) - 1
        maxb = (T.TNS_MAX_BANDS_SHORT if short else T.TNS_MAX_BANDS_LONG)[sfi]
        for w, filters in enumerate(ics['tns']):
            top = num_swb
            for f in filters:
                start, end, top = tns_range(ics['swb'], num_swb, ics['max_sfb'], maxb, top, f['length'])
                if not f['order'] or end <= start:
                    continue
                a = tns_lpc(f['coefs'])
                x = spec[c, 128 * w + start:128 * w + end]
                idx = range(len(x) - 1, -1, -1) if f['direction'] else range(len(x))
                y = x.copy()
                hist = []
                for i in idx:
                    v = x[i] - sum(a[j] * hist[-1 - j] for j in range(min(len(hist), len(a))))
                    y[i] = v
                    hist.append(v)
                spec[c, 128 * w + start:128 * w + end] = y
    return spec


def decode_packets(packets, sfi, C, offsets=None, st=None):
    """Raw AAC-LC packets -> (float64 (C, len(packets) * 1024) at full scale 1, per-frame list of what was decoded)."""
    st = new_stats() if st is None else st
    st['rates'].add(sfi)
    st['channels'].add(C)
    F = len(packets)
    out = np.zeros((C, F * FRAME))
    tail = np.zeros((C, FRAME))
    prev_shape = [0] * C
    prev_ws = [ONLY_LONG] * C
    frames = []
    for p, pkt in enumerate(packets):
        chans, ms = parse_packet(pkt, sfi, C, p, 0 if offsets is None else int(offsets[p]), st)
        spec = spectral(chans, ms, sfi, p, st)
        rec = []
        for c, ics in enumerate(chans):
            z = synthesis(spec[c], ics['ws'], ics['shape'], prev_shape[c])
            out[c, p * FRAME:(p + 1) * FRAME] = z[:FRAME] + tail[c]
            tail[c] = z[FRAME:]
            st['ws'].add(ics['ws'])
            st['ws_pairs'].add((prev_ws[c], ics['ws']))
            st['shapes'].add((prev_shape[c], ics['shape']))
            if ics['ws'] == EIGHT_SHORT:
                st['groupings'].add(len(ics['group_len']))
            rec.append(dict(ws=ics['ws'], shape=ics['shape'], prev_shape=prev_shape[c], cb=ics['cb'],
                            group_len=ics['group_len'], swb=ics['swb'], max_sfb=ics['max_sfb'], sf=ics['sf'],
                            tns=bool(ics['tns'])))
            prev_shape[c], prev_ws[c] = ics['shape'], ics['ws']
        frames.append(dict(ics=rec, spec=spec, ms=ms))
    return out * OUT_SCALE, frames


def decode(data, stats=None):
    """An .m4a / .mp4 file's bytes -> (float64 (channels, n), rate, info) with the edit list's trim applied."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'vocal-remover_b200'))
    from lib import aac
    t = aac.parse(data)
    packets = [bytes(data[o:o + s]) for o, s in zip(t['offsets'], t['sizes'])]
    y, frames = decode_packets(packets, t['rate_index'], t['channels'], t['offsets'], stats)
    a, b = aac.trim_range(len(packets) * FRAME, t)
    info = dict(frames=len(packets), priming=a, kept=b - a, fragmented=t['fragmented'])
    return y[:, a:b], t['rate'], info


# ------------------------------------------------------------------------------------------------------------ encoder

class BitWriter(object):
    def __init__(self):
        self.v, self.n = 0, 0

    def write(self, value, k):
        if k:
            assert 0 <= value < (1 << k), (value, k)
            self.v = (self.v << k) | value
            self.n += k

    def huff(self, b, sym):
        self.write(int(BOOKS[b]['code_of'][sym]), int(BOOKS[b]['len_of'][sym]))

    def align(self):
        if self.n % 8:
            self.write(0, 8 - self.n % 8)

    def bytes(self):
        self.align()
        return self.v.to_bytes(self.n // 8, 'big')


def _symbols(vals, c):
    dim, signed, mod = T.SPECTRAL_CODEBOOKS[c]
    v = np.asarray(vals, np.int64).reshape(-1, dim)
    u = v + mod // 2 if signed else np.minimum(np.abs(v), 16)
    s = np.zeros(len(v), np.int64)
    for i in range(dim):
        s = s * mod + u[:, i]
    return s, v


def band_bits(vals, c):
    """Bits of a band's values in spectral codebook c (vals fit c)."""
    s, v = _symbols(vals, c)
    bits = int(BOOKS[c]['len_of'][s].sum())
    if not T.SPECTRAL_CODEBOOKS[c][1]:
        a = np.abs(v)
        bits += int((a > 0).sum())
        if c == 11:
            big = a[a >= 16]
            n = np.floor(np.log2(big)).astype(np.int64) - 4
            bits += int((2 * n + 5).sum())
    return bits


def fits(c, m):
    return m <= {1: 1, 2: 1, 3: 2, 4: 2, 5: 4, 6: 4, 7: 7, 8: 7, 9: 12, 10: 12, 11: 8191}[c]


def write_values(bw, vals, c):
    s, v = _symbols(vals, c)
    signed = T.SPECTRAL_CODEBOOKS[c][1]
    for sym, row in zip(s.tolist(), v.tolist()):
        bw.huff(c, sym)
        if signed:
            continue
        for x in row:
            if x:
                bw.write(1 if x < 0 else 0, 1)
        if c == 11:
            for x in row:
                a = abs(x)
                if a >= 16:
                    n = a.bit_length() - 5
                    bw.write((1 << (n + 1)) - 2, n + 1)   # n ones, then a zero
                    bw.write(a - (1 << (n + 4)), n + 4)


def quantise(X, sf):
    q = np.floor((np.abs(X) * 2.0 ** (-0.25 * (sf - 100))) ** 0.75 + 0.4054)
    return (np.sign(X) * np.minimum(q, 8191)).astype(np.int64)


def _bands(ws, sfi, group_len):
    """[(group, band, bin indices in coding order)] of a frame layout."""
    short = ws == EIGHT_SHORT
    swb = T.SWB_SHORT[sfi] if short else T.SWB_LONG[sfi]
    out, w0 = [], 0
    for g, n in enumerate(group_len):
        for b in range(len(swb) - 1):
            idx = np.concatenate([np.arange(128 * w + swb[b], 128 * w + swb[b + 1]) for w in range(w0, w0 + n)])
            out.append((g, b, idx))
        w0 += n
    return out, swb


def _group_len(grouping):
    lens = [1]
    for i in range(7):
        if grouping & (1 << (6 - i)):
            lens[-1] += 1
        else:
            lens.append(1)
    return lens


def _choose(vals, rng, mode):
    m = int(np.abs(vals).max()) if len(vals) else 0
    if m == 0 and (mode != 'random' or rng.random() < 0.7):   # noqa: SIM114
        return 0
    cands = [c for c in range(1, 12) if fits(c, m)]
    if mode == 'fast':
        return cands[0]
    if mode == 'random':
        return int(rng.choice(cands))
    return min(cands, key=lambda c: band_bits(vals, c))


def _tns_plan(rng, short, sfi, max_sfb):
    """Random stable TNS filters per window: [(length, order, direction, res, compress, raw codes)]."""
    num_swb = len((T.SWB_SHORT if short else T.SWB_LONG)[sfi]) - 1
    plan = []
    for w in range(8 if short else 1):
        filters = []
        nf = (int(rng.random() < 0.7) if short else int(rng.integers(1, 3)))
        res = int(rng.integers(3, 5))
        for _ in range(nf):
            length = int(rng.integers(1, (16 if short else 64)))
            order = int(rng.integers(0, (8 if short else 13)))
            comp = int(rng.integers(0, 2))
            lo = -(1 << (res - comp - 1))
            vals = rng.integers(max(lo, -2), min(-lo, 3), size=order)
            filters.append((length, order, int(rng.integers(0, 2)), res, comp, [int(v) for v in vals]))
        plan.append((res, filters))
    return plan


def _apply_tns_fir(X, plan, sfi, max_sfb, short):
    swb = (T.SWB_SHORT if short else T.SWB_LONG)[sfi]
    num_swb = len(swb) - 1
    maxb = (T.TNS_MAX_BANDS_SHORT if short else T.TNS_MAX_BANDS_LONG)[sfi]
    X = X.copy()
    for w, (res, filters) in enumerate(plan):
        top = num_swb
        for length, order, d, _, comp, vals in filters:
            start, end, top = tns_range(swb, num_swb, max_sfb, maxb, top, length)
            if not order or end <= start:
                continue
            a = tns_lpc([T.TNS_COEF_3[v + 4] if res == 3 else T.TNS_COEF_4[v + 8] for v in vals])
            x = X[128 * w + start:128 * w + end]
            xs = x[::-1] if d else x
            e = xs.copy()
            for j in range(1, order + 1):
                e[j:] += a[j - 1] * xs[:-j]
            X[128 * w + start:128 * w + end] = e[::-1] if d else e
    return X


def _write_tns(bw, plan, short):
    for res, filters in plan:
        bw.write(len(filters), 1 if short else 2)
        if filters:
            bw.write(res - 3, 1)
        for length, order, d, _, comp, vals in filters:
            bw.write(length, 4 if short else 6)
            bw.write(order, 3 if short else 5)
            if order:
                bw.write(d, 1)
                bw.write(comp, 1)
                wd = res - comp
                for v in vals:
                    bw.write(v & ((1 << wd) - 1), wd)


def _ics_info(bw, fr, max_sfb):
    bw.write(0, 1)
    bw.write(fr['ws'], 2)
    bw.write(fr['shape'], 1)
    if fr['ws'] == EIGHT_SHORT:
        bw.write(max_sfb, 4)
        bw.write(fr['grouping'], 7)
    else:
        bw.write(max_sfb, 6)
        bw.write(0, 1)


def _channel(X, fr, sfi, g, kinds, rng, mode, max_sfb):
    """Quantise one channel: -> dict(cb, sf, q) over the frame's bands (q in coding order per band)."""
    bands, swb = _bands(fr['ws'], sfi, fr['group_len'])
    cbs, sfs, qs = {}, {}, {}
    jitter = fr.get('jitter', 0)
    for gi, b, idx in bands:
        if b >= max_sfb:
            continue
        kind = kinds.get((gi, b), 'reg')
        if kind == 'noise':
            nwin = fr['group_len'][gi]
            e = np.sum(X[idx] ** 2) / nwin
            cbs[gi, b], sfs[gi, b], qs[gi, b] = 13, int(np.clip(round(2 * np.log2(max(e, 1e-3))), -100, 155)), None
            continue
        if kind in ('is+', 'is-'):
            cbs[gi, b], sfs[gi, b], qs[gi, b] = kinds[(gi, b, 'cb')], kinds[(gi, b, 'pos')], None
            continue
        sf = int(np.clip(g + (rng.integers(-jitter, jitter + 1) if jitter else 0), 0, 255))
        q = quantise(X[idx], sf)
        cbs[gi, b], sfs[gi, b], qs[gi, b] = _choose(q, rng, mode), sf, q
    return dict(cb=cbs, sf=sfs, q=qs)


def _chan_bits(ch):
    return sum(band_bits(q, c) for (k, c), q in zip(ch['cb'].items(), ch['q'].values()) if c and c < 13 and q is not None)


def _write_ics(bw, ch, fr, sfi, max_sfb, common, pulse=None, tns=None):
    short = fr['ws'] == EIGHT_SHORT
    G = len(fr['group_len'])
    regular = [ch['sf'][k] for k in sorted(ch['cb']) if 0 < ch['cb'][k] < 13]
    gg = regular[0] if regular else 100
    bw.write(gg, 8)
    if not common:
        _ics_info(bw, fr, max_sfb)
    sbits = 3 if short else 5
    esc = (1 << sbits) - 1
    splits = fr.get('split_sections', False)
    for gi in range(G):
        b = 0
        while b < max_sfb:
            c = ch['cb'][gi, b]
            n = 1
            while b + n < max_sfb and ch['cb'][gi, b + n] == c and not (splits and n >= 2):
                n += 1
            bw.write(c, 4)
            k = n
            while k >= esc:
                bw.write(esc, sbits)
                k -= esc
            bw.write(k, sbits)
            b += n
    scale, is_pos, nrg, first = gg, 0, gg - 90, True
    for gi in range(G):
        for b in range(max_sfb):
            c = ch['cb'][gi, b]
            if c == 0:
                continue
            v = ch['sf'][gi, b]
            if c in (14, 15):
                bw.huff(0, v - is_pos + 60)
                is_pos = v
            elif c == 13:
                if first:
                    v = int(np.clip(v, nrg - 256, nrg + 255))
                    bw.write(v - nrg + 256, 9)
                    first = False
                else:
                    v = int(np.clip(v, nrg - 60, nrg + 60))
                    bw.huff(0, v - nrg + 60)
                nrg = v
            else:
                d = int(np.clip(v - scale, -60, 60))
                bw.huff(0, d + 60)
                scale += d
                if scale != v:   # a clipped step: requantise the band at the scale factor reached
                    raise AssertionError('scale-factor step out of range')
    if pulse:
        bw.write(1, 1)
        start, plist = pulse
        bw.write(len(plist) - 1, 2)
        bw.write(start, 6)
        for off, amp in plist:
            bw.write(off, 5)
            bw.write(amp, 4)
    else:
        bw.write(0, 1)
    if tns:
        bw.write(1, 1)
        _write_tns(bw, tns, short)
    else:
        bw.write(0, 1)
    bw.write(0, 1)   # gain_control_data_present
    for gi in range(G):
        for b in range(max_sfb):
            c = ch['cb'][gi, b]
            if 0 < c < 13:
                write_values(bw, ch['q'][gi, b], c)


def _pulses(ch, fr, sfi):
    """Move up to four pulse amplitudes of the first band with |q| >= 2 out of q into pulse data."""
    swb = T.SWB_LONG[sfi]
    for (gi, b), q in sorted(ch['q'].items()):
        if q is None or not (0 < ch['cb'][gi, b] < 13):
            continue
        pos = [int(i) for i in np.flatnonzero(np.abs(q) >= 2)]
        if not pos or pos[0] > 31:
            continue
        plist, last = [], 0
        for p in pos:
            if p - last > 31 or len(plist) == 4:
                break
            amp = int(min(abs(q[p]) - 1, 15))
            plist.append((p - last, amp))
            last = p
            q[p] -= amp if q[p] > 0 else -amp
        m = int(np.abs(q).max())
        if not fits(ch['cb'][gi, b], m) or ch['cb'][gi, b] == 0:
            ch['cb'][gi, b] = 11
        return b, plist
    return None


def encode(x, rate, kbps=128, plan=None, seed=0, pad_to=None):
    """x: float (channels, n) at full scale 1 -> (list of raw_data_block packets, AudioSpecificConfig bytes).

    plan(k, rng, prev) -> the frame's dict: ws, shape, grouping (EIGHT_SHORT), ms (0, 1, 2; stereo), common (stereo),
    is_bands, pns_bands (number of top bands), tns, pulse, esc (finer quantisation), cb ('best' or 'random'), jitter,
    split_sections, fill / dse (extra elements).  Without a plan every frame is ONLY_LONG, sine, cheapest codebooks.
    pad_to: fill every packet to that many bytes with a FIL element (constant-size samples)."""
    x = np.asarray(x, np.float64)
    C, n = x.shape
    sfi = T.RATES.index(rate)
    F = -(-(n + FRAME) // FRAME)
    s = np.zeros((C, (F + 1) * FRAME))
    s[:, FRAME:FRAME + n] = x * 32768.0
    rng = np.random.default_rng(seed)
    budget = kbps * 1000 * FRAME // rate
    packets, prev, prev_shape = [], dict(ws=ONLY_LONG, shape=0), 0
    for k in range(F):
        fr = dict(ws=ONLY_LONG, shape=0, grouping=0, ms=1 if C == 2 else 0, common=1, cb='best')
        if plan is not None:
            fr.update(plan(k, rng, prev))
        fr['group_len'] = _group_len(fr['grouping']) if fr['ws'] == EIGHT_SHORT else [1]
        short = fr['ws'] == EIGHT_SHORT
        swb = (T.SWB_SHORT if short else T.SWB_LONG)[sfi]
        num_swb = len(swb) - 1
        max_sfb = fr.get('max_sfb', num_swb)
        X = np.stack([analysis(s[c, k * FRAME:k * FRAME + 2 * FRAME], fr['ws'], fr['shape'], prev_shape)
                      for c in range(C)])
        tns = [_tns_plan(rng, short, sfi, max_sfb) if fr.get('tns') else None for _ in range(C)]
        X = np.stack([_apply_tns_fir(X[c], tns[c], sfi, max_sfb, short) if tns[c] else X[c] for c in range(C)])
        bands, _ = _bands(fr['ws'], sfi, fr['group_len'])
        kinds = [dict() for _ in range(C)]
        G = len(fr['group_len'])
        used = np.zeros((G, max(max_sfb, 1)), np.int64)
        if C == 2 and fr['common']:
            if fr['ms'] == 2:
                used[:] = 1
            elif fr['ms'] == 1:
                used[:] = rng.integers(0, 2, size=used.shape)
        n_is, n_pns = fr.get('is_bands', 0), fr.get('pns_bands', 0)
        for gi, b, idx in bands:
            if b >= max_sfb:
                continue
            if n_pns and b >= max_sfb - n_pns:
                for c in range(C):
                    kinds[c][gi, b] = 'noise'
                if C == 2 and fr['ms'] == 1 and b % 2:
                    used[gi, b] = 1   # both channels noise in an M/S band: one noise vector
            elif C == 2 and fr['common'] and n_is and max_sfb - n_pns - n_is <= b < max_sfb - n_pns:
                el, er = np.sum(X[0, idx] ** 2) + 1e-9, np.sum(X[1, idx] ** 2) + 1e-9
                pos = int(np.clip(round(2 * np.log2(el / er)), -20, 20))
                want = 1 if (b % 2 or np.dot(X[0, idx], X[1, idx]) >= 0) else -1
                inv = -1 if fr['ms'] == 1 and used[gi, b] else 1
                kinds[1][gi, b] = 'is+'
                kinds[1][gi, b, 'cb'] = 15 if want * inv > 0 else 14
                kinds[1][gi, b, 'pos'] = pos
            elif C == 2 and used[gi, b]:
                L, R = X[0, idx].copy(), X[1, idx].copy()
                X[0, idx], X[1, idx] = (L + R) / 2, (L - R) / 2
        lo, hi = 0, 255
        mode = fr.get('cb', 'best')
        while lo < hi:   # the finest global scale factor whose frame fits the budget
            mid = (lo + hi) // 2
            bits = sum(_chan_bits(_channel(X[c], dict(fr, jitter=0), sfi, mid, kinds[c], None, 'fast',
                                           max_sfb)) for c in range(C))
            if bits + 60 * C + 40 <= budget:
                hi = mid
            else:
                lo = mid + 1
        g = max(lo - (24 if fr.get('esc') else 0), 0)
        chans = [_channel(X[c], fr, sfi, g, kinds[c], rng, mode, max_sfb) for c in range(C)]
        pulses = [None] * C
        if fr.get('pulse') and not short:
            pulses[0] = _pulses(chans[0], fr, sfi)
        bw = BitWriter()
        if fr.get('dse'):
            bw.write(DSE, 3)
            bw.write(0, 4)
            bw.write(1, 1)
            bw.write(3, 8)
            bw.align()
            bw.write(0xABCDEF, 24)
        if C == 1:
            bw.write(SCE, 3)
            bw.write(0, 4)
            _write_ics(bw, chans[0], fr, sfi, max_sfb, False, pulses[0], tns[0])
        else:
            bw.write(CPE, 3)
            bw.write(0, 4)
            bw.write(fr['common'], 1)
            if fr['common']:
                _ics_info(bw, fr, max_sfb)
                bw.write(fr['ms'], 2)
                if fr['ms'] == 1:
                    for gi in range(G):
                        for b in range(max_sfb):
                            bw.write(int(used[gi, b]), 1)
            for c in range(2):
                _write_ics(bw, chans[c], fr, sfi, max_sfb, fr['common'], pulses[c], tns[c])
        if fr.get('fill'):
            bw.write(FIL, 3)
            bw.write(2, 4)
            bw.write(0, 4)   # EXT_FILL
            bw.write(0xA5, 8)
            bw.write(0, 4)
        if pad_to:   # a FIL element of nb bytes: 3 + 4 (+ 8 when nb >= 15) + 8 nb bits, then END and alignment
            nb = (8 * pad_to - bw.n - 10) // 8
            if nb >= 15:
                nb = (8 * pad_to - bw.n - 18) // 8
            if nb < 0 or nb > 269:
                raise ValueError('packet %d does not fit %d bytes' % (k, pad_to))
            bw.write(FIL, 3)
            if nb >= 15:
                bw.write(15, 4)
                bw.write(nb - 14, 8)
            else:
                bw.write(nb, 4)
            if nb:
                bw.write(0, 4)   # EXT_FILL
                bw.write(0, 8 * nb - 4)
        bw.write(END, 3)
        pkt = bw.bytes()
        if pad_to:
            assert len(pkt) == pad_to, (len(pkt), pad_to)
        packets.append(pkt)
        prev, prev_shape = fr, fr['shape']
    return packets, asc(sfi, C)


def asc(sfi, C, aot=2, frame960=False, sbr_ext=None):
    """AudioSpecificConfig bytes (GASpecificConfig; sbr_ext: a sync extension with sbrPresentFlag 0 or 1)."""
    bw = BitWriter()
    bw.write(aot, 5)
    bw.write(sfi, 4)
    bw.write(C, 4)
    bw.write(int(frame960), 1)
    bw.write(0, 1)
    bw.write(0, 1)
    if sbr_ext is not None:
        bw.write(0x2B7, 11)
        bw.write(5, 5)
        bw.write(sbr_ext, 1)
    return bw.bytes()


def adts(packet, sfi, C):
    """A packet with a 7-byte ADTS header (no CRC), for decoders that take ADTS."""
    n = len(packet) + 7
    h = (0xFFF << 44) | (0 << 43) | (0 << 41) | (1 << 40) | (1 << 38) | (sfi << 34) | (C << 30) | (n << 13) | \
        (0x7FF << 2)
    return h.to_bytes(7, 'big') + packet


# ------------------------------------------------------------------------------------------------------------ MP4

def _box(t, payload):
    if len(payload) + 8 > 0xFFFFFFFF:
        return struct.pack('>I4sQ', 1, t, len(payload) + 16) + payload
    return struct.pack('>I4s', len(payload) + 8, t) + payload


def _full(t, version, flags, payload):
    return _box(t, struct.pack('>I', (version << 24) | flags) + payload)


_MATRIX = struct.pack('>9I', 0x10000, 0, 0, 0, 0x10000, 0, 0, 0, 0x40000000)


def _esds(asc_bytes, oti=0x40):
    dsi = b'\x05' + bytes([len(asc_bytes)]) + asc_bytes
    dcd = b'\x04' + bytes([13 + len(dsi)]) + bytes([oti, 0x15]) + b'\0\0\0' + struct.pack('>II', 128000, 128000) + dsi
    sl = b'\x06\x01\x02'
    es = b'\x03' + bytes([3 + len(dcd) + len(sl)]) + b'\0\x01\0' + dcd + sl
    return _full(b'esds', 0, 0, es)


def _sample_entry(fmt, C, rate, asc_bytes, oti=0x40):
    body = b'\0' * 6 + struct.pack('>H', 1) + b'\0' * 8 + struct.pack('>HHHHI', C, 16, 0, 0, (rate & 0xFFFF) << 16)
    if fmt == b'mp4a':
        body += _esds(asc_bytes, oti)
    return _box(fmt, body)


def _trak(track_id, handler, stsd_entry, tables, rate, duration, movie_ts):
    tkhd = _full(b'tkhd', 0, 7, struct.pack('>IIIII', 0, 0, track_id, 0, duration * movie_ts // max(rate, 1)) +
                 b'\0' * 8 + struct.pack('>hhhH', 0, 0, 0x100 if handler == b'soun' else 0, 0) + _MATRIX +
                 struct.pack('>II', 0, 0))
    mdhd = _full(b'mdhd', 0, 0, struct.pack('>IIIIHH', 0, 0, rate, duration, 0x55C4, 0))
    hdlr = _full(b'hdlr', 0, 0, struct.pack('>I4s', 0, handler) + b'\0' * 12 + b'Handler\0')
    mh = _full(b'smhd', 0, 0, b'\0' * 4) if handler == b'soun' else _full(b'vmhd', 0, 1, b'\0' * 8)
    dinf = _box(b'dinf', _full(b'dref', 0, 0, struct.pack('>I', 1) + _full(b'url ', 0, 1, b'')))
    stsd = _full(b'stsd', 0, 0, struct.pack('>I', 1) + stsd_entry)
    stbl = _box(b'stbl', stsd + tables)
    mdia = _box(b'mdia', mdhd + hdlr + _box(b'minf', mh + dinf + stbl))
    return _box(b'trak', tkhd + mdia)


def rescale(a, b, c):
    """a * b / c rounded to nearest, halves away from zero (FFmpeg's av_rescale)."""
    return (a * b + c // 2) // c


def mp4(packets, asc_bytes, rate, C, layout='plain', edit=None, video=False, movie_ts=1000, fmt=b'mp4a', oti=0x40,
        stts_delta=FRAME, frag=7):
    """An ISO BMFF file holding the packets.  layout: 'plain' (moov first, one chunk), 'moov_last', 'co64' (64-bit
    chunk offsets and a 64-bit mdat size), 'chunks' (chunks of varying length with junk between them: stsc runs),
    'fragmented' (empty sample tables, mvex/trex, then moof/traf/tfhd/trun + mdat per ``frag`` packets, alternating
    default-base-is-moof and an explicit base offset).  edit: None, or (priming samples, kept samples), written as one
    elst entry in the movie timescale ``movie_ts``; a list writes that many entries.  A constant sample size goes into
    stsz's sample_size.  Returns (bytes, truth) where truth has the offsets, sizes and the expected trim."""
    F = len(packets)
    sizes = [len(p) for p in packets]
    ftyp = _box(b'ftyp', b'M4A \0\0\0\0M4A mp42isom')
    seg = None
    edits = None
    if edit is not None:
        edits = edit if isinstance(edit, list) else [edit]
        seg = [(rescale(k, movie_ts, rate), m) for m, k in edits]
    movie_dur = F * FRAME * movie_ts // rate
    mvhd = _full(b'mvhd', 0, 0, struct.pack('>IIII', 0, 0, movie_ts, movie_dur) + struct.pack('>IH', 0x10000, 0x100) +
                 b'\0' * 10 + _MATRIX + b'\0' * 24 + struct.pack('>I', 3))
    entry = _sample_entry(fmt, C, rate, asc_bytes, oti)

    def elst_box():
        if seg is None:
            return b''
        return _box(b'edts', _full(b'elst', 0, 0, struct.pack('>I', len(seg)) +
                                   b''.join(struct.pack('>IiI', s, m, 0x10000) for s, m in seg)))

    def trak_audio(tables):
        t = _trak(2, b'soun', entry, tables, rate, F * FRAME, movie_ts)
        if seg is None:
            return t
        body = t[8:]
        tk_len = struct.unpack('>I', body[:4])[0]
        return _box(b'trak', body[:tk_len] + elst_box() + body[tk_len:])

    vtrak = b''
    if video:
        ventry = _box(b'avc1', b'\0' * 6 + struct.pack('>H', 1) + b'\0' * 16 + struct.pack('>HH', 64, 64) + b'\0' * 50)
        vt = _full(b'stts', 0, 0, struct.pack('>I', 0)) + _full(b'stsc', 0, 0, struct.pack('>I', 0)) + \
            _full(b'stsz', 0, 0, struct.pack('>II', 0, 0)) + _full(b'stco', 0, 0, struct.pack('>I', 0))
        vtrak = _trak(1, b'vide', ventry, vt, 25, 0, movie_ts)
    stts = _full(b'stts', 0, 0, struct.pack('>III', 1, F, stts_delta))
    const = len(set(sizes)) == 1
    stsz = _full(b'stsz', 0, 0, struct.pack('>II', sizes[0], F) if const else
                 struct.pack('>II', 0, F) + struct.pack('>%dI' % F, *sizes))
    truth = dict(sizes=sizes, priming=None, kept=None, fragmented=layout == 'fragmented')
    if edits is not None and len(edits) == 1:
        m, k = edits[0]
        truth['priming'] = m
        truth['kept'] = min(rescale(seg[0][0], rate, movie_ts), F * FRAME - m)
    if layout == 'fragmented':
        empty = _full(b'stts', 0, 0, struct.pack('>I', 0)) + _full(b'stsc', 0, 0, struct.pack('>I', 0)) + \
            _full(b'stsz', 0, 0, struct.pack('>II', 0, 0)) + _full(b'stco', 0, 0, struct.pack('>I', 0))
        mvex = _box(b'mvex', _full(b'trex', 0, 0, struct.pack('>IIIII', 2, 1, FRAME, 0, 0)))
        moov = _box(b'moov', mvhd + vtrak + trak_audio(empty) + mvex)
        out = bytearray(ftyp + moov)
        offsets = []
        for fi, a in enumerate(range(0, F, frag)):
            part = packets[a:a + frag]
            explicit = fi % 2 == 1
            mfhd = _full(b'mfhd', 0, 0, struct.pack('>I', fi + 1))
            tfdt = _full(b'tfdt', 1, 0, struct.pack('>Q', a * FRAME))

            def build(data_offset, base):
                if explicit:
                    tfhd = _full(b'tfhd', 0, 0x1 | 0x8, struct.pack('>IQI', 2, base, FRAME))
                else:
                    tfhd = _full(b'tfhd', 0, 0x20000 | 0x8, struct.pack('>II', 2, FRAME))
                trun = _full(b'trun', 0, 0x1 | 0x200, struct.pack('>Ii', len(part), data_offset) +
                             b''.join(struct.pack('>I', len(p)) for p in part))
                return _box(b'moof', mfhd + _box(b'traf', tfhd + tfdt + trun))
            moof_at = len(out)
            size = len(build(0, 0))
            payload_at = moof_at + size + 8
            moof = build(0, payload_at) if explicit else build(size + 8, 0)
            out += moof + _box(b'mdat', b''.join(part))
            o = payload_at
            for p in part:
                offsets.append(o)
                o += len(p)
        truth['offsets'] = offsets
        return bytes(out), truth
    # chunk layout
    if layout == 'chunks':
        runs, i, lens = [], 0, []
        pattern = [3, 3, 5, 1, 4]
        while i < F:
            n = min(pattern[len(lens) % len(pattern)], F - i)
            lens.append(n)
            i += n
        junk = b'\xEE' * 5
    else:
        lens, junk = [F], b''
    stsc_rows = []
    for ci, n in enumerate(lens):
        if not stsc_rows or stsc_rows[-1][1] != n:
            stsc_rows.append((ci + 1, n, 1))
    stsc = _full(b'stsc', 0, 0, struct.pack('>I', len(stsc_rows)) + b''.join(struct.pack('>III', *r) for r in stsc_rows))
    big = layout == 'co64'

    def moov_with(chunk_offsets):
        co = _full(b'co64', 0, 0, struct.pack('>I', len(lens)) + b''.join(struct.pack('>Q', o) for o in chunk_offsets)) \
            if big else _full(b'stco', 0, 0, struct.pack('>I', len(lens)) +
                              b''.join(struct.pack('>I', o) for o in chunk_offsets))
        return _box(b'moov', mvhd + vtrak + trak_audio(stts + stsc + stsz + co))

    body, rel, i = bytearray(), [], 0
    for n in lens:
        body += junk
        rel.append(len(body))
        body += b''.join(packets[i:i + n])
        i += n
    mdat_hdr = 16 if big else 8
    mdat = (struct.pack('>I4sQ', 1, b'mdat', len(body) + 16) if big else struct.pack('>I4s', len(body) + 8, b'mdat')) \
        + bytes(body)
    moov_len = len(moov_with([0] * len(lens)))
    free = _box(b'free', b'\0' * 4)
    if layout == 'moov_last':
        base = len(ftyp) + len(free) + mdat_hdr
        data = ftyp + free + mdat + moov_with([base + r for r in rel])
    else:
        base = len(ftyp) + moov_len + mdat_hdr
        data = ftyp + moov_with([base + r for r in rel]) + mdat
    offsets, i = [], 0
    for r, n in zip(rel, lens):
        o = base + r
        for p in packets[i:i + n]:
            offsets.append(o)
            o += len(p)
        i += n
    truth['offsets'] = offsets
    return bytes(data), truth


# ------------------------------------------------------------------------------------------------------------ matrix

def sine_mix(n, rate, channels, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    out = np.zeros((channels, n))
    for c in range(channels):
        for _ in range(6):
            f = rng.uniform(60, 0.45 * rate)
            out[c] += rng.uniform(0.03, 0.15) * np.sin(2 * np.pi * f * t + rng.uniform(0, 6.3))
        out[c] += 0.02 * rng.standard_normal(n)
        out[c] *= 0.5 + 0.5 * np.abs(np.sin(2 * np.pi * 3.0 * t + c))   # attacks
    if channels == 2:
        out[1] = 0.6 * out[1] + 0.5 * out[0]
    return out


WS_CYCLE = (ONLY_LONG, ONLY_LONG, LONG_START, EIGHT_SHORT, EIGHT_SHORT, LONG_STOP, LONG_START, EIGHT_SHORT, LONG_STOP,
            ONLY_LONG)


def tools_plan(pns=False, tns=True, stereo_tools=True):
    """A plan cycling through every window sequence transition, both shapes each way, groupings, and by frame:
    random codebooks, pulse, escapes, TNS, M/S 0 / 1 / 2, intensity, PNS, fill and data elements."""
    def plan(k, rng, prev):
        ws = WS_CYCLE[k % len(WS_CYCLE)]
        fr = dict(ws=ws, shape=(k // 2) % 2 if k % 7 else int(rng.integers(0, 2)),
                  grouping=int(rng.integers(0, 128)), cb='random' if k % 3 else 'best', jitter=(k % 4) * 2,
                  ms=(0, 1, 2, 1)[k % 4], common=0 if k % 11 == 5 else 1, split_sections=k % 5 == 1,
                  pulse=ws != EIGHT_SHORT and k % 3 == 0, esc=k % 4 == 1, tns=tns and k % 2 == 0,
                  fill=k % 6 == 2, dse=k % 6 == 4)
        if stereo_tools and fr['common'] and fr['ms'] != 2:
            fr['is_bands'] = 3 if k % 3 != 2 else 0
        if pns and k % 2 == 1:
            fr['pns_bands'] = 4
            fr['tns'] = False
        if k % 9 == 8:
            fr['max_sfb'] = 3
        return fr
    return plan


def matrix():
    """[(name, .m4a bytes)]: every rate index, mono and stereo, every container layout, with and without edit list."""
    out = []
    layouts = ('plain', 'moov_last', 'co64', 'chunks', 'fragmented', 'plain')
    for sfi, rate in enumerate(T.RATES):
        C = 1 if sfi in (1, 8, 11) else 2
        n = 12 * FRAME + 300
        x = sine_mix(n, rate, C, seed=sfi)
        kbps = max(24, min(256, rate * C * 2 // 1000))
        packets, a = encode(x, rate, kbps, plan=tools_plan(), seed=sfi)
        layout = layouts[sfi % len(layouts)]
        edit = (FRAME, n) if sfi % 3 != 2 else None
        data, _ = mp4(packets, a, rate, C, layout=layout, edit=edit, video=sfi == 4, movie_ts=(1000, 600, rate)[sfi % 3])
        out.append(('%s_%dk_%s_%s' % ('tools', rate // 1000, 'mono' if C == 1 else 'stereo', layout), data))
    for sfi, C in ((4, 2), (8, 1)):
        rate = T.RATES[sfi]
        n = 10 * FRAME
        x = sine_mix(n, rate, C, seed=40 + sfi)
        packets, a = encode(x, rate, 96 * C, plan=tools_plan(pns=True), seed=40 + sfi)
        data, _ = mp4(packets, a, rate, C, edit=(FRAME, n))
        out.append(('pns_%dk_%s' % (rate // 1000, 'mono' if C == 1 else 'stereo'), data))
    rate = 48000
    x = sine_mix(8 * FRAME, rate, 2, seed=77)
    packets, a = encode(x, rate, 128, seed=77, pad_to=420)
    data, _ = mp4(packets, a, rate, 2, layout='fragmented', edit=(FRAME, 8 * FRAME))
    out.append(('cbr_48k_stereo_fragmented', data))
    return out


def is_pns(name):
    return name.startswith('pns_')
