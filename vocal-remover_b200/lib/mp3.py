"""MPEG-1 Audio Layer III input (ISO/IEC 11172-3) decoded on the GPU:
``decode(path_or_bytes, device) -> (CUDA float32 (channels, n), rate, info)``.

The host finds the audio (an ID3v2 tag at the start is skipped; ID3v1 and APEv2 tags at the end are dropped), copies
the bytes to the device once, and runs csrc/mp3.cu with a host step in between:

1. ``vr_mp3_scan`` lists every 11-bit frame sync with its header word.
2. ``build_chain`` (numpy) starts at the first MPEG-1 Layer III header that is followed by a consistent one (same
   rate and channel mode) at the distance its frame length gives, and follows the chain frame by frame to the end of
   the audio.  A last frame cut short is dropped.  A chain that breaks (junk between frames), a rate or mode that
   changes, and headers out of scope (MPEG-2 / 2.5, Layers I and II, free format, reserved fields) raise ValueError.
3. A first frame carrying a Xing, Info or VBRI header is not audio; its LAME extension, if any, gives the gapless trim:
   the first ``delay + 529`` and the last ``max(padding - 529, 0)`` samples are dropped (FFmpeg's mp3 demuxer and
   mpg123 do the same).
4. The main-data byte count of each frame follows from its header; their exclusive scan places every frame's main
   data in one reservoir buffer, and ``vr_mp3_decode`` does the rest (side info, Huffman decoding, stereo, hybrid
   filterbank, polyphase synthesis) and leaves a status per frame.

A frame whose main data would begin before the stream (a file cut from a longer one) decodes as an all-zero spectrum
and is counted in ``info['zeroed']``.  Every other status raises ValueError naming the file, the frame and its byte
offset.  The output is float32 at full scale 1, not clipped, at the file's own rate.
"""
import numpy as np

from . import codec

BITRATES = (0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320)   # kbit/s, MPEG-1 Layer III
RATES = (44100, 48000, 32000)
FRAME = 1152
GAPLESS = 529   # decoder delay the LAME tag's delay and padding leave out

# status codes of csrc/mp3.cu (code 1, ZEROED, is not an error)
ZEROED = 1
ERRORS = {
    2: 'window switching with block type 0 (reserved)',
    3: 'big_values above 288',
    4: 'the granules\' part2_3 bits run past the main data available to the frame',
    5: 'scale factors or big values run past the granule\'s part2_3_length',
}


def header_fields(words):
    """Header words (array) -> dict of field arrays."""
    w = np.asarray(words, np.int64)
    return dict(version=(w >> 19) & 3, layer=(w >> 17) & 3, crc=((w >> 16) & 1) == 0, br=(w >> 12) & 15,
                sr=(w >> 10) & 3, pad=(w >> 9) & 1, mode=(w >> 6) & 3, emph=w & 3)


def header_problem(word):
    """None for an MPEG-1 Layer III header this decoder takes, else why not."""
    f = {k: int(v[0]) for k, v in header_fields([word]).items() if k != 'crc'}
    if f['version'] == 1:
        return 'reserved MPEG version'
    if f['version'] != 3:
        return 'MPEG-2 / MPEG-2.5 (LSF, 8 to 24 kHz) is not supported'
    if f['layer'] == 0:
        return 'reserved layer'
    if f['layer'] != 1:
        return 'Layer %s is not supported (Layer III only)' % ('I' if f['layer'] == 3 else 'II')
    if f['br'] == 0:
        return 'free-format bitrate is not supported'
    if f['br'] == 15:
        return 'reserved bitrate index 15'
    if f['sr'] == 3:
        return 'reserved sampling frequency'
    if f['emph'] == 2:
        return 'reserved emphasis'
    return None


def _valid_and_length(words):
    f = header_fields(words)
    ok = (f['version'] == 3) & (f['layer'] == 1) & (f['br'] > 0) & (f['br'] < 15) & (f['sr'] < 3) & (f['emph'] != 2)
    kbps = np.asarray(BITRATES + (0,), np.int64)[f['br']]
    rate = np.asarray(RATES + (1,), np.int64)[f['sr']]
    return ok, np.where(ok, 144000 * kbps // rate + f['pad'], 0), f


def audio_end(data, start):
    """End of the frames: the file's end less an ID3v1 tag and an APEv2 tag."""
    end = len(data)
    for _ in range(2):
        if end - 128 >= start and data[end - 128:end - 125] == b'TAG':
            end -= 128
            continue
        if end - 32 >= start and data[end - 32:end - 24] == b'APETAGEX':
            size = int.from_bytes(data[end - 20:end - 16], 'little')
            flags = int.from_bytes(data[end - 12:end - 8], 'little')
            end = max(start, end - size - (32 if flags & 0x80000000 else 0))
            continue
        break
    return end


def build_chain(cands, start, end, name='<bytes>'):
    """Frames from the scan's candidate rows (offset, header word), in byte order.

    Returns (frames int64 (F, 2) = (offset, header word), number of cut frames dropped at the end)."""
    cands = np.asarray(cands, np.int64).reshape(-1, 2)
    cands = cands[(cands[:, 0] >= start) & (cands[:, 0] + 4 <= end)]
    offs, words = cands[:, 0], cands[:, 1]
    ok, flen, f = _valid_and_length(words)
    nxt = offs + flen
    j = np.minimum(np.searchsorted(offs, nxt), max(len(offs) - 1, 0))
    has_next = (len(offs) > 0) & (offs[j] == nxt) if len(offs) else np.zeros(0, bool)
    consistent = ok & ((nxt == end) | (has_next & ok[j] & (f['sr'][j] == f['sr']) & (f['mode'][j] == f['mode'])))
    first = np.flatnonzero(consistent)
    if not first.size:
        if len(offs):
            why = header_problem(int(words[0]))
            if why:
                raise ValueError('%s: frame 0 (byte %d): %s' % (name, int(offs[0]), why))
        raise ValueError('%s: no MPEG-1 Layer III frame found (bytes %d to %d)' % (name, start, end))
    i = int(first[0])
    sr0, mode0 = int(f['sr'][i]), int(f['mode'][i])
    # the chain from the first frame by pointer doubling over the successor of every candidate (the candidate where
    # its frame ends; n, absorbing, where none does or the audio ends): about log2(frames) vectorised rounds
    n = len(offs)
    succ = np.append(np.where(ok & has_next & (nxt < end), j, n), n)
    chain = np.array([i], np.int64)
    while chain[-1] != n:   # chain holds the first 2^k frames; succ, composed with itself k times, gives the next 2^k
        chain = np.concatenate([chain, succ[chain]])
        succ = succ[succ]
    chain = chain[:np.searchsorted(chain, n)]
    bad = np.flatnonzero(~ok[chain] | (f['sr'][chain] != sr0) | (f['mode'][chain] != mode0))
    if bad.size:
        k = int(bad[0])
        c = chain[k]
        if not ok[c]:
            raise ValueError('%s: frame %d (byte %d): %s' % (name, k, int(offs[c]), header_problem(int(words[c]))))
        raise ValueError('%s: frame %d (byte %d): the sample rate or channel mode changes (rate %d -> %s, mode %d -> '
                         '%d)' % (name, k, int(offs[c]), RATES[sr0], RATES[f['sr'][c]] if f['sr'][c] < 3 else
                                  'reserved', mode0, int(f['mode'][c])))
    last = chain[-1]
    dropped = 0
    if nxt[last] > end:
        dropped = 1
        chain = chain[:-1]
    elif nxt[last] < end:
        raise ValueError('%s: frame %d (byte %d): no frame header where the previous frame ends: the frame chain '
                         'breaks (junk between frames)' % (name, len(chain), int(nxt[last])))
    if not chain.size:
        raise ValueError('%s: frame 0 (byte %d) is cut short and no whole frame follows' % (name, int(offs[last])))
    chosen = chain
    frames = np.stack([offs[chosen], words[chosen]], axis=1)
    return frames, dropped


def xing_info(data, off, word):
    """None, or dict(delay, padding, lame) of a Xing / Info / VBRI header in the frame at ``off``."""
    f = {k: int(v[0]) for k, v in header_fields([word]).items()}
    o = off + 4 + (2 if f['crc'] else 0) + (17 if f['mode'] == 3 else 32)
    if data[off + 36:off + 40] == b'VBRI':
        return dict(delay=0, padding=0, lame=False)
    if data[o:o + 4] not in (b'Xing', b'Info'):
        return None
    flags = int.from_bytes(data[o + 4:o + 8], 'big')
    p = o + 8 + (4 if flags & 1 else 0) + (4 if flags & 2 else 0) + (100 if flags & 4 else 0) + (4 if flags & 8 else 0)
    flen = 144000 * BITRATES[f['br']] // RATES[f['sr']] + f['pad']
    if data[p:p + 4] in (b'LAME', b'Lavf', b'Lavc') and p + 24 <= off + flen:
        v = int.from_bytes(data[p + 21:p + 24], 'big')
        return dict(delay=v >> 12, padding=v & 0xFFF, lame=True)
    return dict(delay=0, padding=0, lame=False)


def trim_range(n, x):
    """[a, b) of the n decoded samples that the gapless trim keeps (x: xing_info of the first frame, or None)."""
    if x is None or not x['lame']:
        return 0, n
    a = min(x['delay'] + GAPLESS, n)
    return a, max(a, n - max(x['padding'] - GAPLESS, 0))


def main_data_offsets(frames):
    """Exclusive scan of the frames' main-data byte counts (frame length less header, CRC and side info)."""
    ok, flen, f = _valid_and_length(frames[:, 1])
    md = flen - 4 - np.where(f['crc'], 2, 0) - np.where(f['mode'] == 3, 17, 32)
    out = np.zeros(len(frames) + 1, np.int64)
    np.cumsum(md, out=out[1:])
    return out


def sniff(path):
    """True if the file holds MPEG-1 Layer III by content: a valid header, possibly after an ID3v2 tag, followed by a
    consistent second header at the distance its frame length gives."""
    try:
        with open(path, 'rb') as f:
            head = f.read(10)
            skip = codec.id3v2_size(head)
            f.seek(skip)
            b = f.read(4)
            if len(b) < 4 or b[0] != 0xFF or (b[1] & 0xE0) != 0xE0:   # the 11-bit sync
                return False
            w = int.from_bytes(b, 'big')
            ok, flen, fl = _valid_and_length([w])
            if not ok[0]:
                return False
            f.seek(skip + int(flen[0]))
            b2 = f.read(4)
    except OSError:
        return False
    if len(b2) < 4:
        return False
    ok2, _, f2 = _valid_and_length([int.from_bytes(b2, 'big')])
    return bool(b2[0] == 0xFF and (b2[1] & 0xE0) == 0xE0 and ok2[0] and f2['sr'][0] == fl['sr'][0] and f2['mode'][0] == fl['mode'][0])


def decode(src, device=None):
    """MP3 file path or bytes -> (CUDA float32 tensor (channels, n), sample rate, info).  info: frames (audio frames
    decoded), delay and padding (of the LAME tag, 0 without one), dropped (a cut last frame), zeroed (frames whose main
    data began before the stream), xing, lame."""
    import torch
    from . import _native
    name, data = codec.source(src)
    start = codec.id3v2_size(data)
    end = audio_end(data, start)
    dev = codec.cuda_device(name, 'MP3', device)
    lib = _native.load_library()
    with torch.cuda.device(dev):
        d_data = torch.frombuffer(bytearray(data[:end]), dtype=torch.uint8).to(dev) if end else \
            torch.zeros(1, dtype=torch.uint8, device=dev)
        rows = codec.scan(lib, 'vr_mp3_scan', d_data, start, end, 2, 256 + end // 128)
        h_cands = rows[torch.argsort(rows[:, 0])].cpu().numpy()   # in byte order (the scan appends unordered)
        frames, dropped = build_chain(h_cands, start, end, name)
        x = xing_info(data, int(frames[0, 0]), int(frames[0, 1]))
        first = 1 if x is not None else 0
        frames = frames[first:]
        if not len(frames):
            raise ValueError('%s: no audio frame after the Xing / Info header' % name)
        md_off = main_data_offsets(frames)
        F = len(frames)
        C = 1 if int(header_fields(frames[:1, 1])['mode'][0]) == 3 else 2
        sr = int(header_fields(frames[:1, 1])['sr'][0])
        md_bytes = int(md_off[-1])
        ws_bytes = int(lib.vr_mp3_workspace(F, C, md_bytes))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        out = torch.empty((C, F * FRAME), dtype=torch.float32, device=dev)
        status = torch.empty(F, dtype=torch.int64, device=dev)
        d_frames = torch.from_numpy(np.ascontiguousarray(frames)).to(dev)
        d_md_off = torch.from_numpy(md_off).to(dev)
        _native.check(lib, lib.vr_mp3_decode(None, _native.ptr(d_data), end, _native.ptr(d_frames),
                                             _native.ptr(d_md_off), F, C, sr, md_bytes, _native.ptr(ws), ws_bytes,
                                             _native.ptr(out), _native.ptr(status), _native.stream_ptr()),
                      'vr_mp3_decode')
        st = status.cpu().numpy()
    codec.raise_first_bad(st, frames[:, 0], ERRORS, name, 'frame', allowed=(ZEROED,), first=first)
    a, b = trim_range(F * FRAME, x)
    info = dict(frames=F, delay=x['delay'] if x else 0, padding=x['padding'] if x else 0, dropped=dropped,
                zeroed=int(((st >> 40) == ZEROED).sum()), xing=x is not None, lame=bool(x and x['lame']))
    return codec.trim(out, a, b), RATES[sr], info
