"""MPEG-4 AAC-LC in an ISO BMFF container (.m4a, .mp4, .mov) decoded on the GPU:
``decode(path_or_bytes, device) -> (CUDA float32 (channels, n), rate, info)``.

The host walks the boxes (``parse``): the first ``soun`` track whose sample entry is ``mp4a`` with objectTypeIndication
0x40 (other tracks, a video track included, are ignored), its AudioSpecificConfig from ``esds``, and its packets, from
the sample table (``stsz`` constant or per sample, ``stsc`` runs, ``stco`` or ``co64``) or from the fragments
(``mvex``/``trex``, then ``moof``/``traf``/``tfhd``/``trun``), turned into (offset, size) arrays with numpy.  One
``elst`` edit gives the trim as FFmpeg's mov demuxer applies it: ``media_time`` priming samples are dropped and
``segment_duration``, rescaled from the movie to the media timescale, is kept.

AAC-LC packets are independent (no bit reservoir), so ``vr_aac_decode`` (csrc/aac.cu) takes the packet table as it is
and leaves a status per packet.  Everything out of scope raises ValueError naming the file and the reason: HE-AAC (v2),
Main / SSR / LTP, 960-sample frames, channel configurations other than 1 and 2, an ``stts`` delta other than 1024,
``enca`` and ``alac`` entries, more than one edit; a malformed packet names the packet, its byte offset and the bit.
The output is float32 at full scale 1, not clipped, at the file's own rate.
"""
import struct

import numpy as np

from .flac import _name, _read

FRAME = 1024
RATES = (96000, 88200, 64000, 48000, 44100, 32000, 24000, 22050, 16000, 12000, 11025, 8000)
AOT_NAMES = {1: 'AAC Main', 3: 'AAC SSR', 4: 'AAC LTP', 5: 'HE-AAC (SBR)', 29: 'HE-AACv2 (PS)'}

# status codes of csrc/aac.cu
ERRORS = {
    1: 'the bits run past the end of the packet',
    2: 'a section runs past max_sfb',
    3: 'reserved section codebook 12',
    4: 'max_sfb is above the number of scale-factor bands',
    5: 'an escape sequence is longer than 13 bits',
    6: 'pulse data in an EIGHT_SHORT frame, or a pulse past the spectrum',
    7: 'TNS order above the maximum',
    8: 'reserved ms_mask_present 3',
    9: 'predictor_data_present is set: Main-profile or LTP prediction is not AAC-LC',
    10: 'gain_control_data_present is set: AAC SSR is not AAC-LC',
    11: 'a CCE, LFE or PCE element, or a channel element that does not match the channel configuration',
    12: 'an SBR extension payload in a FIL element (HE-AAC, implicit signalling) is not supported',
    13: 'no channel element before END',
    14: 'ics_reserved_bit is set',
    15: 'a scale factor leaves [0, 255]',
}


def sniff(path):
    """True for an ISO BMFF file: an ``ftyp`` box, or a top-level ``moov``, ``mdat`` or ``free`` box, at offset 4."""
    try:
        with open(path, 'rb') as f:
            head = f.read(8)
    except OSError:
        return False
    if len(head) < 8 or head[4:8] not in (b'ftyp', b'moov', b'mdat', b'free'):
        return False
    size = struct.unpack('>I', head[:4])[0]
    return size in (0, 1) or size >= 8


def _boxes(data, start, end, name):
    """(type, payload start, box end, box start) of the boxes in data[start:end]."""
    out, o = [], start
    while o + 8 <= end:
        size, typ = struct.unpack('>I4s', data[o:o + 8])
        hdr = 8
        if size == 1:
            if o + 16 > end:
                raise ValueError('%s: a 64-bit box size is cut short at byte %d' % (name, o))
            size = struct.unpack('>Q', data[o + 8:o + 16])[0]
            hdr = 16
        elif size == 0:
            size = end - o
        if size < hdr or o + size > end:
            raise ValueError('%s: box %r at byte %d runs past its parent (size %d)' % (name, typ, o, size))
        out.append((typ, o + hdr, o + size, o))
        o += size
    return out


def _children(data, start, end, name):
    d = {}
    for typ, a, b, o in _boxes(data, start, end, name):
        d.setdefault(typ, []).append((a, b, o))
    return d


def _one(boxes, typ, parent, name):
    """(payload start, end, box start) of the first ``typ`` child; ValueError naming the file if there is none."""
    if typ not in boxes:
        raise ValueError('%s: no %s box in %s' % (name, typ.decode('latin-1'), parent))
    return boxes[typ][0]


def _descriptor(data, o):
    tag = data[o]
    n, o = 0, o + 1
    for _ in range(4):
        c = data[o]
        o += 1
        n = (n << 7) | (c & 0x7F)
        if not c & 0x80:
            break
    return tag, o, o + n


def parse_esds(data, a, b, name):
    """-> (objectTypeIndication, AudioSpecificConfig bytes)."""
    o = a + 4
    tag, o, end = _descriptor(data, o)
    if tag != 3:
        raise ValueError('%s: esds holds no ES_Descriptor' % name)
    flags = data[o + 2]
    o += 3
    if flags & 0x80:
        o += 2
    if flags & 0x40:
        o += 1 + data[o]
    if flags & 0x20:
        o += 2
    tag, o, end = _descriptor(data, o)
    if tag != 4:
        raise ValueError('%s: esds holds no DecoderConfigDescriptor' % name)
    oti = data[o]
    o += 13
    asc = b''
    if o < end:
        tag, p, q = _descriptor(data, o)
        if tag == 5:
            asc = bytes(data[p:q])
    return oti, asc


def parse_asc(asc, name):
    """AudioSpecificConfig -> (sampling-frequency index, channel configuration); ValueError out of scope."""
    v = int.from_bytes(asc + b'\0' * 8, 'big')
    n = 8 * (len(asc) + 8)
    pos = [0]

    def rd(k):
        pos[0] += k
        return (v >> (n - pos[0])) & ((1 << k) - 1)
    if len(asc) < 2:
        raise ValueError('%s: the AudioSpecificConfig is missing or shorter than 2 bytes' % name)
    aot = rd(5)
    if aot == 31:
        aot = 32 + rd(6)
    sfi = rd(4)
    if sfi == 15:
        raise ValueError('%s: an explicit sampling frequency (index 15) is not supported' % name)
    if sfi > 11:
        raise ValueError('%s: reserved sampling-frequency index %d' % (name, sfi))
    ch = rd(4)
    if aot != 2:
        raise ValueError('%s: audio object type %d (%s) is not supported: AAC-LC (2) only' %
                         (name, aot, AOT_NAMES.get(aot, 'not AAC-LC')))
    if ch == 0:
        raise ValueError('%s: channel configuration 0 (a PCE) is not supported: 1 or 2 channels only' % name)
    if ch > 2:
        raise ValueError('%s: channel configuration %d is not supported: 1 or 2 channels only' % (name, ch))
    if rd(1):
        raise ValueError('%s: 960-sample frames (frameLengthFlag) are not supported' % name)
    if rd(1):
        rd(14)
    rd(1)
    if 8 * len(asc) - pos[0] >= 16 and rd(11) == 0x2B7:
        if rd(5) == 5 and rd(1):
            raise ValueError('%s: an SBR sync extension (HE-AAC, explicit signalling) is not supported' % name)
    return sfi, ch


def _full_payload(data, a):
    word = struct.unpack('>I', data[a:a + 4])[0]
    return word >> 24, word & 0xFFFFFF, a + 4


def _audio_entry(data, stsd, name):
    """First sample entry of an stsd -> (format, oti, asc, why-not or None)."""
    a, b, _ = stsd
    entries = _boxes(data, a + 8, b, name)
    if not entries:
        return None, None, None, 'an empty sample description'
    typ, p, q, _ = entries[0]
    if typ == b'enca':
        return typ, None, None, 'an encrypted (enca) sample entry is not supported'
    if typ == b'alac':
        return typ, None, None, 'an ALAC sample entry is not supported (AAC-LC only)'
    if typ != b'mp4a':
        return typ, None, None, 'sample entry %r is not mp4a' % typ.decode('latin-1')
    version = struct.unpack('>H', data[p + 8:p + 10])[0]
    kids = p + 28 + {0: 0, 1: 16, 2: 36}.get(version, 0)
    sub = _children(data, kids, q, name)
    if b'esds' not in sub:
        return typ, None, None, 'the mp4a entry has no esds'
    oti, asc = parse_esds(data, sub[b'esds'][0][0], sub[b'esds'][0][1], name)
    if oti != 0x40:
        return typ, oti, asc, 'objectTypeIndication 0x%02x is not MPEG-4 audio (0x40)' % oti
    return typ, oti, asc, None


def _sample_table(data, stbl, name):
    k = _children(data, stbl[0], stbl[1], name)
    for need in (b'stsz', b'stsc'):
        if need not in k:
            raise ValueError('%s: the audio track has no %s' % (name, need.decode()))
    _, _, a = _full_payload(data, k[b'stsz'][0][0])
    size, count = struct.unpack('>II', data[a:a + 8])
    sizes = np.full(count, size, np.int64) if size else \
        np.frombuffer(data, '>u4', count, a + 8).astype(np.int64)
    _, _, a = _full_payload(data, k[b'stsc'][0][0])
    n = struct.unpack('>I', data[a:a + 4])[0]
    stsc = np.frombuffer(data, '>u4', 3 * n, a + 4).reshape(n, 3).astype(np.int64)
    if b'co64' in k:
        _, _, a = _full_payload(data, k[b'co64'][0][0])
        n = struct.unpack('>I', data[a:a + 4])[0]
        chunks = np.frombuffer(data, '>u8', n, a + 4).astype(np.int64)
    elif b'stco' in k:
        _, _, a = _full_payload(data, k[b'stco'][0][0])
        n = struct.unpack('>I', data[a:a + 4])[0]
        chunks = np.frombuffer(data, '>u4', n, a + 4).astype(np.int64)
    else:
        raise ValueError('%s: the audio track has neither stco nor co64' % name)
    if b'stts' in k:
        _, _, a = _full_payload(data, k[b'stts'][0][0])
        n = struct.unpack('>I', data[a:a + 4])[0]
        stts = np.frombuffer(data, '>u4', 2 * n, a + 4).reshape(n, 2)
        bad = np.flatnonzero((stts[:, 1] != FRAME) & (stts[:, 0] > 0))
        if bad.size:
            raise ValueError('%s: stts delta %d is not supported (1024-sample frames only)' % (name, stts[bad[0], 1]))
    if not count:
        return np.zeros(0, np.int64), sizes
    # samples per chunk from the stsc runs, then each sample's chunk and its place in the chunk
    firsts = stsc[:, 0] - 1
    run_len = np.diff(np.append(firsts, len(chunks)))
    per_chunk = np.repeat(stsc[:, 1], np.maximum(run_len, 0))
    ends = np.cumsum(per_chunk)
    if ends.size == 0 or ends[-1] < count:
        raise ValueError('%s: stsc and the chunk offsets hold %d samples, stsz %d' % (name, int(ends[-1]) if ends.size
                                                                                      else 0, count))
    chunk_of = np.searchsorted(ends, np.arange(count), side='right')
    csum = np.concatenate([[0], np.cumsum(sizes)])
    first_in_chunk = np.concatenate([[0], ends])[chunk_of]
    offsets = chunks[chunk_of] + csum[:count] - csum[first_in_chunk]
    return offsets, sizes


def _fragments(data, top, track_id, trex, name):
    """(offsets, sizes) of the track's samples in every moof, in file order."""
    offs, sizes = [], []
    for typ, a, b, o in top:
        if typ != b'moof':
            continue
        for ta, tb, _ in _children(data, a, b, name).get(b'traf', []):
            k = _children(data, ta, tb, name)
            _, flags, p = _full_payload(data, _one(k, b'tfhd', 'traf', name)[0])
            tid = struct.unpack('>I', data[p:p + 4])[0]
            if tid != track_id:
                continue
            p += 4
            base = o   # default-base-is-moof, or no base given: the moof's first byte
            if flags & 0x1:
                base = struct.unpack('>Q', data[p:p + 8])[0]
                p += 8
            if flags & 0x2:
                p += 4
            dur = trex.get('duration', FRAME)
            if flags & 0x8:
                dur = struct.unpack('>I', data[p:p + 4])[0]
                p += 4
            dsize = trex.get('size', 0)
            if flags & 0x10:
                dsize = struct.unpack('>I', data[p:p + 4])[0]
            pos = base
            for ra, rb, _ in k.get(b'trun', []):
                _, rf, q = _full_payload(data, ra)
                n = struct.unpack('>I', data[q:q + 4])[0]
                q += 4
                if rf & 0x1:
                    pos = base + struct.unpack('>i', data[q:q + 4])[0]
                    q += 4
                if rf & 0x4:
                    q += 4
                fields = [(0x100, 'd'), (0x200, 's'), (0x400, 'f'), (0x800, 'c')]
                per = [f for bit, f in fields if rf & bit]
                rows = np.frombuffer(data, '>u4', n * len(per), q).reshape(n, len(per)) if per else \
                    np.zeros((n, 0), np.uint32)
                ds = rows[:, per.index('d')].astype(np.int64) if 'd' in per else np.full(n, dur, np.int64)
                if np.any(ds != FRAME):
                    raise ValueError('%s: a trun sample duration of %d is not supported (1024-sample frames only)' %
                                     (name, int(ds[ds != FRAME][0])))
                sz = rows[:, per.index('s')].astype(np.int64) if 's' in per else np.full(n, dsize, np.int64)
                offs.append(pos + np.concatenate([[0], np.cumsum(sz)[:-1]]))
                sizes.append(sz)
                pos += int(sz.sum())
    if not offs:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(offs).astype(np.int64), np.concatenate(sizes)


def parse(src, name=None):
    """The container of an .m4a / .mp4 file (path or bytes) -> dict(rate_index, rate, channels, offsets, sizes
    (int64 arrays, one entry per packet), media_time, segment (kept samples, None: to the end), edit (bool),
    fragmented, asc).  ValueError for anything out of scope."""
    name = name or _name(src)
    data = _read(src)
    top = _boxes(data, 0, len(data), name)
    tops = {}
    for typ, a, b, o in top:
        tops.setdefault(typ, []).append((a, b, o))
    if b'moov' not in tops:
        raise ValueError('%s: no moov box (not an MP4 / M4A file, or cut short)' % name)
    moov = _children(data, tops[b'moov'][0][0], tops[b'moov'][0][1], name)
    mvhd = _one(moov, b'mvhd', 'moov', name)[0]
    _, _, p = _full_payload(data, mvhd)
    version = data[mvhd]
    movie_ts = struct.unpack('>I', data[p + 16:p + 20] if version == 1 else data[p + 8:p + 12])[0]
    first_why = None
    for ta, tb, _ in moov.get(b'trak', []):
        trak = _children(data, ta, tb, name)
        a, b, _ = _one(trak, b'mdia', 'trak', name)
        mdia = _children(data, a, b, name)
        _, _, p = _full_payload(data, _one(mdia, b'hdlr', 'mdia', name)[0])
        if data[p + 4:p + 8] != b'soun':
            continue
        a, b, _ = _one(mdia, b'minf', 'mdia', name)
        minf = _children(data, a, b, name)
        stbl = _one(minf, b'stbl', 'minf', name)
        sk = _children(data, stbl[0], stbl[1], name)
        fmt, oti, asc, why = _audio_entry(data, _one(sk, b'stsd', 'stbl', name), name)
        if why:
            first_why = first_why or why
            continue
        sfi, channels = parse_asc(asc, name)
        mdhd = _one(mdia, b'mdhd', 'mdia', name)[0]
        mver = data[mdhd]
        _, _, p = _full_payload(data, mdhd)
        media_ts = struct.unpack('>I', data[p + 16:p + 20] if mver == 1 else data[p + 8:p + 12])[0]
        tk = _one(trak, b'tkhd', 'trak', name)[0]
        _, _, p = _full_payload(data, tk)
        track_id = struct.unpack('>I', data[p + 16:p + 20] if data[tk] == 1 else data[p + 8:p + 12])[0]
        media_time, segment, edit = 0, None, False
        if b'edts' in trak:
            ed = _children(data, trak[b'edts'][0][0], trak[b'edts'][0][1], name)
            if b'elst' in ed:
                ev, _, p = _full_payload(data, ed[b'elst'][0][0])
                n = struct.unpack('>I', data[p:p + 4])[0]
                if n > 1:
                    raise ValueError('%s: an edit list of %d edits is not supported (one edit at most)' % (name, n))
                if n == 1:
                    if ev == 1:
                        seg, mt = struct.unpack('>Qq', data[p + 4:p + 20])
                    else:
                        seg, mt = struct.unpack('>Ii', data[p + 4:p + 12])
                    if mt < 0:
                        raise ValueError('%s: an empty edit (media_time -1) is not supported' % name)
                    edit = True
                    media_time = mt * RATES[sfi] // media_ts if media_ts != RATES[sfi] else mt
                    if seg:   # segment_duration in the movie timescale -> media samples, rounded to nearest
                        segment = (seg * RATES[sfi] + movie_ts // 2) // movie_ts
        fragmented = b'mvex' in moov
        if fragmented:
            trex = {}
            mv = _children(data, moov[b'mvex'][0][0], moov[b'mvex'][0][1], name)
            for ra, rb, _ in mv.get(b'trex', []):
                _, _, p = _full_payload(data, ra)
                tid, _, dur, size, _ = struct.unpack('>IIIII', data[p:p + 20])
                if tid == track_id:
                    trex = dict(duration=dur, size=size)
            o1, s1 = _sample_table(data, stbl, name) if b'stsz' in sk else (np.zeros(0, np.int64),) * 2
            o2, s2 = _fragments(data, top, track_id, trex, name)
            offsets, sizes = np.concatenate([o1, o2]), np.concatenate([s1, s2])
        else:
            offsets, sizes = _sample_table(data, stbl, name)
        if not len(offsets):
            raise ValueError('%s: the audio track has no samples' % name)
        if offsets.min() < 0 or (offsets + sizes).max() > len(data) or sizes.min() <= 0:
            k = int(np.flatnonzero((offsets < 0) | (offsets + sizes > len(data)) | (sizes <= 0))[0])
            raise ValueError('%s: packet %d (byte %d, %d bytes) lies outside the file' % (name, k, int(offsets[k]),
                                                                                    int(sizes[k])))
        return dict(rate_index=sfi, rate=RATES[sfi], channels=channels, offsets=offsets, sizes=sizes,
                    media_time=int(media_time), segment=segment, edit=edit, fragmented=fragmented, asc=asc)
    raise ValueError('%s: no AAC-LC audio track: %s' % (name, first_why or 'no soun track'))


def gather(data, offsets, sizes):
    """The packets' bytes alone, back to back (a video track or other boxes in the file stay on the host), and their
    (offset, size) rows in that buffer.  Packets that follow each other in the file are copied as one run."""
    offsets, sizes = np.asarray(offsets, np.int64), np.asarray(sizes, np.int64)
    brk = np.flatnonzero(offsets[1:] != offsets[:-1] + sizes[:-1]) + 1
    starts = np.concatenate([[0], brk])
    ends = np.concatenate([brk, [len(offsets)]])
    mv = memoryview(data)
    packed = np.frombuffer(bytearray().join(mv[int(offsets[a]):int(offsets[e - 1] + sizes[e - 1])]
                                            for a, e in zip(starts, ends)), np.uint8)
    new = np.zeros(len(offsets), np.int64)
    np.cumsum(sizes[:-1], out=new[1:])
    return packed, np.ascontiguousarray(np.stack([new, sizes], axis=1))


def trim_range(n, t):
    """[a, b) of the n decoded samples that one edit keeps (everything without an edit list)."""
    if not t['edit']:
        return 0, n
    a = min(t['media_time'], n)
    return a, n if t['segment'] is None else min(n, a + t['segment'])


def decode(src, device=None):
    """M4A / MP4 file path or bytes -> (CUDA float32 tensor (channels, n), sample rate, info).  info: frames (packets
    decoded), priming (samples the edit drops at the start), kept (samples returned), fragmented."""
    import torch
    from . import _native
    name = _name(src)
    data = _read(src)
    t = parse(data, name)
    if not torch.cuda.is_available():
        raise RuntimeError('%s: M4A decoding runs on the GPU and no CUDA device is visible' % name)
    dev = torch.device(device if device is not None else 'cuda:0')
    lib = _native.load_library()

    def check(rc, what):
        if rc != 0:
            raise _native.NativeError('%s failed: %s' % (what, lib.vr_last_error(None).decode()))

    F, C, sfi = len(t['offsets']), t['channels'], t['rate_index']
    table = np.stack([t['offsets'], t['sizes']], axis=1).astype(np.int64)   # in the file, for the error messages
    packed, dev_table = gather(data, t['offsets'], t['sizes'])
    with torch.cuda.device(dev):
        d_data = torch.from_numpy(packed).to(dev)
        d_table = torch.from_numpy(dev_table).to(dev)
        ws_bytes = int(lib.vr_aac_workspace(F, C))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        out = torch.empty((C, F * FRAME), dtype=torch.float32, device=dev)
        status = torch.empty(F, dtype=torch.int64, device=dev)
        check(lib.vr_aac_decode(None, _native.ptr(d_data), len(packed), _native.ptr(d_table), F, C, sfi,
                                _native.ptr(ws), ws_bytes, _native.ptr(out), _native.ptr(status),
                                _native.stream_ptr()), 'vr_aac_decode')
        st = status.cpu().numpy()
    codes = st >> 40
    bad = np.flatnonzero(codes != 0)
    if bad.size:
        k = int(bad[0])
        raise ValueError('%s: packet %d (byte %d): %s (bit %d)' % (name, k, int(table[k, 0]),
                                                                  ERRORS.get(int(codes[k]), 'error %d' % codes[k]),
                                                                  int(st[k]) & ((1 << 40) - 1)))
    a, b = trim_range(F * FRAME, t)
    info = dict(frames=F, priming=a, kept=b - a, fragmented=t['fragmented'])
    y = out if (a, b) == (0, F * FRAME) else out[:, a:b].contiguous()
    return y, t['rate'], info
