"""Ogg Vorbis (Vorbis I in an Ogg stream, .ogg) decoded on the GPU:
``decode(path_or_bytes, device) -> (CUDA float32 (channels, n), rate, info)``.

The host reads the Ogg pages (``parse``): every page's CRC is checked, the pages of the first logical stream whose
beginning-of-stream page holds a Vorbis identification header are kept (a multiplexed second stream is ignored), and
their lacing values are turned into packets with numpy.  The identification and setup headers are parsed and the setup
flattened into one int32 array (``flatten``: per codebook its codewords, assigned the specification's lowest-free-leaf
way, sorted and left-aligned, and its VQ vectors expanded; the floor 1 X lists with their sort order and neighbours;
the residue, mapping and mode tables).  Each audio packet's mode is read from its first bits with numpy, so every block
size, output range and spectrum slot is known before ``vr_vorbis_decode`` (csrc/vorbis.cu) runs.  The packets' bytes
go to the device back to back (``gather``: a packet that spans pages becomes contiguous).

Granule positions (the Vorbis I specification's appendix A): the samples run from the centre of the first block to
the centre of the last.  When the first page on which an audio packet ends has a granule position below the samples
those packets return, the difference is trimmed from the front; the last page's granule position ends the output when
it is below the decoded count.

Out of scope, each a ValueError naming the file and the reason: floor type 0, more than 2 channels, a chained stream
(a second Vorbis beginning-of-stream page after the end of the first stream), a page whose CRC does not match (its
number and byte), a malformed or overpopulated setup header (the header and the field).  A malformed audio packet names
the packet, its byte offset and the bit.  The output is float32 at full scale 1, not clipped, at the file's own rate.
"""
import struct
import zlib

import numpy as np

from . import codec

# status codes of csrc/vorbis.cu
ERRORS = {
    1: 'the packet type bit is set: not an audio packet',
    2: 'the mode number is above the setup header\'s last mode',
    3: 'a codeword that the codebook does not hold',
    4: 'a floor 1 value leaves the floor\'s range',
    5: 'the packet ends before its mode and window flags',
}

# the setup array's layout (csrc/vorbis.cu has the same constants)
HDR_WORDS, BOOK_WORDS, FLOOR_WORDS, RES_WORDS, MAP_WORDS = 16, 8, 472, 518, 548
FL_PART_CLASS, FL_CLASS_DIM, FL_CLASS_SUB, FL_CLASS_MASTER, FL_SUB_BOOKS, FL_X, FL_ORDER = 4, 36, 52, 68, 84, 212, 277
FLOOR1_RANGE = (256, 128, 86, 64)
_REV8 = bytes(int('{:08b}'.format(i)[::-1], 2) for i in range(256))


def ogg_crc(page):
    """Ogg's CRC-32 (polynomial 0x04C11DB7, not reflected, initial value 0) through zlib on bit-reversed bytes."""
    c = zlib.crc32(bytes(page).translate(_REV8), 0xFFFFFFFF) ^ 0xFFFFFFFF
    return int('{:032b}'.format(c)[::-1], 2)


def sniff(path):
    """True for an Ogg stream whose first page is a beginning-of-stream page holding a Vorbis identification header.
    Only the first page is looked at: a file whose first page begins another stream (Theora video with Vorbis audio,
    say) is not claimed."""
    try:
        with open(path, 'rb') as f:
            head = f.read(27 + 255 + 7)
    except OSError:
        return False
    if len(head) < 28 or head[:4] != b'OggS' or not head[5] & 2:
        return False
    body = 27 + head[26]
    return head[body:body + 7] == b'\x01vorbis'


class _Bits:
    """LSB-first reads of a header packet; reading past its end is a ValueError naming the header and the field."""
    def __init__(self, data, name, header):
        self.v, self.n, self.pos = int.from_bytes(bytes(data), 'little'), 8 * len(data), 0
        self.name, self.header = name, header

    def read(self, k, field):
        if self.pos + k > self.n:
            raise ValueError('%s: the %s header ends inside %s' % (self.name, self.header, field))
        r = (self.v >> self.pos) & ((1 << k) - 1)
        self.pos += k
        return r

    def bad(self, field, why):
        return ValueError('%s: malformed %s header: %s (%s)' % (self.name, self.header, field, why))


def _ilog(x):
    return int(x).bit_length() if x > 0 else 0


def _float32(x):
    mant = x & 0x1FFFFF
    if x & 0x80000000:
        mant = -mant
    return float(mant) * 2.0 ** (((x & 0x7FE00000) >> 21) - 788)


def _lookup1_values(entries, dims):
    r = int(round(entries ** (1.0 / dims))) if dims else 0
    while r > 0 and r ** dims > entries:
        r -= 1
    while (r + 1) ** dims <= entries:
        r += 1
    return r


def _codes(lengths, bits, b):
    """Lowest-free-leaf codewords of the used entries (MSB-first ints); ValueError when overpopulated."""
    marker = [0] * 33
    out = []
    for e, ln in enumerate(lengths):
        if not ln:
            continue
        entry = marker[ln]
        if entry >> ln:
            raise bits.bad('codebook %d codeword lengths' % b, 'the tree is overpopulated at entry %d' % e)
        out.append((e, ln, entry))
        for j in range(ln, 0, -1):
            if marker[j] & 1:
                marker[j] = marker[1] + 1 if j == 1 else marker[j - 1] << 1
                break
            marker[j] += 1
        for j in range(ln + 1, 33):
            if (marker[j] >> 1) == entry:
                entry = marker[j]
                marker[j] = marker[j - 1] << 1
            else:
                break
    return out


def _book(br, b):
    if br.read(24, 'codebook %d sync pattern' % b) != 0x564342:
        raise br.bad('codebook %d sync pattern' % b, 'not BCV')
    dims, entries = br.read(16, 'codebook %d dimensions' % b), br.read(24, 'codebook %d entries' % b)
    if br.read(1, 'codebook %d ordered flag' % b):
        cur, ln, lengths = 0, br.read(5, 'codebook %d lengths' % b) + 1, []
        while cur < entries:
            num = br.read(_ilog(entries - cur), 'codebook %d lengths' % b)
            if cur + num > entries or ln > 32:
                raise br.bad('codebook %d ordered lengths' % b, 'they run past the entries')
            lengths += [ln] * num
            cur += num
            ln += 1
    else:
        sparse = br.read(1, 'codebook %d sparse flag' % b)
        lengths = []
        for _ in range(entries):
            if sparse and not br.read(1, 'codebook %d lengths' % b):
                lengths.append(0)
            else:
                lengths.append(br.read(5, 'codebook %d lengths' % b) + 1)
    lookup = br.read(4, 'codebook %d lookup type' % b)
    vectors = None
    if lookup in (1, 2):
        minv = _float32(br.read(32, 'codebook %d minimum value' % b))
        delta = _float32(br.read(32, 'codebook %d delta value' % b))
        vbits, seqp = br.read(4, 'codebook %d value bits' % b) + 1, br.read(1, 'codebook %d sequence_p' % b)
        if dims == 0:
            raise br.bad('codebook %d dimensions' % b, 'a VQ book of 0 dimensions')
        nvals = _lookup1_values(entries, dims) if lookup == 1 else entries * dims
        if br.pos + nvals * vbits > br.n:
            raise ValueError('%s: the setup header ends inside codebook %d multiplicands' % (br.name, b))
        mults = np.array([br.read(vbits, '') for _ in range(nvals)], np.float64)
        e = np.arange(entries)
        if lookup == 1:
            offs = (e[:, None] // (nvals ** np.arange(dims))[None, :]) % max(nvals, 1)
        else:
            offs = e[:, None] * dims + np.arange(dims)[None, :]
        vectors = mults[offs] * delta + minv if nvals else np.zeros((entries, dims))
        if seqp:   # each value adds the one before it in the vector
            vectors = np.cumsum(vectors, axis=1)
    elif lookup:
        raise br.bad('codebook %d lookup type' % b, 'type %d' % lookup)
    used = [(e, ln) for e, ln in enumerate(lengths) if ln]
    return dict(dims=dims, entries=entries, lengths=lengths, lookup=lookup, vectors=vectors,
                codes=_codes(lengths, br, b) if len(used) != 1 else [(used[0][0], used[0][1], 0)],
                single=used[0][0] if len(used) == 1 else -1)


def parse_headers(ident, setup, name):
    """The identification and setup headers -> dict (channels, rate, bs, books, floors, residues, mappings, modes)."""
    br = _Bits(ident, name, 'identification')
    if len(ident) < 30 or ident[:7] != b'\x01vorbis':
        raise br.bad('packet type', 'not a Vorbis identification header')
    br.pos = 56
    if br.read(32, 'vorbis_version'):
        raise br.bad('vorbis_version', 'not 0')
    C, rate = br.read(8, 'audio_channels'), br.read(32, 'audio_sample_rate')
    if C > 2:
        raise ValueError('%s: %d channels are not supported (1 or 2 only)' % (name, C))
    if C == 0 or rate == 0:
        raise br.bad('audio_channels' if not C else 'audio_sample_rate', 'zero')
    br.read(96, 'bitrates')
    e0, e1 = br.read(4, 'blocksize_0'), br.read(4, 'blocksize_1')
    if not 6 <= e0 <= e1 <= 13:
        raise br.bad('blocksize_0 / blocksize_1', '%d and %d (64 <= blocksize_0 <= blocksize_1 <= 8192)' % (1 << e0,
                                                                                                        1 << e1))
    if not br.read(1, 'framing bit'):
        raise br.bad('framing bit', 'not set')
    br = _Bits(setup, name, 'setup')
    if len(setup) < 7 or setup[:7] != b'\x05vorbis':
        raise br.bad('packet type', 'not a Vorbis setup header')
    br.pos = 56
    books = [_book(br, b) for b in range(br.read(8, 'codebook count') + 1)]
    nb = len(books)
    for i in range(br.read(6, 'time count') + 1):
        if br.read(16, 'time %d type' % i):
            raise br.bad('time %d type' % i, 'not 0')
    floors = []
    for f in range(br.read(6, 'floor count') + 1):
        t = br.read(16, 'floor %d type' % f)
        if t == 0:
            raise ValueError('%s: floor type 0 (LSP) is not supported (floor 1 only)' % name)
        if t != 1:
            raise br.bad('floor %d type' % f, 'type %d' % t)
        pcl = [br.read(4, 'floor %d partition classes' % f) for _ in range(br.read(5, 'floor %d partitions' % f))]
        classes = []
        for c in range((max(pcl) + 1) if pcl else 0):
            dim, sub = br.read(3, 'floor %d class dimensions' % f) + 1, br.read(2, 'floor %d class subclasses' % f)
            master = br.read(8, 'floor %d masterbook' % f) if sub else -1
            sbooks = [br.read(8, 'floor %d subclass books' % f) - 1 for _ in range(1 << sub)]
            for bk in [master] + sbooks:
                if bk >= nb:
                    raise br.bad('floor %d class %d books' % (f, c), 'book %d of %d' % (bk, nb))
            classes.append(dict(dim=dim, sub=sub, master=master, books=sbooks))
        mult, rb = br.read(2, 'floor %d multiplier' % f) + 1, br.read(4, 'floor %d rangebits' % f)
        X = [0, 1 << rb]
        for c in pcl:
            X += [br.read(rb, 'floor %d X list' % f) for _ in range(classes[c]['dim'])]
        if len(X) > 65:
            raise br.bad('floor %d X list' % f, '%d values (65 at most)' % len(X))
        if len(set(X)) != len(X):
            raise br.bad('floor %d X list' % f, 'a repeated X value')
        floors.append(dict(parts=pcl, classes=classes, mult=mult, X=X))
    residues = []
    for r in range(br.read(6, 'residue count') + 1):
        t = br.read(16, 'residue %d type' % r)
        if t > 2:
            raise br.bad('residue %d type' % r, 'type %d' % t)
        rs = dict(type=t, begin=br.read(24, 'residue %d begin' % r), end=br.read(24, 'residue %d end' % r),
                  psize=br.read(24, 'residue %d partition size' % r) + 1,
                  nclass=br.read(6, 'residue %d classifications' % r) + 1,
                  classbook=br.read(8, 'residue %d classbook' % r))
        if rs['classbook'] >= nb:
            raise br.bad('residue %d classbook' % r, 'book %d of %d' % (rs['classbook'], nb))
        casc = []
        for _ in range(rs['nclass']):
            low, hb = br.read(3, 'residue %d cascade' % r), br.read(1, 'residue %d cascade' % r)
            casc.append(low | (br.read(5, 'residue %d cascade' % r) << 3 if hb else 0))
        rs['books'] = [[br.read(8, 'residue %d books' % r) if c >> j & 1 else -1 for j in range(8)] for c in casc]
        for bks in rs['books']:
            for bk in bks:
                if bk >= nb:
                    raise br.bad('residue %d books' % r, 'book %d of %d' % (bk, nb))
                if bk >= 0 and (books[bk]['lookup'] == 0 or rs['psize'] % books[bk]['dims']):
                    raise br.bad('residue %d books' % r, 'book %d is not a VQ book that divides the partition size '
                                 '%d' % (bk, rs['psize']))
        if books[rs['classbook']]['dims'] == 0:
            raise br.bad('residue %d classbook' % r, 'a book of 0 dimensions')
        residues.append(rs)
    mappings = []
    for m in range(br.read(6, 'mapping count') + 1):
        if br.read(16, 'mapping %d type' % m):
            raise br.bad('mapping %d type' % m, 'not 0')
        subs = br.read(4, 'mapping %d submaps' % m) + 1 if br.read(1, 'mapping %d submaps flag' % m) else 1
        coupling = []
        if br.read(1, 'mapping %d coupling flag' % m):
            for _ in range(br.read(8, 'mapping %d coupling steps' % m) + 1):
                mg = br.read(_ilog(C - 1), 'mapping %d magnitude' % m)
                an = br.read(_ilog(C - 1), 'mapping %d angle' % m)
                if mg == an or mg >= C or an >= C:
                    raise br.bad('mapping %d coupling' % m, 'magnitude %d, angle %d of %d channels' % (mg, an, C))
                coupling.append((mg, an))
        if br.read(2, 'mapping %d reserved' % m):
            raise br.bad('mapping %d reserved field' % m, 'not 0')
        mux = [br.read(4, 'mapping %d mux' % m) for _ in range(C)] if subs > 1 else [0] * C
        if max(mux) >= subs:
            raise br.bad('mapping %d mux' % m, 'submap %d of %d' % (max(mux), subs))
        sm = []
        for _ in range(subs):
            br.read(8, 'mapping %d submap time' % m)
            fl, rs = br.read(8, 'mapping %d submap floor' % m), br.read(8, 'mapping %d submap residue' % m)
            if fl >= len(floors) or rs >= len(residues):
                raise br.bad('mapping %d submap' % m, 'floor %d, residue %d' % (fl, rs))
            sm.append((fl, rs))
        mappings.append(dict(coupling=coupling, mux=mux, submaps=sm))
    modes = []
    for i in range(br.read(6, 'mode count') + 1):
        bf = br.read(1, 'mode %d blockflag' % i)
        if br.read(16, 'mode %d windowtype' % i) or br.read(16, 'mode %d transformtype' % i):
            raise br.bad('mode %d window / transform type' % i, 'not 0')
        mp = br.read(8, 'mode %d mapping' % i)
        if mp >= len(mappings):
            raise br.bad('mode %d mapping' % i, 'mapping %d of %d' % (mp, len(mappings)))
        modes.append((bf, mp))
    if not br.read(1, 'framing bit'):
        raise br.bad('framing bit', 'not set')
    return dict(channels=C, rate=rate, bs=(1 << e0, 1 << e1), books=books, floors=floors, residues=residues,
                mappings=mappings, modes=modes)


def flatten(S):
    """The setup as csrc/vorbis.cu reads it: one int32 array -> (array, total codewords)."""
    books = S['books']
    rows, codes, info, vecs = [], [], [], []
    nvec = 0
    for b in books:
        cs = sorted((c << (32 - ln), e, ln) for e, ln, c in b['codes'])
        rows.append([b['dims'], b['entries'], len(codes), len(cs), nvec if b['vectors'] is not None else -1,
                     b['single'], 0, 0])
        codes += [c for c, _, _ in cs]
        info += [(e << 6) | ln for _, e, ln in cs]
        if b['vectors'] is not None:
            vecs.append(b['vectors'].astype(np.float32).ravel())
            nvec += b['vectors'].size
    fl_words = []
    for f in S['floors']:
        w = np.full(FLOOR_WORDS, 0, np.int64)
        X = f['X']
        w[0], w[1], w[2], w[3] = len(f['parts']), f['mult'], len(X), FLOOR1_RANGE[f['mult'] - 1]
        w[FL_PART_CLASS:FL_PART_CLASS + len(f['parts'])] = f['parts']
        for c, cl in enumerate(f['classes']):
            w[FL_CLASS_DIM + c], w[FL_CLASS_SUB + c], w[FL_CLASS_MASTER + c] = cl['dim'], cl['sub'], cl['master']
            w[FL_SUB_BOOKS + 8 * c:FL_SUB_BOOKS + 8 * c + len(cl['books'])] = cl['books']
        w[FL_X:FL_X + len(X)] = X
        w[FL_ORDER:FL_ORDER + len(X)] = np.argsort(X, kind='stable')
        for i in range(2, len(X)):
            w[FL_ORDER + 65 + i] = max((j for j in range(i) if X[j] < X[i]), key=lambda j: X[j])
            w[FL_ORDER + 130 + i] = min((j for j in range(i) if X[j] > X[i]), key=lambda j: X[j])
        fl_words.append(w)
    rs_words = []
    for r in S['residues']:
        w = np.full(RES_WORDS, -1, np.int64)
        w[:6] = [r['type'], r['begin'], r['end'], r['psize'], r['nclass'], r['classbook']]
        w[6:6 + 8 * len(r['books'])] = np.ravel(r['books'])
        rs_words.append(w)
    mp_words = []
    for m in S['mappings']:
        w = np.zeros(MAP_WORDS, np.int64)
        w[0], w[1] = len(m['submaps']), len(m['coupling'])
        w[2:2 + len(m['mux'])] = m['mux']
        for s, (f, r) in enumerate(m['submaps']):
            w[4 + s], w[20 + s] = f, r
        if m['coupling']:
            w[36:36 + 2 * len(m['coupling'])] = np.ravel(m['coupling'])
        mp_words.append(w)
    parts = [np.zeros(HDR_WORDS, np.int64), np.ravel(rows).astype(np.int64), np.array(codes, np.uint32).view(np.int32),
             np.array(info, np.uint32).view(np.int32),
             np.concatenate(vecs).view(np.int32) if vecs else np.zeros(0, np.int32)] + fl_words + rs_words + mp_words \
        + [np.ravel(S['modes']).astype(np.int64)]
    offs = np.cumsum([0] + [len(p) for p in parts])
    nf, nr, nm = len(fl_words), len(rs_words), len(mp_words)
    hdr = parts[0]
    hdr[:] = [S['channels'], S['bs'][0], S['bs'][1], len(books), offs[1], offs[2], offs[3], offs[4], len(S['floors']),
              offs[5], offs[5 + nf], offs[5 + nf + nr], len(S['modes']), offs[5 + nf + nr + nm], len(codes),
              _ilog(len(S['modes']) - 1)]
    return np.concatenate([p.astype(np.int64) for p in parts]).astype(np.int32), len(codes)


def pages(data, name):
    """[(byte offset, header type, granule, serial, sequence number, lacing values (uint8 array), body start)] of every
    page; ValueError for a missing capture pattern, a page cut short or a CRC that does not match."""
    out, o, n = [], 0, len(data)
    mv = memoryview(data)
    k = 0
    while o < n:
        if data[o:o + 4] != b'OggS':
            raise ValueError('%s: no Ogg capture pattern at byte %d (page %d)' % (name, o, k))
        if o + 27 > n:
            raise ValueError('%s: page %d (byte %d) is cut short' % (name, k, o))
        ver, htype, gran, serial, seq, crc, nseg = struct.unpack_from('<BBqIIIB', data, o + 4)
        if ver:
            raise ValueError('%s: page %d (byte %d) has stream structure version %d' % (name, k, o, ver))
        lac = np.frombuffer(data, np.uint8, nseg, o + 27) if o + 27 + nseg <= n else None
        end = o + 27 + nseg + (int(lac.sum(dtype=np.int64)) if lac is not None else 0)
        if lac is None or end > n:
            raise ValueError('%s: page %d (byte %d) is cut short' % (name, k, o))
        page = bytearray(mv[o:end])
        page[22:26] = b'\0\0\0\0'
        if ogg_crc(page) != crc:
            raise ValueError('%s: page %d (byte %d) fails its CRC check' % (name, k, o))
        out.append((o, htype, gran, serial, seq, lac, o + 27 + nseg))
        o = end
        k += 1
    return out


def parse(src, name=None):
    """The Ogg Vorbis stream of a file (path or bytes) -> dict(channels, rate, setup (the parsed headers), headers
    (the three header packets' bytes), body (the audio packets' bytes back to back, uint8), offsets (int64: the byte
    offset in the file where each audio packet begins), sizes (int64: each audio packet's size), granules (int64, per
    audio packet: the granule position of the page it ends on, -1 where a later packet ends on the same page), eos
    (the stream's end-of-stream page was read)).  ValueError for anything out of scope."""
    src_name, data = codec.source(src)
    name = name or src_name
    pg = pages(data, name)
    serial, done = None, False
    sizes, starts, grans, pieces = [], [], [], []
    carry, carry_start = 0, -1
    for (o, htype, gran, ser, seq, lac, body) in pg:
        if htype & 2:
            is_vorbis = data[body:body + 7] == b'\x01vorbis'
            if serial is None and is_vorbis:
                serial = ser
            elif is_vorbis and done:
                raise ValueError('%s: a chained stream (a second Vorbis stream begins at byte %d) is not supported' %
                                 (name, o))
        if ser != serial or serial is None:
            continue
        if done:
            continue
        if bool(htype & 1) != (carry > 0 or carry_start >= 0):
            if htype & 1:
                raise ValueError('%s: page at byte %d continues a packet that no page began' % (name, o))
            raise ValueError('%s: page at byte %d does not continue the packet the page before left open' % (name, o))
        lac = lac.astype(np.int64)
        cs = np.cumsum(lac)
        ends = np.flatnonzero(lac < 255)
        pieces.append((body, body + int(cs[-1]) if len(cs) else body))
        prev_end = 0
        for k, e in enumerate(ends):
            size = int(cs[e]) - prev_end + carry
            starts.append(carry_start if carry_start >= 0 else body + prev_end)
            sizes.append(size)
            grans.append(gran if k == len(ends) - 1 else -1)
            prev_end = int(cs[e])
            carry, carry_start = 0, -1
        tail = (int(cs[-1]) if len(cs) else 0) - prev_end
        if tail or (len(lac) and lac[-1] == 255):
            if carry_start < 0:
                carry_start = body + prev_end
            carry += tail
        if htype & 4:
            done = True
    if serial is None:
        raise ValueError('%s: no Vorbis stream (no beginning-of-stream page with a Vorbis identification header)' %
                         name)
    if len(sizes) < 3:
        raise ValueError('%s: the Vorbis stream ends before its three headers' % name)
    body = np.frombuffer(b''.join(bytes(data[a:b]) for a, b in pieces), np.uint8)
    sizes = np.asarray(sizes, np.int64)
    offs_in_body = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    headers = [bytes(body[offs_in_body[i]:offs_in_body[i] + sizes[i]]) for i in range(3)]
    if headers[1][:7] != b'\x03vorbis':
        raise ValueError('%s: malformed comment header: packet type (not a Vorbis comment header)' % name)
    S = parse_headers(headers[0], headers[2], name)
    return dict(channels=S['channels'], rate=S['rate'], setup=S, headers=headers, body=body[offs_in_body[3]:]
                if len(sizes) > 3 else np.zeros(0, np.uint8), offsets=np.asarray(starts[3:], np.int64),
                sizes=sizes[3:], granules=np.asarray(grans[3:], np.int64), eos=done)


def packet_modes(body, sizes, S):
    """(block flag, previous and next window flags, mapping, status) of every audio packet, from its first 2 bytes."""
    sizes = np.asarray(sizes, np.int64)
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    b0 = np.where(sizes > 0, body[np.minimum(offs, max(len(body) - 1, 0))] if len(body) else 0, 0).astype(np.int64)
    b1 = np.where(sizes > 1, body[np.minimum(offs + 1, max(len(body) - 1, 0))] if len(body) else 0, 0).astype(np.int64)
    w = b0 | (b1 << 8)
    mb = _ilog(len(S['modes']) - 1)
    modes = (w >> 1) & ((1 << mb) - 1)
    table = np.array(S['modes'], np.int64).reshape(-1, 2)
    ok_mode = modes < len(table)
    bf = np.where(ok_mode, table[np.minimum(modes, len(table) - 1), 0], 0)
    mapping = np.where(ok_mode, table[np.minimum(modes, len(table) - 1), 1], 0)
    prev, nxt = ((w >> (1 + mb)) & 1) * bf, ((w >> (2 + mb)) & 1) * bf
    need = 1 + mb + 2 * bf
    status = np.zeros(len(sizes), np.int64)
    status[~ok_mode] = 2 << 40 | 1
    status[w & 1 == 1] = 1 << 40
    status[8 * sizes < need] = 5 << 40
    return bf, prev, nxt, mapping, status


def layout(bf, bs, C):
    """Block sizes -> (output end of each packet, its spectrum slot offset in floats, slot floats in all)."""
    n = np.where(bf == 1, bs[1], bs[0]).astype(np.int64)
    ret = np.zeros(len(n), np.int64)
    ret[1:] = n[:-1] // 4 + n[1:] // 4
    end = np.cumsum(ret)
    slot = np.concatenate([[0], np.cumsum(C * n // 2)[:-1]]) if len(n) else np.zeros(0, np.int64)
    return end, slot, int(C * n.sum() // 2)


def trim_range(t, end):
    """[a, b) of the decoded samples that the granule positions keep (appendix A)."""
    total = int(end[-1]) if len(end) else 0
    g = t['granules']
    done = np.flatnonzero(g >= 0)
    if not len(done):
        return 0, total
    first, last = int(done[0]), int(done[-1])
    eos = t['eos'] and last == len(g) - 1
    # granule position of output sample 0 (when one page holds every packet, its granule position is the end's)
    base = 0 if eos and first == last else int(g[first]) - int(end[first])
    a = max(0, -base)
    b = total
    if eos:
        b = min(total, int(g[last]) - base)
    return min(a, total), max(min(a, total), b)


def gather(t):
    """The audio packets' bytes back to back (as parse left them) and their byte offsets in that buffer."""
    sizes = t['sizes']
    return t['body'], np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)


def decode(src, device=None):
    """Ogg Vorbis file path or bytes -> (CUDA float32 tensor (channels, n), sample rate, info).  info: packets (audio
    packets decoded), blocksizes, trimmed_front, kept (samples returned)."""
    import torch
    from . import _native
    name, data = codec.source(src)
    t = parse(data, name)
    S, C = t['setup'], t['channels']
    P = len(t['sizes'])
    dev = codec.cuda_device(name, 'Ogg Vorbis', device)
    if P == 0:
        return torch.zeros((C, 0), dtype=torch.float32, device=dev), t['rate'], dict(packets=0, blocksizes=S['bs'],
                                                                                     trimmed_front=0, kept=0)
    packed, offs = gather(t)
    bf, prev, nxt, mapping, st0 = packet_modes(packed, t['sizes'], S)
    codec.raise_first_bad(st0, t['offsets'], ERRORS, name, 'packet')
    end, slot, slot_floats = layout(bf, S['bs'], C)
    table = np.stack([offs, t['sizes'], end, slot, bf | prev << 1 | nxt << 2 | mapping << 8], axis=1).astype(np.int64)
    blob, n_codes = flatten(S)
    n_out = int(end[-1])
    lib = _native.load_library()
    with torch.cuda.device(dev):
        d_data = torch.from_numpy(np.array(packed) if len(packed) else np.zeros(1, np.uint8)).to(dev)
        d_table = torch.from_numpy(np.ascontiguousarray(table)).to(dev)
        d_setup = torch.from_numpy(blob).to(dev)
        ws_bytes = int(lib.vr_vorbis_workspace(P, C, slot_floats))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        out = torch.empty((C, n_out), dtype=torch.float32, device=dev)
        status = torch.empty(P, dtype=torch.int64, device=dev)
        _native.check(lib, lib.vr_vorbis_decode(None, _native.ptr(d_data), len(packed), _native.ptr(d_table), P,
                                                _native.ptr(d_setup), len(blob), C, n_codes, slot_floats,
                                                _native.ptr(ws), ws_bytes, _native.ptr(out), n_out,
                                                _native.ptr(status), _native.stream_ptr()), 'vr_vorbis_decode')
        st = status.cpu().numpy()
    codec.raise_first_bad(st, t['offsets'], ERRORS, name, 'packet')
    a, b = trim_range(t, end)
    return codec.trim(out, a, b), t['rate'], dict(packets=P, blocksizes=S['bs'], trimmed_front=a, kept=b - a)
