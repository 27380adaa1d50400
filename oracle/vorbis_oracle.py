"""Ogg Vorbis for the tests: a float64 decoder restating the Vorbis I specification for the scope of DESIGN.md §15, a
seeded syntax-level encoder, an Ogg page writer, and ``matrix()``, the streams that cover the scope.

Decoder: ``Decoder(headers).decode(packets) -> float64 (channels, n)`` takes the three header packets and the audio
packets (lib/vorbis.py's ``parse`` reads them out of the pages; the Ogg tests check it against ``ogg`` here).  It
follows the specification's text step by step: codebooks with codewords assigned the lowest-free-leaf way and read bit
by bit (a single-used-entry book sinks zero bits), floor 1 (amplitude unwrap, ``render_point``, the integer
``render_line``, the inverse-dB table), residues 0, 1 and 2, channel coupling, the IMDCT of the block (unnormalised),
the power-sine window with its asymmetric overlaps, and the overlap-add from the centre of one window to the centre of
the next.  An end of packet inside a floor leaves the channel's floor unused; inside a residue it ends the residue
decode with what was added so far kept.  ``Decoder.stats`` counts what the streams exercised.

Encoder: ``encode(x, rate, cfg) -> (headers, packets, blocks)``: a setup built from ``cfg`` (books in every length
encoding and lookup type, floor 1 classes with master and subclass books, a residue of the chosen type with up to 8
cascade passes, one or two submaps, square-polar coupling), MDCT analysis with the Vorbis windows of the chosen block
schedule, a floor 1 fit to the spectral envelope and a cascaded VQ of the residue.  ``ogg`` writes Ogg pages.
"""
import zlib

import numpy as np

INVERSE_DB = np.array([
    1.0649863e-07, 1.1341951e-07, 1.2079015e-07, 1.2863978e-07, 1.369995e-07, 1.459025e-07, 1.5538409e-07,
    1.6548181e-07, 1.7623574e-07, 1.8768856e-07, 1.998856e-07, 2.1287531e-07, 2.2670913e-07, 2.4144197e-07,
    2.5713223e-07, 2.7384212e-07, 2.9163792e-07, 3.1059022e-07, 3.307741e-07, 3.5226967e-07, 3.7516213e-07,
    3.995423e-07, 4.2550681e-07, 4.5315863e-07, 4.8260745e-07, 5.1397001e-07, 5.4737063e-07, 5.8294188e-07,
    6.2082472e-07, 6.6116939e-07, 7.0413591e-07, 7.4989464e-07, 7.9862701e-07, 8.5052631e-07, 9.0579829e-07,
    9.6466215e-07, 1.0273513e-06, 1.0941144e-06, 1.1652161e-06, 1.2409384e-06, 1.3215816e-06, 1.4074654e-06,
    1.4989305e-06, 1.5963394e-06, 1.7000785e-06, 1.8105592e-06, 1.9282195e-06, 2.053526e-06, 2.1869757e-06,
    2.3290977e-06, 2.4804558e-06, 2.6416496e-06, 2.813319e-06, 2.9961443e-06, 3.1908505e-06, 3.3982101e-06,
    3.6190449e-06, 3.8542307e-06, 4.1047006e-06, 4.3714472e-06, 4.6555283e-06, 4.9580708e-06, 5.2802739e-06,
    5.6234162e-06, 5.9888571e-06, 6.3780467e-06, 6.7925284e-06, 7.2339453e-06, 7.7040477e-06, 8.2047e-06,
    8.7378876e-06, 9.3057251e-06, 9.9104636e-06, 1.0554501e-05, 1.1240392e-05, 1.1970856e-05, 1.2748789e-05,
    1.3577278e-05, 1.4459606e-05, 1.5399271e-05, 1.6400005e-05, 1.7465769e-05, 1.8600793e-05, 1.9809577e-05,
    2.1096914e-05, 2.2467912e-05, 2.3928002e-05, 2.5482977e-05, 2.7139005e-05, 2.890265e-05, 3.078091e-05,
    3.2781227e-05, 3.4911533e-05, 3.7180282e-05, 3.9596467e-05, 4.2169668e-05, 4.4910092e-05, 4.7828602e-05,
    5.0936775e-05, 5.4246932e-05, 5.7772202e-05, 6.1526567e-05, 6.552491e-05, 6.9783084e-05, 7.4317984e-05,
    7.9147583e-05, 8.4291038e-05, 8.976875e-05, 9.5602423e-05, 0.00010181521, 0.00010843174, 0.00011547824,
    0.00012298267, 0.00013097477, 0.00013948625, 0.00014855085, 0.00015820454, 0.00016848555, 0.00017943469,
    0.00019109536, 0.00020351382, 0.0002167393, 0.00023082423, 0.00024582449, 0.00026179955, 0.00027881275,
    0.00029693157, 0.00031622787, 0.00033677815, 0.00035866388, 0.00038197188, 0.00040679457, 0.00043323037,
    0.0004613841, 0.00049136748, 0.00052329927, 0.00055730622, 0.00059352309, 0.00063209358, 0.00067317061,
    0.00071691698, 0.00076350628, 0.00081312325, 0.00086596457, 0.00092223985, 0.00098217221, 0.0010459992,
    0.0011139743, 0.0011863665, 0.0012634633, 0.0013455702, 0.0014330129, 0.0015261382, 0.0016253153,
    0.0017309374, 0.0018434235, 0.0019632196, 0.0020908006, 0.0022266726, 0.0023713743, 0.0025254795,
    0.0026895993, 0.0028643848, 0.0030505287, 0.0032487691, 0.0034598925, 0.0036847359, 0.0039241905,
    0.0041792067, 0.0044507948, 0.0047400328, 0.0050480668, 0.0053761187, 0.005725489, 0.0060975635,
    0.0064938175, 0.0069158226, 0.0073652514, 0.0078438874, 0.0083536273, 0.0088964924, 0.009474637,
    0.010090352, 0.01074608, 0.011444421, 0.012188144, 0.012980198, 0.013823725, 0.014722068, 0.015678791,
    0.016697686, 0.017782796, 0.018938422, 0.020169148, 0.021479854, 0.022875736, 0.024362329, 0.025945531,
    0.027631618, 0.029427277, 0.031339627, 0.03337625, 0.035545226, 0.037855156, 0.0403152, 0.042935107,
    0.045725275, 0.048696756, 0.051861349, 0.05523159, 0.058820851, 0.062643364, 0.066714279, 0.07104975,
    0.075666964, 0.080584228, 0.085821047, 0.09139818, 0.097337745, 0.1036633, 0.11039993, 0.11757434,
    0.12521498, 0.13335215, 0.14201812, 0.15124726, 0.16107617, 0.17154381, 0.18269168, 0.19456401, 0.20720787,
    0.22067343, 0.23501402, 0.25028655, 0.26655158, 0.28387362, 0.30232131, 0.32196787, 0.34289113, 0.36517414,
    0.3889052, 0.41417846, 0.44109413, 0.4697589, 0.50028646, 0.53279793, 0.56742209, 0.60429639, 0.64356697,
    0.68538958, 0.72993004, 0.77736503, 0.82788259, 0.88168305, 0.9389798, 1
], np.float32)

FLOOR1_RANGE = {1: 256, 2: 128, 3: 86, 4: 64}


class EndOfPacket(Exception):
    pass


class Malformed(ValueError):
    """An audio packet the decoder rejects: ``code`` is lib/vorbis.py's status code, ``bit`` the bit offset."""
    def __init__(self, code, bit, msg):
        super().__init__(msg)
        self.code, self.bit = code, bit


def ilog(x):
    return int(x).bit_length() if x > 0 else 0


def float32_unpack(x):
    mant = x & 0x1FFFFF
    exp = (x & 0x7FE00000) >> 21
    if x & 0x80000000:
        mant = -mant
    return float(mant) * 2.0 ** (exp - 788)


def float32_pack(v):
    """The exact 32-bit Vorbis float of v (v must have a 21-bit mantissa)."""
    if v == 0:
        return 788 << 21
    sign = v < 0
    m, e = abs(v), 0
    while m != int(m):
        m *= 2
        e -= 1
    m = int(m)
    while m >= 1 << 21:
        assert m & 1 == 0
        m >>= 1
        e += 1
    return (0x80000000 if sign else 0) | ((e + 788) << 21) | m


def lookup1_values(entries, dims):
    """The largest r with r ** dims <= entries, in integers."""
    r = int(round(entries ** (1.0 / dims)))
    while r > 0 and r ** dims > entries:
        r -= 1
    while (r + 1) ** dims <= entries:
        r += 1
    return r


def assign_codes(lengths):
    """The specification's codeword assignment: each used entry in order takes the lowest free leaf of its length.
    -> list of codes (MSB-first ints, None for unused); ValueError when the tree is overpopulated."""
    marker = [0] * 33
    codes = []
    for ln in lengths:
        if not ln:
            codes.append(None)
            continue
        entry = marker[ln]
        if entry >> ln:
            raise ValueError('overpopulated')
        codes.append(entry)
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
    return codes


def ogg_crc_reference(data):
    """Ogg's CRC-32 (polynomial 0x04C11DB7, not reflected, initial value 0), one byte at a time."""
    crc = 0
    for b in data:
        crc ^= b << 24
        for _ in range(8):
            crc = ((crc << 1) ^ 0x04C11DB7) if crc & 0x80000000 else crc << 1
            crc &= 0xFFFFFFFF
    return crc


_REV8 = bytes(int('{:08b}'.format(i)[::-1], 2) for i in range(256))


def ogg_crc(data):
    """The same CRC through zlib on bit-reversed bytes."""
    c = zlib.crc32(bytes(data).translate(_REV8), 0xFFFFFFFF) ^ 0xFFFFFFFF
    return int('{:032b}'.format(c)[::-1], 2)


# ------------------------------------------------------------------------------------------------------------ bits

class Reader:
    """LSB-first bits of a packet; a read past its end raises EndOfPacket."""
    def __init__(self, data):
        self.v = int.from_bytes(bytes(data), 'little')
        self.n = 8 * len(data)
        self.pos = 0

    def read(self, k):
        if self.pos + k > self.n:
            self.pos = self.n + 1
            raise EndOfPacket()
        r = (self.v >> self.pos) & ((1 << k) - 1)
        self.pos += k
        return r


class Writer:
    def __init__(self):
        self.v, self.pos = 0, 0

    def write(self, value, k):
        assert 0 <= value < (1 << k) or k == 0, (value, k)
        self.v |= value << self.pos
        self.pos += k

    def bytes(self):
        return self.v.to_bytes((self.pos + 7) // 8, 'little')


# ------------------------------------------------------------------------------------------------------------ setup

class Book:
    def __init__(self, dims, lengths, lookup=0, minv=0.0, delta=0.0, value_bits=0, seqp=0, mults=()):
        self.dims, self.lengths, self.lookup = dims, list(lengths), lookup
        self.minv, self.delta, self.value_bits, self.seqp, self.mults = minv, delta, value_bits, seqp, list(mults)
        self.entries = len(self.lengths)
        used = [e for e, ln in enumerate(self.lengths) if ln]
        self.single = used[0] if len(used) == 1 else None
        self.codes = assign_codes(self.lengths) if self.single is None else [None] * self.entries
        if self.single is not None:
            self.codes[self.single] = 0
        self.table = {(ln, c): e for e, (ln, c) in enumerate(zip(self.lengths, self.codes)) if ln and c is not None}
        self.prefixes = {(k, c >> (ln - k)) for (ln, c) in self.table for k in range(1, ln + 1)}
        self.vectors = self._vectors()
        self.underpopulated = self.single is None and sum(2.0 ** -ln for ln in self.lengths if ln) < 1.0

    def _vectors(self):
        if self.lookup == 0:
            return None
        out = np.zeros((self.entries, self.dims))
        for e in range(self.entries):
            last, div = 0.0, 1
            for i in range(self.dims):
                if self.lookup == 1:
                    off = (e // div) % len(self.mults)
                    div *= len(self.mults)
                else:
                    off = e * self.dims + i
                v = self.mults[off] * self.delta + self.minv + last
                if self.seqp:
                    last = v
                out[e, i] = v
        return out

    def read(self, br, single_bits=0):
        """The next entry: bit by bit down the tree (a single-used-entry book reads no bit, or ``single_bits``)."""
        if self.single is not None:
            br.read(single_bits)
            return self.single
        code, ln, start = 0, 0, br.pos
        while True:
            code = (code << 1) | br.read(1)
            ln += 1
            if (ln, code) in self.table:
                return self.table[(ln, code)]
            if (ln, code) not in self.prefixes:
                raise Malformed(3, start, 'a codeword that the codebook does not hold')


def read_book(br):
    if br.read(24) != 0x564342:
        raise ValueError('codebook sync pattern')
    dims, entries = br.read(16), br.read(24)
    ordered = br.read(1)
    kind = 'ordered'
    if not ordered:
        sparse = br.read(1)
        kind = 'sparse' if sparse else 'dense'
        lengths = []
        for _ in range(entries):
            if sparse and not br.read(1):
                lengths.append(0)
            else:
                lengths.append(br.read(5) + 1)
    else:
        cur, ln, lengths = 0, br.read(5) + 1, []
        while cur < entries:
            num = br.read(ilog(entries - cur))
            if cur + num > entries:
                raise ValueError('ordered lengths overrun')
            lengths += [ln] * num
            cur += num
            ln += 1
    lookup = br.read(4)
    if lookup == 0:
        b = Book(dims, lengths)
    elif lookup in (1, 2):
        minv, delta = float32_unpack(br.read(32)), float32_unpack(br.read(32))
        vbits, seqp = br.read(4) + 1, br.read(1)
        nvals = lookup1_values(entries, dims) if lookup == 1 else entries * dims
        mults = [br.read(vbits) for _ in range(nvals)]
        b = Book(dims, lengths, lookup, minv, delta, vbits, seqp, mults)
    else:
        raise ValueError('lookup type %d' % lookup)
    b.kind = kind
    return b


def parse_headers(headers):
    """(identification, comment, setup) packets -> setup dict."""
    ident, _, setup = headers
    br = Reader(ident)
    assert br.read(8) == 1 and bytes(ident[1:7]) == b'vorbis'
    br.pos = 7 * 8
    assert br.read(32) == 0
    S = dict(channels=br.read(8), rate=br.read(32))
    br.read(96)
    S['bs'] = (1 << br.read(4), 1 << br.read(4))
    br = Reader(setup)
    assert br.read(8) == 5
    br.pos = 56
    S['books'] = [read_book(br) for _ in range(br.read(8) + 1)]
    for _ in range(br.read(6) + 1):
        assert br.read(16) == 0
    S['floors'] = []
    for _ in range(br.read(6) + 1):
        t = br.read(16)
        if t != 1:
            raise ValueError('floor type %d' % t)
        parts = br.read(5)
        pcl = [br.read(4) for _ in range(parts)]
        classes = []
        for _ in range((max(pcl) + 1) if pcl else 0):
            dim, sub = br.read(3) + 1, br.read(2)
            master = br.read(8) if sub else -1
            books = [br.read(8) - 1 for _ in range(1 << sub)]
            classes.append(dict(dim=dim, sub=sub, master=master, books=books))
        mult, rb = br.read(2) + 1, br.read(4)
        X = [0, 1 << rb]
        for c in pcl:
            X += [br.read(rb) for _ in range(classes[c]['dim'])]
        S['floors'].append(dict(parts=pcl, classes=classes, mult=mult, X=X))
    S['residues'] = []
    for _ in range(br.read(6) + 1):
        t = br.read(16)
        r = dict(type=t, begin=br.read(24), end=br.read(24), psize=br.read(24) + 1, nclass=br.read(6) + 1,
                 classbook=br.read(8))
        casc = []
        for _ in range(r['nclass']):
            low, hb = br.read(3), br.read(1)
            casc.append(low | (br.read(5) << 3 if hb else 0))
        r['books'] = [[br.read(8) if c >> j & 1 else -1 for j in range(8)] for c in casc]
        S['residues'].append(r)
    S['mappings'] = []
    C = S['channels']
    for _ in range(br.read(6) + 1):
        assert br.read(16) == 0
        subs = br.read(4) + 1 if br.read(1) else 1
        coupling = []
        if br.read(1):
            for _ in range(br.read(8) + 1):
                coupling.append((br.read(ilog(C - 1)), br.read(ilog(C - 1))))
        assert br.read(2) == 0
        mux = [br.read(4) for _ in range(C)] if subs > 1 else [0] * C
        sm = []
        for _ in range(subs):
            br.read(8)
            sm.append((br.read(8), br.read(8)))
        S['mappings'].append(dict(coupling=coupling, mux=mux, submaps=sm))
    S['modes'] = []
    for _ in range(br.read(6) + 1):
        bf = br.read(1)
        assert br.read(16) == 0 and br.read(16) == 0
        S['modes'].append(dict(blockflag=bf, mapping=br.read(8)))
    assert br.read(1) == 1
    return S


# ------------------------------------------------------------------------------------------------------------ dsp

def _dct4(X):
    """u[n] = sum_k X[k] cos(pi / M (n + 1/2)(k + 1/2)) through an M/2-point complex FFT."""
    M = len(X)
    k = np.arange(M // 2)
    t = (X[2 * k] + 1j * X[M - 1 - 2 * k]) * np.exp(-1j * np.pi * (4 * k + 1) / (4 * M))
    w = np.fft.fft(t) * np.exp(-1j * np.pi * k / M)
    u = np.empty(M)
    u[2 * k], u[M - 1 - 2 * k] = w.real, -w.imag
    return u


def imdct(X):
    """y[n] = sum_k X[k] cos(pi / M (n + 1/2 + M/2)(k + 1/2)), n < 2M: the DCT-IV of X, unfolded."""
    u = _dct4(np.asarray(X, np.float64))
    M = len(u)
    y = np.empty(2 * M)
    m = np.arange(M)
    y[3 * M // 2 - 1 - m] = -u
    y[m[M // 2:] - M // 2] = u[M // 2:]
    y[m[:M // 2] + 3 * M // 2] = -u[:M // 2]
    return y


def mdct(x):
    """The forward transform whose ``imdct`` overlap-adds back to x under the Vorbis windows: (2 / M) times the
    transpose of ``imdct`` (the input folded, then the DCT-IV, which is symmetric)."""
    x = np.asarray(x, np.float64)
    M = len(x) // 2
    m = np.arange(M)
    f = -x[3 * M // 2 - 1 - m]
    f[M // 2:] += x[m[M // 2:] - M // 2]
    f[:M // 2] -= x[m[:M // 2] + 3 * M // 2]
    return (2.0 / M) * _dct4(f)


def window(n, bs0, blockflag, prev, nxt):
    """The Vorbis window of a block of n samples (the specification's slopes for the flags)."""
    w = np.zeros(n)
    i = np.arange(n)
    if blockflag and not prev:
        ls, le, ln = n // 4 - bs0 // 4, n // 4 + bs0 // 4, bs0 // 2
    else:
        ls, le, ln = 0, n // 2, n // 2
    if blockflag and not nxt:
        rs, re, rn = 3 * n // 4 - bs0 // 4, 3 * n // 4 + bs0 // 4, bs0 // 2
    else:
        rs, re, rn = n // 2, n, n // 2
    a = (i >= ls) & (i < le)
    w[a] = np.sin(np.pi / 2 * np.sin((i[a] - ls + 0.5) / ln * np.pi / 2) ** 2)
    w[(i >= le) & (i < rs)] = 1.0
    b = (i >= rs) & (i < re)
    w[b] = np.sin(np.pi / 2 * np.sin((i[b] - rs + 0.5) / rn * np.pi / 2 + np.pi / 2) ** 2)
    return w


def render_point(x0, y0, x1, y1, x):
    dy, adx = y1 - y0, x1 - x0
    off = abs(dy) * (x - x0) // adx
    return y0 - off if dy < 0 else y0 + off


def render_line(x0, y0, x1, y1, v):
    dy, adx = y1 - y0, x1 - x0
    ady = abs(dy)
    base = int(dy / adx)   # C division: toward zero
    sy = base - 1 if dy < 0 else base + 1
    ady -= abs(base) * adx
    x, y, err = x0, y0, 0
    if x < len(v):
        v[x] = y
    for x in range(x0 + 1, x1):
        err += ady
        if err >= adx:
            err -= adx
            y += sy
        else:
            y += base
        if x < len(v):
            v[x] = y


def floor1_curve(fl, Y, n2):
    """Floor 1 step 2: the amplitude unwrap and the rendered curve (n2 = half the block) -> float64 curve, or None
    when a value leaves the range (status 4)."""
    X, mult = fl['X'], fl['mult']
    rng = FLOOR1_RANGE[mult]
    V = len(X)
    flag = [True, True] + [False] * (V - 2)
    fy = [Y[0], Y[1]] + [0] * (V - 2)
    for i in range(2, V):
        low = max((j for j in range(i) if X[j] < X[i]), key=lambda j: X[j])
        high = min((j for j in range(i) if X[j] > X[i]), key=lambda j: X[j])
        pred = render_point(X[low], fy[low], X[high], fy[high], X[i])
        val, hr, lr = Y[i], rng - pred, pred
        room = 2 * min(hr, lr)
        if val:
            flag[low] = flag[high] = flag[i] = True
            if val >= room:
                fy[i] = val - lr + pred if hr > lr else pred - val + hr - 1
            else:
                fy[i] = pred - (val + 1) // 2 if val & 1 else pred + val // 2
        else:
            fy[i] = pred
    if any(not 0 <= y < rng for y in fy):
        return None
    order = sorted(range(V), key=lambda j: X[j])
    v = np.zeros(n2, np.int64)
    lx, ly, hx, hy = 0, fy[order[0]] * mult, 0, 0
    for j in order[1:]:
        if flag[j]:
            hy, hx = fy[j] * mult, X[j]
            render_line(lx, ly, hx, hy, v)
            lx, ly = hx, hy
    if hx < n2:
        render_line(hx, hy, n2, hy, v)
    return INVERSE_DB.astype(np.float64)[v]


# ------------------------------------------------------------------------------------------------------------ decoder

def new_stats():
    return dict(blocksizes=set(), long_flags=set(), kinds=set(), lookups=set(), underpopulated=0, single=0,
                max_codeword=0, mults=set(), rangebits=set(), unused_subclass=0, residue_types=set(), max_passes=0, clamped=0,
                submaps=set(), coupling=0, eop_floor=0, eop_residue=0, floor_unused=0, channels=set(), rates=set(),
                packets=0)


class Decoder:
    """``zero_magnitude``: the branch inverse coupling takes for a magnitude of exactly 0 - 'negative' is the
    specification's ("greater than zero" fails), 'positive' FFmpeg's (its vector code tests the sign bit), used only
    to pin the rest of the decoder against FFmpeg."""
    def __init__(self, headers, stats=None, zero_magnitude='negative', single_bits=0):
        self.S = parse_headers(headers)
        self.single_bits = single_bits
        self.zero_positive = zero_magnitude == 'positive'
        self.stats = stats if stats is not None else new_stats()
        st, S = self.stats, self.S
        st['channels'].add(S['channels'])
        st['rates'].add(S['rate'])
        for b in S['books']:
            st['kinds'].add(b.kind)
            if b.lookup:
                st['lookups'].add((b.lookup, b.seqp))
            st['underpopulated'] += b.underpopulated
            st['single'] += b.single is not None
            st['max_codeword'] = max([st['max_codeword']] + b.lengths)
        for fl in S['floors']:
            st['mults'].add(fl['mult'])
            st['rangebits'].add(ilog(fl['X'][1]) - 1)
            st['unused_subclass'] += sum(bk < 0 for c in fl['classes'] for bk in c['books'])
        for r in S['residues']:
            st['residue_types'].add(r['type'])
            st['max_passes'] = max([st['max_passes']] + [max((j + 1 for j in range(8) if b[j] >= 0), default=0)
                                                         for b in r['books']])
        for m in S['mappings']:
            st['submaps'].add(len(m['submaps']))
            st['coupling'] += len(m['coupling'])

    def _floor(self, br, fl, n2):
        """-> curve or None (unused)."""
        B = self.S['books']
        rng = FLOOR1_RANGE[fl['mult']]
        try:
            if not br.read(1):
                return None
            Y = [br.read(ilog(rng - 1)), br.read(ilog(rng - 1))]
            for c in fl['parts']:
                cl = fl['classes'][c]
                cval = B[cl['master']].read(br) if cl['sub'] else 0
                for _ in range(cl['dim']):
                    book = cl['books'][cval & ((1 << cl['sub']) - 1)]
                    cval >>= cl['sub']
                    Y.append(B[book].read(br) if book >= 0 else 0)
        except EndOfPacket:
            self.stats['eop_floor'] += 1
            return None
        curve = floor1_curve(fl, Y, n2)
        if curve is None:
            raise Malformed(4, br.pos, 'a floor 1 value leaves the floor\'s range')
        return curve

    def _residue(self, br, r, vecs, skip, n2):
        """Residue decode of format r['type'] into the vectors (float64 arrays of n2) not in skip."""
        B = self.S['books']
        ch = len(vecs)
        if r['type'] == 2:
            if all(skip):
                return
            big = np.zeros(n2 * ch)
            self._residue01(br, r, [big], [False], n2 * ch, 1)
            for j in range(ch):
                vecs[j] += big[j::ch]
            return
        self._residue01(br, r, vecs, skip, n2, r['type'])

    def _residue01(self, br, r, vecs, skip, size, fmt):
        B = self.S['books']
        lb, le = min(r['begin'], size), min(r['end'], size)
        if (lb, le) != (r['begin'], r['end']):
            self.stats['clamped'] += 1
        cb = B[r['classbook']]
        cw = cb.dims
        psize = r['psize']
        nparts = (le - lb) // psize if le > lb else 0
        if nparts == 0:
            return
        cls = [[0] * (nparts + cw) for _ in vecs]
        try:
            for p in range(8):
                pc = 0
                while pc < nparts:
                    if p == 0:
                        for j, v in enumerate(vecs):
                            if skip[j]:
                                continue
                            t = cb.read(br, self.single_bits)
                            for i in range(cw - 1, -1, -1):
                                cls[j][i + pc] = t % r['nclass']
                                t //= r['nclass']
                    for _ in range(cw):
                        if pc >= nparts:
                            break
                        for j, v in enumerate(vecs):
                            if skip[j]:
                                continue
                            bk = r['books'][cls[j][pc]][p]
                            if bk < 0:
                                continue
                            book = B[bk]
                            off = lb + pc * psize
                            if fmt == 0:
                                step = psize // book.dims
                                for i in range(step):
                                    e = book.read(br)
                                    v[off + i + step * np.arange(book.dims)] += book.vectors[e]
                            else:
                                i = 0
                                while i < psize:
                                    e = book.read(br)
                                    v[off + i:off + i + book.dims] += book.vectors[e]
                                    i += book.dims
                        pc += 1
        except EndOfPacket:
            self.stats['eop_residue'] += 1
            raise

    def packet(self, data, prev_long=None):
        """One audio packet -> (blockflag, prev, next, windowed block (channels, n)); Malformed for a bad one."""
        S, st, B = self.S, self.stats, self.S['books']
        C = S['channels']
        br = Reader(data)
        try:
            if br.read(1):
                raise Malformed(1, 0, 'packet type')
            mode = br.read(ilog(len(S['modes']) - 1))
            if mode >= len(S['modes']):
                raise Malformed(2, 1, 'mode number')
            md = S['modes'][mode]
            bf = md['blockflag']
            prev = nxt = 0
            if bf:
                prev, nxt = br.read(1), br.read(1)
        except EndOfPacket:
            raise Malformed(5, 0, 'header cut short')
        n = S['bs'][bf]
        n2 = n // 2
        st['blocksizes'].add(n)
        st['packets'] += 1
        if bf:
            st['long_flags'].add((prev, nxt))
        mp = S['mappings'][md['mapping']]
        floors = []
        for c in range(C):
            fl = S['floors'][mp['submaps'][mp['mux'][c]][0]]
            floors.append(self._floor(br, fl, n2))
        st['floor_unused'] += sum(f is None for f in floors)
        no_res = [f is None for f in floors]
        for m, a in mp['coupling']:
            if not no_res[m] or not no_res[a]:
                no_res[m] = no_res[a] = False
        res = [np.zeros(n2) for _ in range(C)]
        try:
            for s, (_, ri) in enumerate(mp['submaps']):
                chans = [c for c in range(C) if mp['mux'][c] == s]
                self._residue(br, S['residues'][ri], [res[c] for c in chans], [no_res[c] for c in chans], n2)
        except EndOfPacket:
            pass
        for m, a in reversed(mp['coupling']):
            M, A = res[m].copy(), res[a].copy()
            pos = M >= 0 if self.zero_positive else M > 0
            apos = A > 0
            newM = np.where(pos, np.where(apos, M, M + A), np.where(apos, M, M - A))
            newA = np.where(pos, np.where(apos, M - A, M), np.where(apos, M + A, M))
            res[m], res[a] = newM, newA
        w = window(n, S['bs'][0], bf, prev, nxt)
        out = np.zeros((C, n))
        for c in range(C):
            if floors[c] is not None:
                out[c] = imdct(floors[c] * res[c]) * w
        return bf, prev, nxt, out

    def decode(self, packets):
        """Audio packets -> float64 (channels, n): every sample from the centre of the first block to the centre of
        the last (no granule trim)."""
        C = self.S['channels']
        pieces, prev_blk = [], None
        for data in packets:
            _, _, _, blk = self.packet(data)
            if prev_blk is not None:
                n0, n1 = prev_blk.shape[1], blk.shape[1]
                seg = np.zeros((C, n0 // 4 + n1 // 4))
                # previous block's right half from its centre, current block's left half up to its centre
                a = prev_blk[:, n0 // 2:]
                seg[:, :min(len(seg[0]), n0 // 2)] += a[:, :len(seg[0])]
                b = blk[:, :n1 // 2]
                k = min(len(seg[0]), n1 // 2)
                seg[:, len(seg[0]) - k:] += b[:, n1 // 2 - k:]
                pieces.append(seg)
            prev_blk = blk
        return np.concatenate(pieces, axis=1) if pieces else np.zeros((C, 0))


def returned(bs):
    """Samples each packet returns, from the block sizes (the first returns none)."""
    bs = np.asarray(bs, np.int64)
    out = np.zeros(len(bs), np.int64)
    out[1:] = bs[:-1] // 4 + bs[1:] // 4
    return out


# ------------------------------------------------------------------------------------------------------------ encoder

def huffman_lengths(weights):
    """Code lengths of a complete prefix code for the weights (Huffman)."""
    import heapq
    heap = [(float(w), i, [i]) for i, w in enumerate(weights)]
    heapq.heapify(heap)
    lens = [0] * len(weights)
    k = len(weights)
    while len(heap) > 1:
        a, _, la = heapq.heappop(heap)
        b, _, lb = heapq.heappop(heap)
        for i in la + lb:
            lens[i] += 1
        heapq.heappush(heap, (a + b, k, la + lb))
        k += 1
    return lens


def write_book(bw, b, kind):
    bw.write(0x564342, 24)
    bw.write(b.dims, 16)
    bw.write(b.entries, 24)
    if kind == 'ordered':
        bw.write(1, 1)
        ln, cur = b.lengths[0], 0
        bw.write(ln - 1, 5)
        while cur < b.entries:
            num = 0
            while cur + num < b.entries and b.lengths[cur + num] == ln:
                num += 1
            bw.write(num, ilog(b.entries - cur))
            cur += num
            ln += 1
    else:
        bw.write(0, 1)
        bw.write(kind == 'sparse', 1)
        for ln in b.lengths:
            if kind == 'sparse':
                bw.write(ln > 0, 1)
                if ln:
                    bw.write(ln - 1, 5)
            else:
                bw.write(ln - 1, 5)
    bw.write(b.lookup, 4)
    if b.lookup:
        bw.write(float32_pack(b.minv), 32)
        bw.write(float32_pack(b.delta), 32)
        bw.write(b.value_bits - 1, 4)
        bw.write(b.seqp, 1)
        for m in b.mults:
            bw.write(m, b.value_bits)


def write_code(bw, book, e, single_bits=0):
    """Entry e's codeword; a single-used-entry book writes none (``single_bits``: the single entry written as that
    many zero bits instead, as decoders that read its declared length expect)."""
    if book.single is not None:
        assert e == book.single
        bw.write(0, single_bits)
        return
    ln, c = book.lengths[e], book.codes[e]
    bw.write(int('{:0{}b}'.format(c, ln)[::-1], 2), ln)


class _Nearest:
    def __init__(self, book):
        self.book = book
        self.used = np.array([e for e in range(book.entries) if book.lengths[e]])
        self.vec = book.vectors[self.used]

    def __call__(self, Q):
        d = ((Q[:, None, :] - self.vec[None]) ** 2).sum(-1)
        return self.used[np.argmin(d, axis=1)]


def _shuffled(rng, lens):
    lens = list(lens)
    rng.shuffle(lens)
    return lens


def build_setup(cfg, C):
    """Books, floors, residues, mappings and modes for cfg -> (setup dict as parse_headers gives it, kinds)."""
    rng = np.random.RandomState(cfg.get('seed', 0) + 1000)
    e0, e1 = cfg.get('bs', (8, 11))
    books, kinds = [], []

    def add(b, kind):
        books.append(b)
        kinds.append(kind)
        return len(books) - 1
    m4 = add(Book(1, _shuffled(rng, [1, 2, 3, 3])), 'dense')
    m64 = add(Book(1, [6] * 64), 'ordered')
    b16 = add(Book(1, [2, 2, 3, 3, 5, 5, 5, 5, 6, 6, 6, 6, 6, 6, 6, 6]), 'ordered')
    b256 = add(Book(1, huffman_lengths(1.0 / (1.0 + np.arange(256)) + rng.rand(256) * 0.01)), 'dense')
    skew = _shuffled(rng, list(range(1, 33)) + [32]) + [0] * 7
    skew = _shuffled(rng, skew)
    bskew = add(Book(1, skew), 'sparse')
    if cfg.get('single_classbook'):
        cbook = add(Book(2, [0] * 8 + [1]), 'sparse')
    else:
        cbook = add(Book(2, huffman_lengths([1, 2, 4, 2, 3, 6, 4, 6, 12])), 'dense')
    g = np.arange(15) - 7
    vc = add(Book(2, huffman_lengths((1.0 / (1.0 + np.abs(g[:, None]) + np.abs(g[None, :]))).ravel()), 1, -7.0,
                  1.0, 4, 0, range(15)), 'dense')
    # FFmpeg's decoder refuses underpopulated trees and lookup type 2, so the streams that carry them ask for them
    v4 = add(Book(4, [7] * 81 if cfg.get('underpopulated') else huffman_lengths(np.ones(81) + rng.rand(81)), 1, -1.0,
                  1.0, 2, 1, range(3)), 'dense')
    if cfg.get('lookup2'):
        v2f = add(Book(2, huffman_lengths(np.ones(25) + rng.rand(25)), 2, -0.5, 0.25, 3, cfg.get('v2_seqp', 0),
                       [v for i in range(5) for j in range(5) for v in (i, j)]), 'dense')
    else:
        v2f = add(Book(2, huffman_lengths(np.ones(25) + rng.rand(25)), 1, -0.5, 0.25, 3, 0, range(5)), 'dense')
    vf1 = add(Book(1, huffman_lengths([1, 2, 3, 4, 6, 4, 3, 2, 1]), 1, -0.25, 1.0 / 16, 4, 0, range(9)), 'dense')
    mult = cfg.get('mult', 2)
    classes = [dict(dim=2, sub=1, master=m4, books=[b16, b256]),
               dict(dim=3, sub=2, master=m64, books=[-1, b16, b256, bskew]),
               dict(dim=1, sub=0, master=-1, books=[b256])]
    floors = []
    for e in (e0, e1):
        # long_rangebits: the long floor's X range (up to 2^15, past the block: the curve's last segment then runs
        # toward a point beyond the last bin)
        rb = cfg.get('long_rangebits', e - 1) if e == e1 else e - 1
        nparts = min(10, max(1, (1 << rb) // 16))
        pcl = [i % 3 for i in range(nparts)]
        nvals = sum(classes[c]['dim'] for c in pcl)
        xs = set()
        while len(xs) < nvals:
            v = int(np.exp(rng.uniform(0, np.log(1 << rb))))
            if 1 <= v < (1 << rb):
                xs.add(v)
            if len(xs) >= (1 << rb) - 1:
                break
        xs = list(rng.permutation(sorted(xs)))
        nvals = len(xs)
        while sum(classes[c]['dim'] for c in pcl) > nvals:
            pcl.pop()
        xs = xs[:sum(classes[c]['dim'] for c in pcl)]
        floors.append(dict(parts=pcl, classes=classes, mult=mult, X=[0, 1 << rb] + [int(v) for v in xs]))
    cascade = [[-1] * 8, [vc] + [-1] * 7, [v4, vc, v2f, -1, -1, -1, -1, vf1]]
    rtype = cfg.get('rtype', 1)
    residues = []
    two = cfg.get('submaps', 1) == 2 and C == 2
    for e, t in ((e0, rtype), (e1, rtype), (e0, (rtype + 1) % 3), (e1, (rtype + 1) % 3)):
        vc_ = 1 if two else C   # channels of the submap the residue serves
        size = (1 << e) // 2 * (vc_ if t == 2 else 1)
        # clamp: every residue ends where a long block's would, past the end of a short block's vector
        end = (1 << e1) // 2 * (vc_ if t == 2 else 1) if cfg.get('clamp') else size
        residues.append(dict(type=t, begin=cfg.get('begin', 0), end=end,
                             psize=32, nclass=3, classbook=cbook, books=cascade))
    coupling = [(0, 1)] if C == 2 and cfg.get('coupling', True) else []
    mappings = []
    for bf in (0, 1):
        if cfg.get('submaps', 1) == 2 and C == 2:
            mappings.append(dict(coupling=coupling, mux=[0, 1], submaps=[(bf, bf), (bf, 2 + bf)]))
        else:
            mappings.append(dict(coupling=coupling, mux=[0] * C, submaps=[(bf, bf)]))
    modes = [dict(blockflag=0, mapping=0), dict(blockflag=1, mapping=1)]
    return dict(channels=C, bs=(1 << e0, 1 << e1), books=books, floors=floors, residues=residues,
                mappings=mappings, modes=modes), kinds


def write_headers(S, rate, kinds, floor_type=1):
    bw = Writer()
    bw.write(1, 8)
    for ch in b'vorbis':
        bw.write(ch, 8)
    bw.write(0, 32)
    bw.write(S['channels'], 8)
    bw.write(rate, 32)
    bw.write(0, 32)
    bw.write(128000, 32)
    bw.write(0, 32)
    bw.write(ilog(S['bs'][0]) - 1, 4)
    bw.write(ilog(S['bs'][1]) - 1, 4)
    bw.write(1, 1)
    ident = bw.bytes()
    bw = Writer()
    bw.write(3, 8)
    for ch in b'vorbis':
        bw.write(ch, 8)
    vendor = b'vorbis_oracle'
    bw.write(len(vendor), 32)
    for ch in vendor:
        bw.write(ch, 8)
    bw.write(0, 32)
    bw.write(1, 1)
    comment = bw.bytes()
    bw = Writer()
    bw.write(5, 8)
    for ch in b'vorbis':
        bw.write(ch, 8)
    bw.write(len(S['books']) - 1, 8)
    for b, k in zip(S['books'], kinds):
        write_book(bw, b, k)
    bw.write(0, 6)
    bw.write(0, 16)
    bw.write(len(S['floors']) - 1, 6)
    for fl in S['floors']:
        bw.write(floor_type, 16)
        bw.write(len(fl['parts']), 5)
        for c in fl['parts']:
            bw.write(c, 4)
        for c in fl['classes'][:max(fl['parts']) + 1]:
            bw.write(c['dim'] - 1, 3)
            bw.write(c['sub'], 2)
            if c['sub']:
                bw.write(c['master'], 8)
            for bk in c['books']:
                bw.write(bk + 1, 8)
        bw.write(fl['mult'] - 1, 2)
        rb = ilog(fl['X'][1]) - 1
        bw.write(rb, 4)
        for x in fl['X'][2:]:
            bw.write(x, rb)
    bw.write(len(S['residues']) - 1, 6)
    for r in S['residues']:
        bw.write(r['type'], 16)
        bw.write(r['begin'], 24)
        bw.write(r['end'], 24)
        bw.write(r['psize'] - 1, 24)
        bw.write(r['nclass'] - 1, 6)
        bw.write(r['classbook'], 8)
        for bks in r['books']:
            c = sum(1 << j for j in range(8) if bks[j] >= 0)
            bw.write(c & 7, 3)
            bw.write(c >= 8, 1)
            if c >= 8:
                bw.write(c >> 3, 5)
        for bks in r['books']:
            for j in range(8):
                if bks[j] >= 0:
                    bw.write(bks[j], 8)
    C = S['channels']
    bw.write(len(S['mappings']) - 1, 6)
    for m in S['mappings']:
        bw.write(0, 16)
        bw.write(len(m['submaps']) > 1, 1)
        if len(m['submaps']) > 1:
            bw.write(len(m['submaps']) - 1, 4)
        bw.write(bool(m['coupling']), 1)
        if m['coupling']:
            bw.write(len(m['coupling']) - 1, 8)
            for a, b in m['coupling']:
                bw.write(a, ilog(C - 1))
                bw.write(b, ilog(C - 1))
        bw.write(0, 2)
        if len(m['submaps']) > 1:
            for c in m['mux']:
                bw.write(c, 4)
        for f, r in m['submaps']:
            bw.write(0, 8)
            bw.write(f, 8)
            bw.write(r, 8)
    bw.write(len(S['modes']) - 1, 6)
    for md in S['modes']:
        bw.write(md['blockflag'], 1)
        bw.write(0, 16)
        bw.write(0, 16)
        bw.write(md['mapping'], 8)
    bw.write(1, 1)
    return [ident, comment, bw.bytes()]


def _floor_values(fl, target):
    """Coded values for the wanted final Y of every post (in X-list order) -> (Y list, final Y)."""
    X, rng = fl['X'], FLOOR1_RANGE[fl['mult']]
    fy = [target[0], target[1]]
    Y = [target[0], target[1]]
    for i in range(2, len(X)):
        low = max((j for j in range(i) if X[j] < X[i]), key=lambda j: X[j])
        high = min((j for j in range(i) if X[j] > X[i]), key=lambda j: X[j])
        pred = render_point(X[low], fy[low], X[high], fy[high], X[i])
        hr, lr = rng - pred, pred
        room = 2 * min(hr, lr)
        d = target[i] - pred
        if d == 0:
            val = 0
        elif d > 0:
            val = 2 * d if 2 * d < room else d + lr
        else:
            val = 2 * -d - 1 if 2 * -d - 1 < room else -d + hr - 1
        if val:
            if val >= room:
                f = val - lr + pred if hr > lr else pred - val + hr - 1
            else:
                f = pred - (val + 1) // 2 if val & 1 else pred + val // 2
        else:
            f = pred
        assert f == target[i] or val == 0
        Y.append(val)
        fy.append(f)
    return Y


def encode(x, rate, cfg):
    """x: float (channels, n) -> (headers, packets, block sizes, info).  cfg: bs (two exponents), schedule (block
    flags, repeated), mult, rtype, submaps, coupling, clamp, single_classbook, v2_seqp, gain, skew, seed."""
    x = np.atleast_2d(np.asarray(x, np.float64))
    C, N = x.shape
    rs = np.random.RandomState(cfg.get('seed', 0))
    S, kinds = build_setup(cfg, C)
    headers = write_headers(S, rate, kinds)
    B = S['books']
    near = {i: _Nearest(b) for i, b in enumerate(B) if b.lookup}
    bs = S['bs']
    sched = cfg.get('schedule', [1])
    flags = []
    c = 0
    while True:
        flags.append(sched[len(flags) % len(sched)])
        if len(flags) > 1:
            c += bs[flags[-2]] // 4 + bs[flags[-1]] // 4
        if c >= N:
            break
    pad = bs[1]
    xp = np.zeros((C, N + 3 * pad))
    xp[:, pad:pad + N] = x
    gain = cfg.get('gain', 8.0)
    packets, blocks, centre = [], [], 0
    floor_bits = []
    for p, bf in enumerate(flags):
        if p:
            centre += bs[flags[p - 1]] // 4 + bs[bf] // 4
        n = bs[bf]
        n2 = n // 2
        prev = flags[p - 1] if p else bf
        nxt = flags[p + 1] if p + 1 < len(flags) else bf
        w = window(n, bs[0], bf, prev, nxt)
        seg = xp[:, pad + centre - n2:pad + centre + n2] * w
        spec = np.stack([mdct(seg[ch]) for ch in range(C)])
        bw = Writer()
        bw.write(0, 1)
        bw.write(bf, 1)
        if bf:
            bw.write(prev, 1)
            bw.write(nxt, 1)
        mp = S['mappings'][bf]
        curves = []
        for ch in range(C):
            fl = S['floors'][mp['submaps'][mp['mux'][ch]][0]]
            if not np.any(seg[ch]):
                bw.write(0, 1)
                curves.append(None)
                continue
            bw.write(1, 1)
            rng = FLOOR1_RANGE[fl['mult']]
            order = sorted(fl['X'])
            target = []
            for xv in fl['X']:
                k = order.index(xv)
                lo = order[k - 1] if k else 0
                hi = order[k + 1] if k + 1 < len(order) else n2
                a, b = max(0, min(n2 - 1, (lo + xv) // 2)), max(1, min(n2, (xv + hi) // 2 + 1))
                env = np.abs(spec[ch, a:b]).max() if b > a else 0.0
                idx = int(np.searchsorted(INVERSE_DB, env / gain))
                target.append(min(rng - 1, -(-min(idx, 255) // fl['mult'])))
            Y = _floor_values(fl, target)
            bits = ilog(rng - 1)
            bw.write(Y[0], bits)
            bw.write(Y[1], bits)
            o = 2
            for cl_i in fl['parts']:
                cl = fl['classes'][cl_i]
                vals = Y[o:o + cl['dim']]
                o += cl['dim']
                if cl['sub'] == 0:
                    for v in vals:
                        write_code(bw, B[cl['books'][0]], v)
                    continue
                picks = []
                for v in vals:
                    if cl['sub'] == 1:
                        picks.append(0 if v < 16 else 1)
                    elif v == 0:
                        picks.append(0)
                    elif v < 33 and cfg.get('skew') and B[cl['books'][3]].lengths[v]:
                        picks.append(3)
                    else:
                        picks.append(1 if v < 16 else 2)
                cval = sum(pk << (cl['sub'] * j) for j, pk in enumerate(picks))
                write_code(bw, B[cl['master']], cval)
                for v, pk in zip(vals, picks):
                    if cl['books'][pk] >= 0:
                        write_code(bw, B[cl['books'][pk]], v)
            curve = floor1_curve(fl, Y, n2)
            assert curve is not None
            curves.append(curve)
        floor_bits.append(bw.pos)
        no_res = [cv is None for cv in curves]
        for m, a in mp['coupling']:
            if not no_res[m] or not no_res[a]:
                no_res[m] = no_res[a] = False
        res = [spec[ch] / curves[ch] if curves[ch] is not None else np.zeros(n2) for ch in range(C)]
        for m, a in mp['coupling']:
            L, R = res[m], res[a]
            big = np.abs(L) > np.abs(R)
            M = np.where(big, L, R)
            A = np.where(big, np.where(L > 0, L - R, R - L), np.where(R > 0, L - R, R - L))
            res[m], res[a] = M, A
        for s, (_, ri) in enumerate(mp['submaps']):
            chans = [ch for ch in range(C) if mp['mux'][ch] == s]
            _encode_residue(bw, S['residues'][ri], B, near, [res[ch] for ch in chans], [no_res[ch] for ch in chans],
                            n2, rs, cfg)
        packets.append(bw.bytes())
        blocks.append(n)
    return headers, packets, blocks, dict(floor_bits=floor_bits, samples=N)


def _encode_residue(bw, r, B, near, vecs, skip, n2, rs, cfg):
    if r['type'] == 2:
        if all(skip):
            return
        big = np.zeros(n2 * len(vecs))
        for j, v in enumerate(vecs):
            big[j::len(vecs)] = v
        vecs, skip, size, fmt = [big], [False], n2 * len(vecs), 1
    else:
        size, fmt = n2, r['type']
    lb, le = min(r['begin'], size), min(r['end'], size)
    psize = r['psize']
    nparts = (le - lb) // psize if le > lb else 0
    if not nparts:
        return
    cb = B[r['classbook']]
    cw, ncl = cb.dims, r['nclass']
    cls, picks = [], []
    for j, v in enumerate(vecs):
        cj, pj = [], []
        for p in range(nparts):
            off = lb + p * psize
            part = v[off:off + psize].copy()
            m = np.abs(part).max()
            if cb.single is not None:
                k = 2
            else:
                k = 0 if m < 1.0 / 32 else (1 if rs.rand() < 0.25 else 2)
            cj.append(k)
            ents = []
            for ps in range(8):
                bk = r['books'][k][ps]
                if bk < 0:
                    ents.append(None)
                    continue
                d = B[bk].dims
                if fmt == 0:
                    step = psize // d
                    idx = np.arange(step)[:, None] + step * np.arange(d)[None, :]
                else:
                    idx = np.arange(psize).reshape(-1, d)
                e = near[bk](part[idx])
                part[idx] -= B[bk].vectors[e]
                ents.append(e)
            pj.append(ents)
        cls.append(cj)
        picks.append(pj)
    for ps in range(8):
        pc = 0
        while pc < nparts:
            if ps == 0:
                for j in range(len(vecs)):
                    if skip[j]:
                        continue
                    t = 0
                    for i in range(cw):
                        t = t * ncl + (cls[j][pc + i] if pc + i < nparts else 0)
                    if cb.single is not None:
                        t = cb.single
                    write_code(bw, cb, t, cfg.get('single_bits', 0))
            for _ in range(cw):
                if pc >= nparts:
                    break
                for j in range(len(vecs)):
                    if skip[j]:
                        continue
                    bk = r['books'][cls[j][pc]][ps]
                    if bk < 0:
                        continue
                    for e in picks[j][pc][ps]:
                        write_code(bw, B[bk], int(e))
                pc += 1


# ------------------------------------------------------------------------------------------------------------ ogg

def _page(flags, granule, serial, seq, lacing, body, bad_crc=False):
    import struct
    hdr = b'OggS' + struct.pack('<BBqIII', 0, flags, granule, serial, seq, 0) + bytes([len(lacing)]) + bytes(lacing)
    page = bytearray(hdr + body)
    crc = ogg_crc(page) ^ (1 if bad_crc else 0)
    page[22:26] = crc.to_bytes(4, 'little')
    return bytes(page)


def ogg(headers, packets, blocks, serial=0x5EED, segments=255, per_page=None, start=0, end_cut=0, other=None,
        bad_crc_page=None, chain=None, fresh_page=()):
    """Ogg pages of one Vorbis stream -> (bytes, info).  Audio pages hold up to ``segments`` lacing values and
    ``per_page`` packets (a packet longer than the room left continues on the next page).  Granule positions count
    the samples the packets return, from ``start`` (below 0: the first page's granule is below its decoded count and -start
    samples are trimmed from the front); the last page's is ``end_cut`` below the end.  ``other``: packets of a
    second logical stream whose pages are interleaved; a packet in ``fresh_page`` starts a page.  ``chain``:
    (headers, packets, blocks) of a second Vorbis stream after the end of this one.  info: packets and the trims a
    reader must apply, ``spans`` (packets split across pages), ``run_at_end`` (a 255-lacing run ending exactly at a
    page end)."""
    gran = np.cumsum(returned(blocks)) + start
    gran[-1] -= end_cut
    pages, seq = [], 0
    pages.append(_page(2, 0, serial, 0, _lacing(len(headers[0])), headers[0]))
    seq = 1
    lac, body = [], b''
    for h in headers[1:]:
        lac += _lacing(len(h))
        body += h
    while lac:
        pages.append(_page(0, 0, serial, seq, lac[:255], body[:sum(lac[:255])]))
        body = body[sum(lac[:255]):]
        lac = lac[255:]
        seq += 1
    info = dict(spans=0, run_at_end=0, pages_with_many=0)
    cur_lac, cur_body, cur_gran, cont, count = [], b'', -1, False, 0
    queue = [(i, _lacing(len(p)), p) for i, p in enumerate(packets)]
    out_pages = []
    pending = None
    while queue or pending:
        if pending is None:
            i, lv, data = queue.pop(0)
            pending = [i, lv, data]
            if i in fresh_page and cur_lac:
                out_pages.append(_page(1 if cont else 0, cur_gran, serial, seq, cur_lac, cur_body,
                                       bad_crc=seq == bad_crc_page))
                seq += 1
                cont = False
                cur_lac, cur_body, cur_gran, count = [], b'', -1, 0
        i, lv, data = pending
        room = segments - len(cur_lac)
        take = lv[:room]
        cur_lac += take
        nb = sum(take)
        cur_body += data[:nb]
        if len(take) < len(lv):
            pending = [i, lv[len(take):], data[nb:]]
            info['spans'] += 1
        else:
            pending = None
            cur_gran = int(gran[i])
            count += 1
        last = not queue and pending is None
        if len(cur_lac) == segments or last or (per_page and count >= per_page):
            if pending is not None and pending[1] == [0]:
                info['run_at_end'] += 1
            info['pages_with_many'] += count > 3
            out_pages.append(_page((1 if cont else 0) | (4 if last else 0), cur_gran, serial, seq, cur_lac,
                                   cur_body, bad_crc=seq == bad_crc_page))
            seq += 1
            cont = pending is not None
            cur_lac, cur_body, cur_gran, count = [], b'', -1, 0
    if other:
        mixed, osq = [], 0
        opages = []
        for k, p in enumerate(other):
            opages.append(_page(2 if k == 0 else (4 if k == len(other) - 1 else 0), k, serial + 1, osq, _lacing(len(p)),
                                p))
            osq += 1
        pages = pages[:1] + opages[:1] + pages[1:]
        opages = opages[1:]
        for k, p in enumerate(out_pages):
            mixed.append(p)
            if opages and k % 2 == 0:
                mixed.append(opages.pop(0))
        out_pages = mixed + opages
    data = b''.join(pages + out_pages)
    if chain is not None:
        data += ogg(*chain, serial=serial + 7)[0]
    return data, dict(info, packets=len(packets), pages=len(pages) + len(out_pages))


def _lacing(n):
    return [255] * (n // 255) + [n % 255]


# ------------------------------------------------------------------------------------------------------------ matrix

def signal(n, rate, C, seed=0, silent=None):
    """Seeded test signal: sines, noise bursts and clicks, about -10 dBFS; ``silent`` (channel, a, b) zeroes a range."""
    rs = np.random.RandomState(seed)
    t = np.arange(n) / rate
    x = np.zeros((C, n))
    for c in range(C):
        for _ in range(5):
            f = rs.uniform(50, min(rate / 2 - 100, 12000))
            x[c] += rs.uniform(0.02, 0.08) * np.sin(2 * np.pi * f * t + rs.uniform(0, 6))
        env = (np.sin(2 * np.pi * rs.uniform(1, 6) * t) > 0.6).astype(float)
        x[c] += 0.05 * env * rs.randn(n)
        for k in rs.randint(0, n, 3):
            x[c, k:k + 64] += 0.3 * np.hanning(64 if k + 64 <= n else n - k)
    if silent:
        c, a, b = silent
        x[c, a:b] = 0.0
    return x


MATRIX = [
    # name, rate, channels, n, cfg, ogg options
    ('r1_stereo_44k', 44100, 2, 9000, dict(bs=(8, 11), schedule=[1, 1, 0, 0, 1, 0, 1, 1], rtype=1, mult=2, seed=1,
                                            skew=True), dict(per_page=4)),
    ('r0_mono_8k', 8000, 1, 3000, dict(bs=(6, 9), schedule=[1, 0, 1, 1, 0, 0], rtype=0, mult=1, seed=2),
     dict(segments=17)),
    ('r2_stereo_48k', 48000, 2, 9000, dict(bs=(8, 11), schedule=[0, 1, 1, 0], rtype=2, mult=3, seed=3),
     dict(start=-300, end_cut=200, per_page=5)),
    ('submaps_22k', 22050, 2, 6000, dict(bs=(7, 10), schedule=[1, 0, 0, 1], rtype=0, mult=4, seed=4, submaps=2,
                                          coupling=False), dict(other=[b'OpusHead' + bytes(11), b'OpusTags' +
                                                                       bytes(8)] + [bytes(40)] * 9)),
    ('long_8192_96k', 96000, 2, 30000, dict(bs=(9, 13), schedule=[1, 1, 0, 1], rtype=1, mult=2, seed=5),
     dict(start=500, end_cut=1000)),
    ('short_64_11k', 11025, 1, 2000, dict(bs=(6, 6), schedule=[0], rtype=2, mult=3, seed=6), dict(per_page=40)),
    ('single_classbook_32k', 32000, 2, 5000, dict(bs=(8, 10), schedule=[1, 0], rtype=1, mult=2, seed=7,
                                                  single_classbook=True), dict()),
    ('silent_channel_16k', 16000, 2, 6000, dict(bs=(7, 10), schedule=[1, 1, 0], rtype=2, mult=1, seed=8,
                                                silent=(1, 0, 6000)), dict(segments=255)),
    # FFmpeg cannot open these two: lookup type 2 books, an underpopulated tree in the first and residues whose end
    # is clamped to a short block's in the second; nor X values past the block (rangebits 15 on 1024-sample blocks)
    ('lookup2_seqp_12k', 12000, 2, 4000, dict(bs=(7, 9), schedule=[1, 0, 1], rtype=1, mult=2, seed=9, lookup2=True,
                                              v2_seqp=1, underpopulated=True), dict()),
    ('lookup2_24k', 24000, 1, 4000, dict(bs=(7, 10), schedule=[1, 1, 0], rtype=0, mult=3, seed=10, lookup2=True,
                                        clamp=True, long_rangebits=15),
     dict()),
]
# FFmpeg also rejects the spec's zero-bit read of a single-used-entry book (tests/test_vorbis.py pins what it does)
FFMPEG_CANNOT = ('lookup2_seqp_12k', 'lookup2_24k', 'single_classbook_32k')


def matrix(eop=True):
    """[dict(name, data (the .ogg bytes), headers, packets, blocks, rate, channels, ogg info, trim (a, b))]."""
    out = []
    for name, rate, C, n, cfg, opts in MATRIX:
        x = signal(n, rate, C, seed=cfg['seed'], silent=cfg.get('silent'))
        headers, packets, blocks, einfo = encode(x, rate, cfg)
        if name == 'r1_stereo_44k' and eop:
            # end of packet inside a floor (packet 3) and inside a residue (packet 5)
            packets = list(packets)
            packets[3] = packets[3][:max(1, einfo['floor_bits'][3] // 16)]
            packets[5] = packets[5][:(einfo['floor_bits'][5] + 7) // 8 + 20]
        if name == 'r0_mono_8k':
            # a 255-lacing run that ends exactly at a page end: a packet of 17 * 255 bytes behind a page boundary
            packets = list(packets)
            packets[4] = packets[4] + bytes(17 * 255 - len(packets[4]))
            opts = dict(opts, fresh_page=(4,))
        data, info = ogg(headers, packets, blocks, **opts)
        total = int(np.sum(returned(blocks)))
        start, cut = opts.get('start', 0), opts.get('end_cut', 0)
        out.append(dict(name=name, data=data, headers=headers, packets=packets, blocks=blocks, rate=rate, channels=C,
                        info=info, trim=(max(0, -start), total - cut)))
    return out
