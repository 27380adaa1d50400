"""Ogg Vorbis input: the float64 oracle (oracle/vorbis_oracle.py) against FFmpeg, the host Ogg and setup layer
(lib/vorbis.py), and on the GPU the decoder (csrc/vorbis.cu) against the oracle."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import PKG, ROOT

sys.path.insert(0, ROOT)
from oracle import ffmpeg_vorbis as ff  # noqa: E402
from oracle import vorbis_oracle as vo  # noqa: E402

MAX_BOUND = 2.0 ** -14
RMS_BOUND = 2.0 ** -15 / np.sqrt(12.0)
# oracle against FFmpeg's float decoder: the largest difference measured over the matrix is 8.8e-8
FFMPEG_BOUND = 5.0e-7


@pytest.fixture(scope='module')
def matrix():
    return vo.matrix()


def _vorbis():
    sys.path.insert(0, PKG)
    from lib import vorbis
    return vorbis


def _oracle(e, **kw):
    a, b = e['trim']
    return vo.Decoder(e['headers'], **kw).decode(e['packets'])[:, a:b]


def test_inverse_db_table_matches_the_kernel_copy():
    src = open(os.path.join(PKG, 'csrc', 'vorbis.cu')).read()
    body = re.search(r'kVorbisInverseDb\[256\] = \{(.*?)\};', src, re.S).group(1)
    vals = np.array([float(v.rstrip('f')) for v in re.findall(r'[0-9.e+-]+f', body)], np.float32)
    assert vals.shape == (256,) and np.array_equal(vals, vo.INVERSE_DB)
    assert np.all(np.diff(vo.INVERSE_DB) > 0) and vo.INVERSE_DB[255] == 1.0


def test_matrix_covers_the_contract(matrix):
    st = vo.new_stats()
    for e in matrix:
        vo.Decoder(e['headers'], st).decode(e['packets'])
    assert st['blocksizes'] >= {64, 8192} and len(st['blocksizes']) >= 6
    assert st['long_flags'] == {(0, 0), (0, 1), (1, 0), (1, 1)}
    assert st['kinds'] == {'ordered', 'dense', 'sparse'}
    assert st['lookups'] == {(1, 0), (1, 1), (2, 0), (2, 1)}
    assert st['underpopulated'] and st['single'] and st['max_codeword'] == 32 and st['unused_subclass']
    assert 15 in st['rangebits']
    assert st['mults'] == {1, 2, 3, 4} and st['residue_types'] == {0, 1, 2} and st['max_passes'] == 8
    assert st['clamped'] and st['submaps'] == {1, 2} and st['coupling']
    assert st['eop_floor'] and st['eop_residue'] and st['floor_unused'] and st['channels'] == {1, 2}
    info = {e['name']: e['info'] for e in matrix}
    assert sum(i['spans'] for i in info.values()) and sum(i['pages_with_many'] for i in info.values())
    assert sum(i['run_at_end'] for i in info.values()) and any(i['pages'] > 10 for i in info.values())
    assert any(e['trim'][0] > 0 for e in matrix)
    assert any(e['trim'][1] < int(np.sum(vo.returned(e['blocks']))) for e in matrix)


def test_oracle_matches_ffmpeg(matrix):
    """Every stream FFmpeg can open, decoded by both (no trim: FFmpeg runs without a demuxer).  FFmpeg takes a
    coupled magnitude of exactly 0 as positive (the specification: 'greater than zero' fails), so the oracle decodes
    with that convention here.  FFmpeg cannot open lookup type 2 books, underpopulated trees, clamped residue ends or
    floor X values past the block, reads a single-used-entry book's declared length, and does not stop at an end of
    packet, so those streams are pinned against the oracle alone (the EOP stream is compared here without its
    truncated packets)."""
    ok, why = ff.available()
    if not ok:
        pytest.skip('FFmpeg harness unavailable: ' + why)
    eop_free = {e['name']: e for e in vo.matrix(eop=False)}
    for e in matrix:
        if e['name'] in vo.FFMPEG_CANNOT:
            continue
        e = eop_free[e['name']]
        y = vo.Decoder(e['headers'], zero_magnitude='positive').decode(e['packets'])
        f = ff.decode(e['headers'], e['packets'], e['channels']).astype(np.float64)
        assert f.shape == y.shape, e['name']
        assert np.abs(y - f).max() < FFMPEG_BOUND, e['name']


def test_spec_coupling_differs_from_ffmpeg_only_at_zero_magnitude(matrix):
    e = next(e for e in vo.matrix(eop=False) if e['name'] == 'r1_stereo_44k')
    spec = vo.Decoder(e['headers']).decode(e['packets'])
    ffc = vo.Decoder(e['headers'], zero_magnitude='positive').decode(e['packets'])
    assert np.abs(spec - ffc).max() > 1e-3


def test_single_entry_book_pinned_against_ffmpeg():
    """The specification: a book with one used entry sinks zero bits.  FFmpeg reads the entry's declared length
    instead: it rejects the zero-bit stream and decodes the one-bit stream as the oracle does when told to read it."""
    ok, why = ff.available()
    if not ok:
        pytest.skip('FFmpeg harness unavailable: ' + why)
    cfg = dict(bs=(8, 10), schedule=[1, 0], rtype=1, mult=2, seed=7, single_classbook=True)
    x = vo.signal(4000, 32000, 2, seed=3)
    h, p, _, _ = vo.encode(x, 32000, cfg)
    with pytest.raises(RuntimeError):
        ff.decode(h, p, 2)
    h1, p1, _, _ = vo.encode(x, 32000, dict(cfg, single_bits=1))
    y = vo.Decoder(h1, zero_magnitude='positive', single_bits=1).decode(p1)
    assert np.abs(y - ff.decode(h1, p1, 2)).max() < FFMPEG_BOUND


def test_oracle_parses_ffmpeg_encoder_setup():
    ok, why = ff.available()
    if not ok:
        pytest.skip('FFmpeg harness unavailable: ' + why)
    h = ff.encoder_headers(44100, 2)
    S = vo.parse_headers(h)
    assert S['channels'] == 2 and S['rate'] == 44100 and len(S['books']) > 10
    vorbis = _vorbis()
    S2 = vorbis.parse_headers(h[0], h[2], 'ffmpeg')
    assert len(S2['books']) == len(S['books']) and vorbis.flatten(S2)[1] > 0


def test_mdct_and_window_round_trip_through_block_switching():
    rs = np.random.RandomState(0)
    bs = (256, 2048)
    flags = [1, 1, 0, 0, 1, 0, 1, 1, 1]
    centres = np.concatenate([[0], np.cumsum([bs[a] // 4 + bs[b] // 4 for a, b in zip(flags, flags[1:])])])
    n = int(centres[-1])
    x = rs.uniform(-1, 1, n + 4096)
    out = np.zeros(n + 8192)
    pad = 4096
    xp = np.concatenate([np.zeros(pad), x, np.zeros(pad)])
    for p, bf in enumerate(flags):
        N = bs[bf]
        w = vo.window(N, bs[0], bf, flags[p - 1] if p else bf, flags[p + 1] if p + 1 < len(flags) else bf)
        c = int(centres[p]) + pad
        y = vo.imdct(vo.mdct(xp[c - N // 2:c + N // 2] * w)) * w
        out[c - N // 2:c + N // 2] += y
    assert np.abs(out[pad:pad + n] - x[:n]).max() < 1e-12   # measured 1.1e-15


def test_ogg_layer_returns_the_writers_packets_and_trims(matrix):
    vorbis = _vorbis()
    for e in matrix:
        t = vorbis.parse(e['data'])
        offs = np.concatenate([[0], np.cumsum(t['sizes'])[:-1]])
        assert [bytes(t['body'][o:o + s]) for o, s in zip(offs, t['sizes'])] == [bytes(p) for p in e['packets']]
        assert t['headers'] == [bytes(h) for h in e['headers']]
        bf, _, _, _, st = vorbis.packet_modes(t['body'], t['sizes'], t['setup'])
        end, _, _ = vorbis.layout(bf, t['setup']['bs'], t['channels'])
        assert not st.any() and vorbis.trim_range(t, end) == e['trim'], e['name']
    names = {e['name']: e['info'] for e in matrix}
    assert names['r0_mono_8k']['spans'] and names['long_8192_96k']['spans']
    assert names['short_64_11k']['pages_with_many'] and names['r0_mono_8k']['run_at_end']


def test_ogg_crc_identity():
    rs = np.random.RandomState(1)
    vorbis = _vorbis()
    for n in (0, 1, 27, 1000):
        d = rs.bytes(n)
        assert vorbis.ogg_crc(d) == vo.ogg_crc_reference(d) == vo.ogg_crc(d)


def _stream(name):
    return next(e for e in vo.matrix(eop=False) if e['name'] == name)


def test_bad_page_crc_names_the_page():
    e = _stream('r0_mono_8k')
    data, _ = vo.ogg(e['headers'], e['packets'], e['blocks'], segments=17, bad_crc_page=3)
    with pytest.raises(ValueError, match=r'page 3 \(byte \d+\) fails its CRC check'):
        _vorbis().parse(data, 'x.ogg')


@pytest.mark.parametrize('case,msg', [
    ('floor0', 'floor type 0 \\(LSP\\) is not supported'),
    ('channels3', '3 channels are not supported'),
    ('chained', 'a chained stream'),
    ('overpopulated', 'malformed setup header: codebook 0 codeword lengths \\(the tree is overpopulated'),
    ('coupling', 'malformed setup header: mapping 0 coupling'),
    ('mux', 'malformed setup header: mapping 0 mux'),
    ('residue_type', 'malformed setup header: residue 0 type'),
    ('x_repeat', 'malformed setup header: floor 0 X list \\(a repeated X value\\)'),
    ('cut', 'the setup header ends inside'),
])
def test_out_of_scope_and_malformed_setups_raise(case, msg):
    vorbis = _vorbis()
    e = _stream('r1_stereo_44k')
    S, kinds = vo.build_setup(dict(seed=1, bs=(8, 11)), 2)
    h = vo.write_headers(S, 44100, kinds)
    if case == 'floor0':
        h = vo.write_headers(S, 44100, kinds, floor_type=0)
    elif case == 'channels3':
        h = [h[0][:11] + bytes([3]) + h[0][12:], h[1], h[2]]
    elif case == 'overpopulated':
        S['books'][0].lengths = [1, 1, 1, 2]   # three 1-bit codes
        h = vo.write_headers(S, 44100, kinds)
    elif case == 'coupling':
        S['mappings'][0]['coupling'] = [(1, 1)]
        h = vo.write_headers(S, 44100, kinds)
    elif case == 'mux':
        S['mappings'][0]['mux'] = [0, 3]
        S['mappings'][0]['submaps'] = [(0, 0), (0, 0)]
        h = vo.write_headers(S, 44100, kinds)
    elif case == 'residue_type':
        S['residues'][0]['type'] = 3
        h = vo.write_headers(S, 44100, kinds)
    elif case == 'x_repeat':
        S['floors'][0]['X'][3] = S['floors'][0]['X'][2]
        h = vo.write_headers(S, 44100, kinds)
    elif case == 'cut':
        h = [h[0], h[1], h[2][:len(h[2]) // 2]]
    chain = (e['headers'], e['packets'][:3], e['blocks'][:3]) if case == 'chained' else None
    data, _ = vo.ogg(h, e['packets'][:3], e['blocks'][:3], chain=chain)
    with pytest.raises(ValueError, match=msg):
        vorbis.parse(data, 'x.ogg')


def _empty_classbook_stream():
    """r1_stereo_44k with its residue classbook replaced by a book with no used entry, appended last."""
    e = _stream('r1_stereo_44k')
    S, kinds = vo.build_setup(dict(bs=(8, 11), schedule=[1, 1, 0, 0, 1, 0, 1, 1], rtype=1, mult=2, seed=1, skew=True),
                              2)
    S['books'].append(vo.Book(2, [0] * 9))
    kinds.append('sparse')
    for r in S['residues']:
        r['classbook'] = len(S['books']) - 1
    h = vo.write_headers(S, 44100, kinds)
    return e, h


def test_book_without_used_entries_reads_as_a_bad_codeword():
    """A setup may hold a book with no used entry; every read from it is a codeword the book does not hold."""
    vorbis = _vorbis()
    e, h = _empty_classbook_stream()
    with pytest.raises(vo.Malformed) as exc:
        vo.Decoder(h).decode(e['packets'])
    assert exc.value.code == 3
    t = vorbis.parse(vo.ogg(h, e['packets'], e['blocks'])[0])
    blob, n_codes = vorbis.flatten(t['setup'])
    rows = blob[vorbis.HDR_WORDS:vorbis.HDR_WORDS + len(t['setup']['books']) * vorbis.BOOK_WORDS].reshape(-1, 8)
    assert rows[-1][3] == 0 and rows[-1][2] == n_codes and rows[-1][5] == -1


def test_opus_in_ogg_is_not_sniffed(tmp_path):
    vorbis = _vorbis()
    page = vo._page(2, 0, 1, 0, [19], b'OpusHead' + bytes(11))
    (tmp_path / 'a.opus').write_bytes(page)
    e = _stream('short_64_11k')
    (tmp_path / 'a.ogg').write_bytes(e['data'])
    assert not vorbis.sniff(str(tmp_path / 'a.opus')) and vorbis.sniff(str(tmp_path / 'a.ogg'))


def test_header_status_codes_are_read_on_the_host():
    vorbis = _vorbis()
    e = _stream('r1_stereo_44k')
    t = vorbis.parse(e['data'])
    S = dict(t['setup'], modes=t['setup']['modes'] + [(0, 0)])   # 3 modes: 2 mode bits, mode 3 does not exist
    body = np.array([0b110, 1, 0, 0], np.uint8)   # mode 3; an empty packet; the type bit; mode 0 (short)
    _, _, _, _, st = vorbis.packet_modes(body, np.array([1, 0, 1, 2]), S)
    assert list(st >> 40) == [2, 5, 1, 0]


def test_ogg_without_gpu_or_soundfile_says_why(tmp_path, monkeypatch):
    import builtins
    import torch
    sys.path.insert(0, PKG)
    from lib import audio_io
    e = _stream('short_64_11k')
    p = tmp_path / 'a.ogg'
    p.write_bytes(e['data'])
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    real = builtins.__import__

    def no_soundfile(name, *a, **k):
        if name == 'soundfile':
            raise ImportError('no soundfile')
        return real(name, *a, **k)
    monkeypatch.setattr(builtins, '__import__', no_soundfile)
    with pytest.raises(RuntimeError, match='is an Ogg Vorbis file: decoding it needs a CUDA device \\(lib/vorbis.py\\) '
                                           'or the soundfile module'):
        audio_io.load(str(p), sr=44100)


# ------------------------------------------------------------------------------------------------------------ GPU

def _within_bound(y, ref):
    y = y.cpu().numpy().astype(np.float64) if hasattr(y, 'cpu') else np.asarray(y, np.float64)
    assert y.shape == ref.shape, (y.shape, ref.shape)
    d = y - ref
    assert np.isfinite(y).all()
    assert np.abs(d).max() < MAX_BOUND, np.abs(d).max()
    assert np.sqrt(np.mean(d ** 2)) < RMS_BOUND


@pytest.mark.gpu
def test_gpu_decodes_every_matrix_stream(matrix):
    vorbis = _vorbis()
    for e in matrix:
        y, rate, info = vorbis.decode(e['data'])
        assert rate == e['rate'] and info['packets'] == len(e['packets']), e['name']
        assert info['trimmed_front'] == e['trim'][0] and info['kept'] == e['trim'][1] - e['trim'][0]
        _within_bound(y, _oracle(e))


def _tile(gain, seconds=4.0):
    rate = 44100
    x = vo.signal(int(rate * seconds), rate, 2, seed=int(gain))
    cfg = dict(bs=(8, 11), schedule=[1], rtype=2, mult=2, seed=int(gain), gain=gain)
    h, p, b, _ = vo.encode(x, rate, cfg)
    return h, p, b


@pytest.mark.gpu
@pytest.mark.parametrize('gain', [4.0, 32.0])
def test_gpu_decodes_four_minute_track(gain):
    vorbis = _vorbis()
    h, p, b = _tile(gain)
    reps = 60
    data, _ = vo.ogg(h, p * reps, b * reps)
    y, rate, info = vorbis.decode(data)
    ref = vo.Decoder(h).decode(p * 2)
    n = int(np.sum(vo.returned(b * 2))) - int(np.sum(vo.returned(b)))   # one tile's samples after the first
    first = int(np.sum(vo.returned(b)))
    assert info['packets'] == len(p) * reps and y.shape[1] == first + (reps - 1) * n
    _within_bound(y[:, :first + n], ref)
    for t in range(1, reps):
        _within_bound(y[:, first + (t - 1) * n:first + t * n], ref[:, first:])


def _codeword_bits(e, book_index):
    """(packet, bit) of the first codeword read from book ``book_index`` in the stream."""
    d = vo.Decoder(e['headers'])
    book = d.S['books'][book_index]
    seen = []
    real = book.read

    def spy(br, single_bits=0):
        seen.append(br.pos)
        return real(br, single_bits)
    book.read = spy
    for k, p in enumerate(e['packets']):
        seen.clear()
        d.packet(p)
        if seen:
            return k, seen[0], book.lengths
    raise AssertionError('book not used')


def _malformed(decoder, packet):
    try:
        decoder.packet(packet)
    except vo.Malformed:
        return True
    return False


def _set_bits(packet, bit, width, value):
    v = int.from_bytes(packet, 'little')
    v &= ~(((1 << width) - 1) << bit)
    v |= value << bit
    return v.to_bytes(len(packet), 'little')


@pytest.mark.gpu
@pytest.mark.parametrize('case,code', [('type', 1), ('codeword', 3), ('empty_book', 3), ('floor_range', 4),
                                       ('empty', 5)])
def test_gpu_malformed_packets_raise_and_leave_the_decoder_usable(tmp_path, case, code):
    """Each status code, provoked by a bit edit of one packet (an unassigned codeword of an underpopulated book, a
    floor 1 Y0 above the range, the packet type bit), by a residue classbook with no used entry, or by an empty packet:
    a ValueError naming the packet, its byte and the reason; the next call decodes a good file."""
    vorbis = _vorbis()
    if case == 'codeword':
        e = _stream('lookup2_seqp_12k')
        k, bit, lengths = _codeword_bits(e, 7)      # the underpopulated 81-entry book of 7-bit codes
        pk = list(e['packets'])
        pk[k] = _set_bits(pk[k], bit, 7, 0x7F)      # code 1111111 is not assigned
    elif case == 'empty_book':
        e, h = _empty_classbook_stream()          # the last book, with no codes: no read may leave it
        e = dict(e, headers=h)
        pk = list(e['packets'])
        d = vo.Decoder(h)
        k = next(i for i, p in enumerate(pk) if _malformed(d, p))   # the first packet with a used floor
    elif case == 'floor_range':
        e = _stream('r2_stereo_48k')                 # multiplier 3: range 86, 7-bit Y0
        pk = list(e['packets'])
        k = 1
        bf = e['blocks'][k] == 2048
        pk[k] = _set_bits(pk[k], 1 + 1 + (2 if bf else 0) + 1, 7, 127)
    else:
        e = _stream('r1_stereo_44k')
        pk = list(e['packets'])
        k = 2
        pk[k] = bytes([pk[k][0] | 1]) + pk[k][1:] if case == 'type' else b''
    data, _ = vo.ogg(e['headers'], pk, e['blocks'])
    t = vorbis.parse(data)
    path = tmp_path / 'x.ogg'
    path.write_bytes(data)
    with pytest.raises(ValueError, match=r'x\.ogg: packet %d \(byte %d\): %s' % (k, t['offsets'][k],
                                                                                re.escape(vorbis.ERRORS[code]))):
        vorbis.decode(str(path))
    good = _stream('short_64_11k')
    y, _, _ = vorbis.decode(good['data'])
    _within_bound(y, _oracle(good))


def _write_ogg(path, x, rate):
    cfg = dict(bs=(8, 11), schedule=[1, 1, 0, 1], rtype=1 if x.shape[0] == 1 else 2, mult=2, seed=rate)
    h, p, b, _ = vo.encode(x, rate, cfg)
    total = int(np.sum(vo.returned(b)))
    path.write_bytes(vo.ogg(h, p, b, end_cut=total - x.shape[1], per_page=8)[0])


@pytest.mark.gpu
@pytest.mark.parametrize('rate,channels', [(44100, 2), (48000, 2), (44100, 1)])
def test_gpu_audio_io_ogg_equals_decode(tmp_path, rate, channels):
    sys.path.insert(0, PKG)
    from lib import audio_io
    vorbis = _vorbis()
    x = vo.signal(int(rate * 1.5), rate, channels, seed=rate + channels)
    _write_ogg(tmp_path / 'a.ogg', x, rate)
    y, sr = audio_io.load(str(tmp_path / 'a.ogg'), sr=44100, mono=False)
    d, r, info = vorbis.decode(str(tmp_path / 'a.ogg'))
    assert info['kept'] == x.shape[1]
    d = d.cpu().numpy()
    if channels == 1:
        d = d.mean(axis=0)
    if r != 44100:
        d = audio_io.resample(d, r, 44100)
    assert sr == 44100 and y.dtype == np.float32 and np.array_equal(y, d)


@pytest.mark.gpu
def test_gpu_inference_cli_ogg_equals_python_path(tmp_path):
    import torch
    sys.path.insert(0, PKG)
    import inference
    from lib import audio_io, nets, spec_utils, synth
    vorbis = _vorbis()
    x = vo.signal(44100 * 3, 44100, 2, seed=11)
    (tmp_path / 'in').mkdir()
    _write_ogg(tmp_path / 'in' / 'song.ogg', x, 44100)
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
    out = tmp_path / 'out_cli'
    r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt,
                        '-i', str(tmp_path / 'in' / 'song.ogg'), '-o', str(out)],
                       capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 0, r.stderr
    args = inference.build_parser().parse_args(['-P', ckpt, '-i', 'unused'])
    device = torch.device('cuda:0')
    model = nets.CascadedNet(args.n_fft, args.hop_length, 32, 128)
    model.load_state_dict(torch.load(ckpt, map_location='cpu'))
    model.to(device)
    spec_utils.set_device(0)
    X = vorbis.decode(str(tmp_path / 'in' / 'song.ogg'))[0].cpu().numpy()
    sp = inference.Separator(model=model, device=device, batchsize=args.batchsize, cropsize=args.cropsize,
                             postprocess=args.postprocess, wiener_iterations=args.wiener_iterations)
    inst, voc = sp.separate_wave(X)[:2]
    ref = tmp_path / 'out_py'
    ref.mkdir()
    audio_io.write(str(ref / 'song_Instruments.wav'), inst.T, 44100)
    audio_io.write(str(ref / 'song_Vocals.wav'), voc.T, 44100)
    for f in ('song_Instruments.wav', 'song_Vocals.wav'):
        assert (out / f).read_bytes() == (ref / f).read_bytes()


@pytest.mark.gpu
def test_gpu_cache_or_load_on_ogg_pairs(tmp_path):
    sys.path.insert(0, PKG)
    from lib import audio_io, spec_utils
    mix = vo.signal(44100 * 2, 44100, 2, seed=21)
    _write_ogg(tmp_path / 'mix.ogg', mix, 44100)
    _write_ogg(tmp_path / 'inst.ogg', 0.5 * mix, 44100)
    X, y, pm, pi = spec_utils.cache_or_load(str(tmp_path / 'mix.ogg'), str(tmp_path / 'inst.ogg'), 44100, 1024, 2048)
    assert os.path.exists(pm) and os.path.exists(pi)
    a, _ = audio_io.load(str(tmp_path / 'mix.ogg'), sr=44100)
    assert X.shape[0] == 2 and X.shape[1] == 1025 and X.shape[2] == 1 + a.shape[1] // 1024
    X2, y2, _, _ = spec_utils.cache_or_load(str(tmp_path / 'mix.ogg'), str(tmp_path / 'inst.ogg'), 44100, 1024, 2048)
    assert np.array_equal(X, X2) and np.array_equal(y, y2)
