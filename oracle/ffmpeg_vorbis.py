"""FFmpeg's native ``vorbis`` decoder (and encoder) through ctypes: a Vorbis I decoder independent of
oracle/vorbis_oracle.py.

OpenCV's wheel bundles libavcodec and libavutil (``opencv_python_headless.libs``).  The three header packets go in as
the context's extradata (Xiph lacing) through ``avcodec_parameters_alloc`` / ``avcodec_parameters_to_context``:
``codec_type``, ``codec_id``, ``extradata`` and ``extradata_size`` are the leading fields of AVCodecParameters (bytes
0, 4, 16 and 24).  ``decode(headers, packets, channels)`` sends each audio packet and returns the planar float output,
every sample the decoder produces (no demuxer: no granule trim).  The first decoded frame is checked (format
AV_SAMPLE_FMT_FLTP) and the parameters read back after ``avcodec_parameters_from_context`` must hold what was
written; anything else makes the harness report itself unavailable rather than guess.  ``encoder_headers(rate,
channels)`` opens FFmpeg's own (experimental) vorbis encoder and returns its three headers; the sample format goes in
through AVCodecParameters.format (byte 44), which reads -1 before it is set.  ``available()`` is (True, '') or (False,
reason).
"""
import ctypes
import glob
import os

import numpy as np

AV_SAMPLE_FMT_FLTP = 8
AVMEDIA_TYPE_AUDIO = 1
AVERROR_EAGAIN = -11
_OFF_PAR_TYPE, _OFF_PAR_ID, _OFF_PAR_EXTRA, _OFF_PAR_EXTRA_SIZE, _OFF_PAR_FORMAT = 0, 4, 16, 24, 44
_OFF_PKT_DATA = 24
_OFF_FRAME_NB_SAMPLES = 112
_OFF_FRAME_FORMAT = 116

_state = {}


def _load():
    if 'lib' in _state or 'why' in _state:
        return _state.get('lib')
    try:
        import cv2
    except ImportError as e:
        _state['why'] = 'cv2 (which bundles libavcodec) is not importable: %s' % e
        return None
    d = os.path.join(os.path.dirname(os.path.dirname(cv2.__file__)))
    libs = glob.glob(os.path.join(d, 'opencv_python*.libs', 'libavcodec*.so*'))
    utils = glob.glob(os.path.join(d, 'opencv_python*.libs', 'libavutil*.so*'))
    if not libs or not utils:
        _state['why'] = 'no libavcodec / libavutil next to cv2'
        return None
    try:
        util = ctypes.CDLL(utils[0])
        lib = ctypes.CDLL(libs[0])
        util.av_log_set_level(-8)
    except OSError as e:
        _state['why'] = 'libavcodec does not load: %s' % e
        return None
    vp = ctypes.c_void_p
    for name, res, args in (('avcodec_find_decoder_by_name', vp, [ctypes.c_char_p]),
                            ('avcodec_find_encoder_by_name', vp, [ctypes.c_char_p]),
                            ('avcodec_alloc_context3', vp, [vp]), ('avcodec_open2', ctypes.c_int, [vp, vp, vp]),
                            ('avcodec_free_context', None, [ctypes.POINTER(vp)]), ('av_packet_alloc', vp, []),
                            ('av_packet_free', None, [ctypes.POINTER(vp)]),
                            ('av_new_packet', ctypes.c_int, [vp, ctypes.c_int]), ('av_packet_unref', None, [vp]),
                            ('av_frame_alloc', vp, []), ('av_frame_free', None, [ctypes.POINTER(vp)]),
                            ('av_frame_unref', None, [vp]), ('avcodec_send_packet', ctypes.c_int, [vp, vp]),
                            ('avcodec_receive_frame', ctypes.c_int, [vp, vp]),
                            ('avcodec_parameters_alloc', vp, []),
                            ('avcodec_parameters_free', None, [ctypes.POINTER(vp)]),
                            ('avcodec_parameters_to_context', ctypes.c_int, [vp, vp]),
                            ('avcodec_parameters_from_context', ctypes.c_int, [vp, vp])):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    util.av_malloc.restype, util.av_malloc.argtypes = vp, [ctypes.c_size_t]
    util.av_opt_set.restype, util.av_opt_set.argtypes = ctypes.c_int, [vp, ctypes.c_char_p, ctypes.c_char_p,
                                                                      ctypes.c_int]
    if not lib.avcodec_find_decoder_by_name(b'vorbis'):
        _state['why'] = 'this libavcodec has no vorbis decoder'
        return None
    _state['lib'], _state['util'] = lib, util
    return lib


def available():
    lib = _load()
    if lib is None:
        return False, _state['why']
    return True, ''


class Unavailable(RuntimeError):
    pass


def xiph_lace(headers):
    out = bytearray([len(headers) - 1])
    for h in headers[:-1]:
        n = len(h)
        out += bytes([255] * (n // 255) + [n % 255])
    for h in headers:
        out += h
    return bytes(out)


def _unavailable(why):
    _state.pop('lib', None)
    _state['why'] = why
    raise Unavailable(why)


def _context(lib, codec, headers):
    """A decoder context with the headers as extradata, set through AVCodecParameters."""
    vp = ctypes.c_void_p
    util = _state['util']
    ext = xiph_lace(headers)
    par = vp(lib.avcodec_parameters_alloc())
    buf = util.av_malloc(len(ext) + 64)
    ctypes.memset(buf, 0, len(ext) + 64)
    ctypes.memmove(buf, ext, len(ext))
    ctypes.c_int.from_address(par.value + _OFF_PAR_TYPE).value = AVMEDIA_TYPE_AUDIO
    ctypes.c_void_p.from_address(par.value + _OFF_PAR_EXTRA).value = buf
    ctypes.c_int.from_address(par.value + _OFF_PAR_EXTRA_SIZE).value = len(ext)
    ctx = vp(lib.avcodec_alloc_context3(codec))
    rc = lib.avcodec_parameters_to_context(ctx, par)
    back = vp(lib.avcodec_parameters_alloc())
    lib.avcodec_parameters_from_context(back, ctx)
    n = ctypes.c_int.from_address(back.value + _OFF_PAR_EXTRA_SIZE).value
    p = ctypes.c_void_p.from_address(back.value + _OFF_PAR_EXTRA).value
    same = rc >= 0 and n == len(ext) and p and ctypes.string_at(p, n) == ext
    lib.avcodec_parameters_free(ctypes.byref(back))
    lib.avcodec_parameters_free(ctypes.byref(par))
    if not same:
        lib.avcodec_free_context(ctypes.byref(ctx))
        _unavailable('AVCodecParameters does not have the assumed layout (extradata did not round-trip)')
    return ctx


def decode(headers, packets, channels):
    """Header packets and audio packets -> float32 (channels, n), the decoder's whole output."""
    lib = _load()
    if lib is None:
        raise Unavailable(_state['why'])
    vp = ctypes.c_void_p
    codec = lib.avcodec_find_decoder_by_name(b'vorbis')
    ctx = _context(lib, codec, headers)
    pkt, frm = vp(lib.av_packet_alloc()), vp(lib.av_frame_alloc())
    out = [[] for _ in range(channels)]
    try:
        if lib.avcodec_open2(ctx, codec, None) < 0:
            raise RuntimeError('FFmpeg rejected the headers')

        def drain():
            while lib.avcodec_receive_frame(ctx, frm) >= 0:
                nb = ctypes.c_int.from_address(frm.value + _OFF_FRAME_NB_SAMPLES).value
                fmt = ctypes.c_int.from_address(frm.value + _OFF_FRAME_FORMAT).value
                if fmt != AV_SAMPLE_FMT_FLTP or nb < 0 or nb > 8192:
                    _unavailable('the AVFrame layout is not the one assumed (nb_samples %d, format %d)' % (nb, fmt))
                for c in range(channels):
                    p = ctypes.c_void_p.from_address(frm.value + 8 * c).value
                    if nb:
                        out[c].append(np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_float)),
                                                            shape=(nb,)).copy())
                lib.av_frame_unref(frm)

        for p in packets:
            if lib.av_new_packet(pkt, max(1, len(p))) < 0:
                raise MemoryError('av_new_packet')
            ctypes.memmove(ctypes.c_void_p.from_address(pkt.value + _OFF_PKT_DATA).value, bytes(p), len(p))
            rc = lib.avcodec_send_packet(ctx, pkt)
            lib.av_packet_unref(pkt)
            if rc < 0 and rc != AVERROR_EAGAIN:
                raise RuntimeError('vorbis rejected a packet (error %d)' % rc)
            drain()
        lib.avcodec_send_packet(ctx, None)
        drain()
    finally:
        lib.av_frame_free(ctypes.byref(frm))
        lib.av_packet_free(ctypes.byref(pkt))
        lib.avcodec_free_context(ctypes.byref(ctx))
    return np.stack([np.concatenate(o) if o else np.zeros(0, np.float32) for o in out])


def encoder_headers(rate=44100, channels=2):
    """The three headers FFmpeg's vorbis encoder writes for (rate, channels)."""
    lib = _load()
    if lib is None:
        raise Unavailable(_state['why'])
    util = _state['util']
    vp = ctypes.c_void_p
    enc = lib.avcodec_find_encoder_by_name(b'vorbis')
    if not enc:
        raise Unavailable('this libavcodec has no vorbis encoder')
    ctx = vp(lib.avcodec_alloc_context3(enc))
    par = vp(lib.avcodec_parameters_alloc())
    try:
        for k, v in ((b'ar', b'%d' % rate), (b'ch_layout', b'stereo' if channels == 2 else b'mono'),
                     (b'strict', b'experimental')):
            if util.av_opt_set(ctx, k, v, 1) < 0:
                raise Unavailable('av_opt_set %s failed' % k.decode())
        lib.avcodec_parameters_from_context(par, ctx)
        if ctypes.c_int.from_address(par.value + _OFF_PAR_FORMAT).value != -1:
            _unavailable('AVCodecParameters.format is not at the assumed offset')
        ctypes.c_int.from_address(par.value + _OFF_PAR_FORMAT).value = AV_SAMPLE_FMT_FLTP
        lib.avcodec_parameters_to_context(ctx, par)
        if lib.avcodec_open2(ctx, enc, None) < 0:
            raise Unavailable('the vorbis encoder does not open')
        lib.avcodec_parameters_from_context(par, ctx)
        n = ctypes.c_int.from_address(par.value + _OFF_PAR_EXTRA_SIZE).value
        ext = ctypes.string_at(ctypes.c_void_p.from_address(par.value + _OFF_PAR_EXTRA).value, n)
    finally:
        lib.avcodec_parameters_free(ctypes.byref(par))
        lib.avcodec_free_context(ctypes.byref(ctx))
    return xiph_unlace(ext)


def xiph_unlace(ext):
    count = ext[0] + 1
    sizes, o = [], 1
    for _ in range(count - 1):
        n = 0
        while True:
            n += ext[o]
            o += 1
            if ext[o - 1] < 255:
                break
        sizes.append(n)
    sizes.append(len(ext) - o - sum(sizes))
    out = []
    for n in sizes:
        out.append(ext[o:o + n])
        o += n
    return out
