"""FFmpeg's ``aac`` decoder through ctypes: an AAC-LC decoder independent of oracle/aac_oracle.py.

OpenCV's wheel bundles libavcodec (``opencv_python_headless.libs/libavcodec-*.so``); ``import cv2`` loads the libraries
it depends on.  ``decode(packets, rate_index, channels)`` sends each raw_data_block behind an ADTS header (so no
extradata has to be set on the context) and returns the planar float output, every sample the decoder produces (no
demuxer: no edit-list trim).  The ``AVFrame`` and ``AVPacket`` fields
read here are the leading ones, whose layout has not changed in many major versions; the first decoded frame is checked
(``nb_samples == 1024``, ``format == AV_SAMPLE_FMT_FLTP``) and anything else makes the harness report itself
unavailable rather than guess.  ``available()`` is (True, '') or (False, reason).
"""
import ctypes
import glob
import os

import numpy as np

AV_SAMPLE_FMT_FLTP = 8
AVERROR_EAGAIN = -11
_OFF_PKT_DATA = 24         # AVPacket: buf, pts, dts, data, size
_OFF_FRAME_NB_SAMPLES = 112   # AVFrame: data[8], linesize[8], extended_data, width, height, nb_samples, format
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
    libs = glob.glob(os.path.join(os.path.dirname(os.path.dirname(cv2.__file__)), 'opencv_python*.libs',
                                  'libavcodec*.so*'))
    if not libs:
        _state['why'] = 'no libavcodec next to cv2'
        return None
    try:
        lib = ctypes.CDLL(libs[0])
        util = glob.glob(os.path.join(os.path.dirname(libs[0]), 'libavutil*.so*'))
        if util:
            ctypes.CDLL(util[0]).av_log_set_level(-8)   # AV_LOG_QUIET
    except OSError as e:
        _state['why'] = 'libavcodec does not load: %s' % e
        return None
    vp = ctypes.c_void_p
    for name, res, args in (('avcodec_find_decoder_by_name', vp, [ctypes.c_char_p]),
                            ('avcodec_alloc_context3', vp, [vp]), ('avcodec_open2', ctypes.c_int, [vp, vp, vp]),
                            ('avcodec_free_context', None, [ctypes.POINTER(vp)]), ('av_packet_alloc', vp, []),
                            ('av_packet_free', None, [ctypes.POINTER(vp)]), ('av_new_packet', ctypes.c_int,
                                                                              [vp, ctypes.c_int]),
                            ('av_packet_unref', None, [vp]), ('av_frame_alloc', vp, []),
                            ('av_frame_free', None, [ctypes.POINTER(vp)]), ('av_frame_unref', None, [vp]),
                            ('avcodec_send_packet', ctypes.c_int, [vp, vp]),
                            ('avcodec_receive_frame', ctypes.c_int, [vp, vp])):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    if not lib.avcodec_find_decoder_by_name(b'aac'):
        _state['why'] = 'this libavcodec has no aac decoder'
        return None
    _state['lib'] = lib
    return lib


def available():
    lib = _load()
    if lib is None:
        return False, _state['why']
    return True, ''


class Unavailable(RuntimeError):
    pass


def decode(packets, rate_index, channels):
    """packets: list of raw_data_block bytes -> float32 (channels, n), the decoder's whole output."""
    from .aac_oracle import adts
    frames = [adts(p, rate_index, channels) for p in packets]
    lib = _load()
    if lib is None:
        raise Unavailable(_state['why'])
    vp = ctypes.c_void_p
    codec = lib.avcodec_find_decoder_by_name(b'aac')
    ctx = vp(lib.avcodec_alloc_context3(codec))
    pkt, frm = vp(lib.av_packet_alloc()), vp(lib.av_frame_alloc())
    out = [[] for _ in range(channels)]
    try:
        if lib.avcodec_open2(ctx, codec, None) < 0:
            raise Unavailable('avcodec_open2 failed for aac')
        checked = False

        def drain():
            nonlocal checked
            while True:
                rc = lib.avcodec_receive_frame(ctx, frm)
                if rc < 0:
                    return
                nb = ctypes.c_int.from_address(frm.value + _OFF_FRAME_NB_SAMPLES).value
                fmt = ctypes.c_int.from_address(frm.value + _OFF_FRAME_FORMAT).value
                if not checked:
                    if nb != 1024 or fmt != AV_SAMPLE_FMT_FLTP:
                        _state.pop('lib', None)
                        _state['why'] = ('the AVFrame layout is not the one assumed (nb_samples %d, format %d on the '
                                         'first AAC-LC frame)' % (nb, fmt))
                        raise Unavailable(_state['why'])
                    checked = True
                for c in range(channels):
                    p = ctypes.c_void_p.from_address(frm.value + 8 * c).value
                    out[c].append(np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_float)),
                                                        shape=(nb,)).copy())
                lib.av_frame_unref(frm)

        for fr in frames:
            if lib.av_new_packet(pkt, len(fr)) < 0:
                raise MemoryError('av_new_packet')
            data = ctypes.c_void_p.from_address(pkt.value + _OFF_PKT_DATA).value
            ctypes.memmove(data, bytes(fr), len(fr))
            rc = lib.avcodec_send_packet(ctx, pkt)
            lib.av_packet_unref(pkt)
            if rc < 0 and rc != AVERROR_EAGAIN:
                raise RuntimeError('aac rejected a packet (error %d)' % rc)
            drain()
        lib.avcodec_send_packet(ctx, None)
        drain()
    finally:
        lib.av_frame_free(ctypes.byref(frm))
        lib.av_packet_free(ctypes.byref(pkt))
        lib.avcodec_free_context(ctypes.byref(ctx))
    return np.stack([np.concatenate(o) if o else np.zeros(0, np.float32) for o in out])
