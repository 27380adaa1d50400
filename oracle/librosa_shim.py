"""``sys.modules`` shim so the UNMODIFIED reference can be imported in the build container.

TEST INFRASTRUCTURE.  ``lib/spec_utils.py:3,5`` imports ``librosa`` and ``soundfile`` at
module top level; neither is installed here and there is no network.  ``install()`` registers
stub modules whose ``stft`` / ``istft`` are the restatements in ``oracle/stft_oracle.py``
(SURVEY.md App. A) so that ``lib.nets``, ``lib.layers``, ``lib.dataset`` and
``inference.Separator`` import and run unmodified from a checkout of the reference (VR_REFERENCE_ROOT).
Used only by ``oracle/make_golden.py``; the tests compare against the fixtures it writes.
"""
import os
import sys
import types

from . import stft_oracle

REFERENCE_ROOT = os.environ.get('VR_REFERENCE_ROOT', '')


def install():
    if 'librosa' not in sys.modules:
        m = types.ModuleType('librosa')
        m.stft = lambda y, n_fft=2048, hop_length=None, **kw: stft_oracle.stft(y, n_fft, hop_length)
        m.istft = lambda S, hop_length=None, **kw: stft_oracle.istft(S, hop_length)

        def _load(*a, **k):
            raise RuntimeError('librosa.load is outside the hot path and not shimmed')
        m.load = _load
        m.effects = types.SimpleNamespace(trim=None)
        m._vr_shim = True
        sys.modules['librosa'] = m
    if 'soundfile' not in sys.modules:
        sf = types.ModuleType('soundfile')

        def _write(*a, **k):
            raise RuntimeError('soundfile.write is outside the hot path and not shimmed')
        sf.write = _write
        sf._vr_shim = True
        sys.modules['soundfile'] = sf


def import_reference():
    """Returns (inference, nets, spec_utils, dataset) modules of the unmodified reference."""
    if not os.path.isdir(REFERENCE_ROOT):
        raise RuntimeError('set VR_REFERENCE_ROOT to a checkout of the reference vocal-remover')
    install()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    # the product package also has modules called ``lib`` / ``inference``; make sure the
    # reference's own are the ones imported here.
    for k in [k for k in sys.modules if k == 'lib' or k.startswith('lib.') or k == 'inference']:
        del sys.modules[k]
    import inference  # noqa
    from lib import nets, spec_utils, dataset  # noqa
    mods = (inference, nets, spec_utils, dataset)
    for k in [k for k in sys.modules if k == 'lib' or k.startswith('lib.') or k == 'inference']:
        sys.modules['_ref_' + k] = sys.modules.pop(k)
    sys.path.remove(REFERENCE_ROOT)
    # the reference modules keep their own references to the stubs; do not leave them importable by anyone else
    for name in ('librosa', 'soundfile'):
        if getattr(sys.modules.get(name), '_vr_shim', False):
            del sys.modules[name]
    return mods
