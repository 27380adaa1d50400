"""The window-sharded multi-GPU separation (lib/distributed.py) on one H100: every rank of a world, run in one process
through the shipped code, against the single-GPU stems bit for bit.

distributed.separate_wave and separate_wave_host run once per rank.  The few torch.distributed calls they make are
replaced, with monkeypatch, by fakes that hand each rank what its peers produced:

* the ranks run one after another, highest rank first: the halo mask frame only flows from rank r + 1 to rank r, and
  in the gathered modes rank 0, which runs last, assembles the stems;
* the normaliser all-reduce takes two sweeps over the ranks: in the first, each rank's max|X| over its own frames is
  recorded and the rank is stopped there; in the second, every rank is handed the largest of them, which must be the
  whole track's vr_normaliser exactly (with --tta every rank computes the whole-track normaliser itself, no all-reduce
  is made and one sweep is enough);
* the completion all-reduces synchronise the device; dist.gather hands rank 0 every rank's block;
* distributed._shared_buffer (a CUDA IPC mapping of rank 0's memory, which cannot be opened in the process that made
  it) returns one device buffer per tag, owned by the test and shared by all ranks, so every rank stores into "rank
  0's" stem or mask buffer as it would over NVLink.

Every rank has its own model, Separator and engine context, as on its own GPU, so its cached workspaces and its two
alternating stem buffer sets are its own.  Before a rank runs, everything it should not read is NaN: its cached
spectrogram and mask workspaces, its device wave and stem workspaces in the host form, and, once per call, the shared
stem and mask buffers.  A NaN that reaches a stem is a read outside the plan; a NaN spectrogram frame that a window
reads is packed as zero (pack_mag_from_spec_kernel), which shows as stems that differ.

Each window's mask does not depend on the batch it runs in (test_gpu_generic_pair.py, test_gpu_halo_conv.py), the
range entry points reproduce the whole-track calls exactly (test_gpu_parity.py), and istft_ola_kernel sums the same
frames in the same order whatever span it is launched for, so the assembled stems must equal Separator.separate_wave
on one context bit for bit.  They are also anchored in float64 to oracle/stft_oracle.py fed the GPU's own spectrogram
and mask, at the inverse-STFT gate of test_gpu_spectral_geometry.py.  Two deliberately wrong orchestrations show that
the bitwise check is not vacuous.

Not covered here: the CUDA IPC mapping, stores over NVLink and NCCL itself.  Those run only in tests/mgpu_check.py,
which test_two_gpus_run_mgpu_check starts under torchrun on a machine with at least two GPUs.
"""
import os
import signal
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, record_parity
from test_gpu_spectral_geometry import ISTFT_GATE, _check_inverse, _frame_scale, _istft_ratio, _ola_weight
from test_gpu_streamed_separation import _anchor

pytestmark = pytest.mark.gpu

SR = 44100
SHARDED_GEOMETRIES = [(1024, 512), (2048, 1024), (4096, 2048)]   # hop = n_fft / 2: every stage is sharded
CROPSIZES = (256, 144)
BATCHES = (1, 4)
WORLDS = (2, 3, 4)
MAX_WORLD = max(WORLDS)
# T = k * roi: the last window holds only padding; k * roi + 1: the last window makes only the track's last frame,
# which is the halo frame of the rank before the last where the last rank holds just that window; and a ragged T.
# k = 6 at cropsize 256 (roi 128, 7 windows: 4+3, 3+3+1, 2+2+2+1 over 2, 3, 4 ranks) and k = 12 at cropsize 144
# (roi 16, 13 windows: 7+6, 5+5+3, 4+4+4+1), so that with batch 4 most ranks end on a ragged batch, and at cropsize
# 144 the rank boundaries lie away from multiples of 128 frames.
LENGTHS = ('multiple', 'halo', 'ragged')
# (form, VR_GATHER, tta).  The host form with --tta is the device-resident --tta call plus a copy on rank 0, so only
# the worlds with an empty last rank run it.
MODES = (('device', 'sharded', False), ('device', 'sharded', True), ('host', 'sharded', False),
         ('device', 'p2p', False), ('device', 'nccl', False))
ALL_MODES = MODES + (('host', 'sharded', True),)
_PATHS = ('_separate_wave_sharded', '_separate_wave_p2p', '_separate_wave_nccl')
_ORIGINAL = {}


def _dev():
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    return torch.device('cuda:0')


def _frames(cropsize, offset, length):
    roi = cropsize - 2 * offset
    k = 6 if roi == 128 else 12
    return k * roi + {'multiple': 0, 'halo': 1, 'ragged': roi // 2 + 5}[length]


def _tracks(hop, T):
    """two tracks of T frames (a ragged last hop) whose masks differ everywhere: a sine mix and white noise"""
    from lib import synth
    L = hop * (T - 1) + hop // 2
    mix = np.ascontiguousarray(synth.sine_mix(L / SR + 0.01, seed=T)[:, :L])
    noise = 0.5 * np.random.default_rng(T + 1).standard_normal((2, L)).astype(np.float32)
    return mix, noise


@pytest.fixture(scope='module')
def rig():
    """rig(n_fft, hop, cropsize, batch) -> (one Separator per emulated rank, a cache of single-GPU references).  Each
    rank has its own model over the seeded synthetic checkpoint, so its own engine context, as on its own GPU; rank
    0's Separator also computes the single-GPU stems.  One configuration is held at a time: when it changes, and at
    teardown, every context's cached workspaces are released (distributed.release) and the contexts are closed."""
    import inference
    from lib import distributed, nets, synth
    held = {'geometry': None, 'key': None, 'models': [], 'seps': None, 'cache': {}}

    def drop_contexts():
        for m in held['models']:
            for ctx in m._ctxs.values():
                distributed.release(ctx)
            m._drop_contexts()
        held['cache'].clear()

    def make(n_fft, hop, cropsize, batch):
        key = (n_fft, hop, cropsize, batch)
        if held['key'] != key:
            drop_contexts()
            if held['geometry'] != (n_fft, hop):
                sd = synth.to_torch_state_dict(synth.make_state_dict(n_fft, 32, 128))
                held['models'] = []
                for _ in range(MAX_WORLD):
                    m = nets.CascadedNet(n_fft, hop, 32, 128)
                    m.load_state_dict(sd)
                    held['models'].append(m.to(_dev()))
                held['geometry'] = (n_fft, hop)
            held['seps'] = [inference.Separator(m, _dev(), batch, cropsize, False) for m in held['models']]
            held['key'] = key
        return held['seps'], held['cache']

    yield make
    drop_contexts()
    held['models'] = []


def _single_gpu(sp, wave, tta):
    """Separator.separate_wave of the CUDA wave on one context, the whole track's vr_normaliser (max|X|), and the
    float64 anchor of those stems: the oracle's inverse STFT of the GPU's own spectrogram and final mask"""
    from lib import _native
    ctx = sp._ctx()
    dev = _dev()
    hop, n_fft = sp.model.hop_length, sp.model.n_fft
    with torch.cuda.device(dev):
        w = torch.from_numpy(wave).to(dev)
        inst, voc = sp.separate_wave(w, tta=tta)
        T = 1 + w.shape[1] // hop
        st = _native.stream_ptr()
        spec = torch.empty((2, n_fft // 2 + 1, T), dtype=torch.complex64, device=dev)
        ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(w), w.shape[1], _native.ptr(spec), T, None, st), 'vr_stft')
        norm = torch.empty(1, dtype=torch.float32, device=dev)
        ctx.check(ctx.lib.vr_normaliser(ctx.handle, _native.ptr(spec), T, 0, _native.ptr(norm), st), 'vr_normaliser')
        mask = sp._mask_device(spec, tta)
        X, m = spec.cpu().numpy(), mask.cpu().numpy()
    stems = (inst.cpu().numpy(), voc.cpu().numpy())
    anchor = _anchor(X, m, hop)
    weight, dead = _ola_weight(n_fft, hop, T)
    scale = _frame_scale(X)
    for name, got, want in zip(('instruments', 'vocals'), stems, anchor):
        _check_inverse(name, got, want, dead)
    ratio = max(_istft_ratio(got, want, weight, scale) for got, want in zip(stems, anchor))
    return {'stems': stems, 'norm': norm.cpu(), 'anchor': anchor, 'weight': weight, 'scale': scale, 'ratio': ratio}


def _references(cache, sp, waves, tta):
    """the single-GPU records of both tracks, kept while the configuration and the track length stay the same"""
    T = 1 + waves[0].shape[1] // sp.model.hop_length
    if cache.get('T') != T:
        cache.clear()
        cache['T'] = T
    if tta not in cache:
        cache[tta] = [_single_gpu(sp, wave, tta) for wave in waves]
    return cache[tta]


# ---- torch.distributed for the ranks of a world, run one after another in this process ---------------------------
class _Stop(Exception):
    """raised by the fake normaliser all-reduce of the first sweep, once the rank has contributed its max|X|"""


class _P2POp(object):
    def __init__(self, op, tensor, peer=None, group=None, tag=0, group_peer=None):
        self.op, self.tensor, self.peer = op, tensor, peer


def _isend(*args, **kwargs):
    raise AssertionError('lib/distributed.py sends its halo frame through batch_isend_irecv')


def _irecv(*args, **kwargs):
    raise AssertionError('lib/distributed.py receives its halo frame through batch_isend_irecv')


class _Done(object):
    def wait(self):
        return True


class _World(object):
    """The fakes of one world.  ``halo``: 'exchange' delivers the right neighbour's mask frame; 'skip' delivers nothing
    (the receive buffer is cleared to zeros, so that the check sees a missing halo frame rather than whatever the
    allocator left in the buffer)."""

    def __init__(self, world, halo='exchange'):
        self.world, self.halo_mode = world, halo
        self.rank = self.sweep = self.norm = None
        self.norms = {}
        self.buffers = {}   # tag -> the device buffer every rank's _shared_buffer(tag) maps
        self.poisoned = set()

    def run(self, call, poison, after=None):
        """call(rank) on every rank, highest first, after poison(rank) and followed by after(rank) when the rank
        returned; a second sweep when the first stopped every rank at the normaliser all-reduce.  Returns {rank: what
        call returned}."""
        self.poisoned = set()   # the shared buffers are poisoned once per call, when a rank first asks for them
        self.norms, self.norm = {}, None
        out = self._sweep(1, call, poison, after)
        if self.norms:
            assert sorted(self.norms) == list(range(self.world)) and not out, \
                'only ranks %s made the normaliser all-reduce' % sorted(self.norms)
            self.norm = torch.stack([self.norms[r] for r in range(self.world)]).max(dim=0).values
            out = self._sweep(2, call, poison, after)
        return out

    def _sweep(self, sweep, call, poison, after):
        self.sweep = sweep
        self.sent, self.received, self.blocks, self.entered = {}, set(), {}, set()
        out = {}
        for rank in reversed(range(self.world)):
            self.rank = rank
            poison(rank)
            try:
                out[rank] = call(rank)
            except _Stop:
                continue
            if after is not None:
                after(rank)
        torch.cuda.synchronize()
        assert set(self.sent) == self.received, 'halo frames sent by ranks %s, received from ranks %s' % (
            sorted(self.sent), sorted(self.received))
        return out

    def spy(self, name, fn):
        def entered(*args, **kwargs):
            self.entered.add(name)
            return fn(*args, **kwargs)
        return entered

    def all_reduce(self, tensor, op=None, group=None, async_op=False):
        import torch.distributed as dist
        if op == dist.ReduceOp.MAX:   # the normaliser
            if self.sweep == 1:
                self.norms[self.rank] = tensor.clone()
                raise _Stop()
            tensor.copy_(self.norm)
        else:                         # a completion flag: every store a rank enqueued before it has landed
            torch.cuda.synchronize()

    def batch_isend_irecv(self, ops):
        for p in ops:
            if p.op is _isend:
                assert p.peer == self.rank - 1, 'rank %d sends its halo frame to rank %d' % (self.rank, p.peer)
                self.sent[self.rank] = p.tensor   # kept to the end of the sweep, so no receive is handed its memory
            else:
                assert p.op is _irecv and p.peer == self.rank + 1, 'rank %d receives from rank %d' % (self.rank, p.peer)
                assert p.peer in self.sent, 'rank %d waits for a halo frame rank %d never sends' % (self.rank, p.peer)
                self.received.add(p.peer)
                if self.halo_mode == 'skip':
                    p.tensor.zero_()
                else:
                    p.tensor.copy_(self.sent[p.peer])
        return [_Done() for _ in ops]

    def gather(self, tensor, gather_list=None, dst=0, group=None, async_op=False):
        assert dst == 0 and (gather_list is not None) == (self.rank == 0)
        self.blocks[self.rank] = tensor
        if gather_list is not None:
            assert sorted(self.blocks) == list(range(self.world)), sorted(self.blocks)
            for r, out in enumerate(gather_list):
                out.copy_(self.blocks[r])

    def shared_buffer(self, ctx, tag, nbytes, world, rank, dev, group):
        from lib import _native
        if tag not in self.buffers:
            self.buffers[tag] = torch.empty(((nbytes + 3) // 4,), dtype=torch.float32, device=dev)
        buf = self.buffers[tag]
        assert 4 * buf.numel() >= nbytes, (tag, nbytes)
        if tag not in self.poisoned:
            buf.fill_(float('nan'))
            self.poisoned.add(tag)
        return _native.c_vp(buf.data_ptr())


def _emulate(monkeypatch, world, halo='exchange'):
    """a _World whose fakes replace what lib/distributed.py calls of torch.distributed (undone at the test's end)"""
    import torch.distributed as dist
    from lib import distributed
    w = _World(world, halo)
    for name in _PATHS:
        fn = _ORIGINAL.setdefault(name, getattr(distributed, name))
        monkeypatch.setattr(distributed, name, w.spy(name, fn))
    monkeypatch.setattr(distributed, '_shared_buffer', w.shared_buffer)
    monkeypatch.setattr(dist, 'all_reduce', w.all_reduce)
    monkeypatch.setattr(dist, 'P2POp', _P2POp)
    monkeypatch.setattr(dist, 'isend', _isend)
    monkeypatch.setattr(dist, 'irecv', _irecv)
    monkeypatch.setattr(dist, 'batch_isend_irecv', w.batch_isend_irecv)
    monkeypatch.setattr(dist, 'gather', w.gather)
    return w


def _poison(sp, T, L, host):
    """NaN in the rank's cached spectrogram and mask workspaces and, in the host form, its device wave and stem
    workspaces.  They live in distributed._shared, the one private cache of lib/distributed.py this file touches; a
    rank that has none of this track's size yet gets them here, shaped as the module makes them."""
    from lib import distributed
    ctx = sp._ctx()
    dev = _dev()
    bins = sp.model.n_fft // 2 + 1
    key = ('ws', ctx)
    if key not in distributed._shared or distributed._shared[key][0] < T:
        distributed._shared[key] = (T, torch.empty((2 * bins * T,), dtype=torch.complex64, device=dev),
                                    torch.empty((2 * bins * T,), dtype=torch.float32, device=dev))
    tensors = list(distributed._shared[key][1:])
    if host:
        key = ('hostws', ctx)
        if key not in distributed._shared or distributed._shared[key][0] < L:
            distributed._shared[key] = (L,) + tuple(torch.empty((2 * L,), dtype=torch.float32, device=dev)
                                                    for _ in range(3))
        tensors += list(distributed._shared[key][1:])
    for t in tensors:
        (torch.view_as_real(t) if t.is_complex() else t).fill_(float('nan'))


def _separate(monkeypatch, seps, world, waves, form, gather, tta, halo='exchange'):
    """Both tracks, one call each, on `world` emulated ranks with VR_GATHER=gather, through
    distributed.separate_wave of the CUDA wave (form 'device') or separate_wave_host of a pinned one ('host').
    Returns one record per track: the assembled stems (numpy), the normaliser the ranks were handed (None without an
    all-reduce), the path separate_wave took, and in the host form every rank's (s0, s1); and whether the first call's
    device stems were left unchanged by the second call."""
    from lib import distributed
    monkeypatch.setenv('VR_GATHER', gather)
    w = _emulate(monkeypatch, world, halo)
    dev = _dev()
    hop = seps[0].model.hop_length
    records, kept = [], None
    for wave in waves:
        L = wave.shape[1]
        T = 1 + L // hop
        Lo = hop * (T - 1)
        host = form == 'host'
        if host:
            h_wave = torch.from_numpy(wave).pin_memory()
            h_out = [(torch.full((2, Lo), float('nan')).pin_memory(), torch.full((2, Lo), float('nan')).pin_memory())
                     for _ in range(world)]

            def call(r):
                return distributed.separate_wave_host(seps[r], h_wave, h_out[r][0], h_out[r][1], tta=tta, world=world,
                                                      rank=r)
        else:
            d_wave = torch.from_numpy(wave).to(dev)

            def call(r):
                return distributed.separate_wave(seps[r], d_wave, tta=tta, world=world, rank=r)

        stray = []

        def below_span_untouched(r):
            """A rank of the device-resident sharded form stores hops [k0, k1) into the shared stem buffers.  The
            ranks below it run later and overwrite what it may have stored below its span, so check here that
            everything below hop * k0 is still the poison."""
            if host or '_separate_wave_sharded' not in w.entered:
                return
            k0 = distributed.shard_plan(T, seps[r].cropsize, seps[r].offset, world, r)[7]
            torch.cuda.synchronize()
            for tag in sorted(t for t in w.poisoned if t.startswith(('inst', 'voc'))):
                below = w.buffers[tag][:2 * Lo].view(2, Lo)[:, :hop * k0]
                if not torch.isnan(below).all():
                    stray.append('rank %d stored %d samples of %s below its span [%d, %d)'
                                 % (r, int((~torch.isnan(below)).sum()), tag, hop * k0, Lo))

        out = w.run(call, lambda r: _poison(seps[r], T, L, host), below_span_untouched)
        assert len(w.entered) == 1, w.entered
        rec = {'norm': None if w.norm is None else w.norm.cpu(), 'path': next(iter(w.entered)), 'stray': stray}
        if host:
            rec['slices'] = [out[r] for r in range(world)]
            stems = [np.full((2, Lo), np.nan, dtype=np.float32) for _ in range(2)]
            for r, (s0, s1) in enumerate(rec['slices']):
                for stem, h in zip(stems, h_out[r]):
                    stem[:, s0:s1] = h[:, s0:s1].numpy()
            rec['stems'] = tuple(stems)
        else:
            assert all(out[r] == (None, None) for r in range(1, world)), 'only rank 0 returns stems'
            inst, voc = out[0]
            rec['stems'] = (inst.cpu().numpy(), voc.cpu().numpy())
            if kept is None:
                kept = (inst, voc, inst.clone(), voc.clone())
        records.append(rec)
    torch.cuda.synchronize()
    unchanged = kept is None or (torch.equal(kept[0], kept[2]) and torch.equal(kept[1], kept[3]))
    return records, unchanged


def _check(tag, rec, ref, failed):
    """the assembled stems == the single-GPU stems bit for bit, and within the float64 gate; returns the anchor ratio"""
    equal = True
    for i, name in enumerate(('instruments', 'vocals')):
        got, want = rec['stems'][i], ref['stems'][i]
        bad = int((~np.isfinite(got)).sum())
        if bad:
            failed.append('%s %s: %d non-finite samples (a read outside the plan)' % (tag, name, bad))
        if not np.array_equal(got, want):
            equal = False
            failed.append('%s %s: %d samples differ from the single-GPU stems' % (tag, name, int((got != want).sum())))
    # identical stems have the reference's ratio; others are measured
    ratio = ref['ratio'] if equal else float(np.max([_istft_ratio(got, want, ref['weight'], ref['scale'])
                                                    for got, want in zip(rec['stems'], ref['anchor'])]))
    if not ratio <= ISTFT_GATE:
        failed.append('%s vs float64: %.4g > gate %.4g' % (tag, ratio, ISTFT_GATE))
    return ratio


def _check_mode(monkeypatch, seps, refs, world, waves, mode, path, tag, failed):
    """one mode of one world on both tracks, against the single-GPU records; `path` is the _separate_wave_* it must
    take"""
    form, gather, tta = mode
    hop = seps[0].model.hop_length
    T = 1 + waves[0].shape[1] // hop
    Lo = hop * (T - 1)
    records, unchanged = _separate(monkeypatch, seps, world, waves, form, gather, tta)
    tag = '%s_%s_%s%s' % (tag, form, gather, '_tta' if tta else '')
    ratio = 0.0
    for i, (rec, ref) in enumerate(zip(records, refs)):
        if rec['path'] != path:
            failed.append('%s: took %s, expected %s' % (tag, rec['path'], path))
        failed += ['%s_track%d: %s' % (tag, i, msg) for msg in rec['stray']]
        ratio = float(np.max([ratio, _check(tag + '_track%d' % i, rec, ref, failed)]))   # keeps a NaN
        two_sweeps = path == '_separate_wave_sharded' and not tta
        if two_sweeps != (rec['norm'] is not None):
            failed.append('%s: the normaliser was %sall-reduced' % (tag, '' if rec['norm'] is not None else 'not '))
        elif two_sweeps and not torch.equal(rec['norm'], ref['norm']):
            failed.append('%s: all-reduced normaliser %r != whole-track vr_normaliser %r'
                          % (tag, rec['norm'].item(), ref['norm'].item()))
        if form == 'host':
            s = rec['slices']
            if path == '_separate_wave_sharded' and not tta:   # every rank copies out its own slice
                tiles = s[0][0] == 0 and s[-1][1] == Lo and all(x[1] == y[0] for x, y in zip(s, s[1:]))
            else:                                             # rank 0 holds the whole stems
                tiles = s == [(0, Lo)] + [(0, 0)] * (world - 1)
            if not tiles:
                failed.append('%s: host slices %s do not tile [0, %d)' % (tag, s, Lo))
    if not unchanged:
        failed.append('%s: the stems the first call returned changed during the second call' % tag)
    record_parity(tag + '_vs_float64', ratio, ISTFT_GATE)


def _expected_path(seps, T, world, gather):
    from lib import distributed
    sp = seps[0]
    n_windows, _ = distributed.window_count(T, sp.cropsize, sp.offset)
    if gather == 'sharded':
        if sp.model.hop_length * 2 == sp.model.n_fft and n_windows >= world:
            return '_separate_wave_sharded'
        return '_separate_wave_p2p'
    return '_separate_wave_' + gather


def _check_world(monkeypatch, seps, cache, world, T, modes, tag):
    """every mode in `modes` on `world` ranks and tracks of T frames; the failures, as messages"""
    hop = seps[0].model.hop_length
    waves = _tracks(hop, T)
    failed = []
    for mode in modes:
        refs = _references(cache, seps[0], waves, mode[2])
        _check_mode(monkeypatch, seps, refs, world, waves, mode, _expected_path(seps, T, world, mode[1]), tag, failed)
    return failed


def _tta_refused(monkeypatch, seps, world, T, gather, form='device'):
    """--tta with a mode that is not sharded raises NotImplementedError before any work"""
    with pytest.raises(NotImplementedError):
        _separate(monkeypatch, seps, world, _tracks(seps[0].model.hop_length, T)[:1], form, gather, True)


def _sharded_cases():
    """every geometry, cropsize and world size; at batch 4 every track length, at batch 1 (each window a batch of its
    own, so no rank ends on a ragged batch) the ragged one, which keeps the file to a few minutes on one H100"""
    for n_fft, hop in SHARDED_GEOMETRIES:
        for cropsize in CROPSIZES:
            for batch in BATCHES:
                for length in (LENGTHS if batch > 1 else LENGTHS[-1:]):
                    for world in WORLDS:
                        yield pytest.param(n_fft, hop, cropsize, batch, length, world,
                                           id='nfft%d-crop%d-batch%d-%s-world%d' % (n_fft, cropsize, batch, length,
                                                                                   world))


@pytest.mark.parametrize('n_fft,hop,cropsize,batch,length,world', list(_sharded_cases()))
def test_every_mode_equals_single_gpu(rig, monkeypatch, n_fft, hop, cropsize, batch, length, world):
    """hop = n_fft / 2: the sharded mode device-resident with and without --tta and in the host form, and the p2p and
    nccl gathers, on `world` emulated ranks == the single-GPU stems bit for bit, and within the float64 gate; p2p and
    nccl refuse --tta."""
    seps, cache = rig(n_fft, hop, cropsize, batch)
    T = _frames(cropsize, seps[0].offset, length)
    tag = 'sharded_nfft%d_crop%d_b%d_T%d_w%d' % (n_fft, cropsize, batch, T, world)
    failed = _check_world(monkeypatch, seps, cache, world, T, MODES, tag)
    for gather in ('p2p', 'nccl'):
        _tta_refused(monkeypatch, seps, world, T, gather)
    if world == MAX_WORLD and batch == max(BATCHES) and length == LENGTHS[0]:
        # cudaMemGetInfo counts every process on the device, so on a shared GPU this bounds the contexts' memory
        free, total = torch.cuda.mem_get_info()
        print('DEVICE MEMORY %s: %.2f of %.2f GiB in use on the device with %d engine contexts at batch %d'
              % (tag, (total - free) / 2 ** 30, total / 2 ** 30, world, batch))
    assert not failed, '\n'.join(failed)


@pytest.mark.parametrize('cropsize,batch', [(c, b) for c in CROPSIZES for b in BATCHES])
def test_hop_below_half_window_gathers_the_mask(rig, monkeypatch, cropsize, batch):
    """n_fft 2048, hop 512: an output hop reads more than one frame past its own, so VR_GATHER=sharded falls back to
    p2p in both forms; p2p and nccl at every world size == the single-GPU stems, and none of the three modes takes
    --tta."""
    n_fft, hop = 2048, 512
    seps, cache = rig(n_fft, hop, cropsize, batch)
    modes = (('device', 'sharded', False), ('host', 'sharded', False), ('device', 'p2p', False),
             ('device', 'nccl', False))
    failed = []
    T = _frames(cropsize, seps[0].offset, 'ragged')
    for world in WORLDS:
        tag = 'hop512_nfft%d_crop%d_b%d_T%d_w%d' % (n_fft, cropsize, batch, T, world)
        failed += _check_world(monkeypatch, seps, cache, world, T, modes, tag)
    for gather, form in (('sharded', 'device'), ('sharded', 'host'), ('p2p', 'device'), ('nccl', 'device')):
        _tta_refused(monkeypatch, seps, MAX_WORLD, T, gather, form)
    assert not failed, '\n'.join(failed)


@pytest.mark.parametrize('n_fft,hop,cropsize', [(n, h, c) for n, h in SHARDED_GEOMETRIES for c in CROPSIZES])
def test_empty_last_rank_and_fewer_windows_than_ranks(rig, monkeypatch, n_fft, hop, cropsize):
    """An empty last rank (5 windows over 4 ranks at cropsize 256, 9 at 144: the ceil split leaves the last rank
    none) in every mode, the host form also with --tta, and a track of 2 windows over 3 and 4 ranks, where
    VR_GATHER=sharded falls back to p2p and --tta is refused."""
    from lib import distributed
    seps, cache = rig(n_fft, hop, cropsize, 4)
    roi = cropsize - 2 * seps[0].offset
    failed = []
    n_windows = 5 if roi == 128 else 9
    T = (n_windows - 1) * roi + roi // 3
    assert distributed.window_count(T, cropsize, seps[0].offset)[0] == n_windows
    assert distributed.shard_windows(n_windows, MAX_WORLD, MAX_WORLD - 1)[1] == 0
    failed += _check_world(monkeypatch, seps, cache, MAX_WORLD, T, ALL_MODES,
                           'empty_rank_nfft%d_crop%d_T%d_w%d' % (n_fft, cropsize, T, MAX_WORLD))
    T = roi + roi // 3
    assert distributed.window_count(T, cropsize, seps[0].offset)[0] == 2
    modes = (('device', 'sharded', False), ('host', 'sharded', False), ('device', 'p2p', False),
             ('device', 'nccl', False))
    for world in (3, 4):
        failed += _check_world(monkeypatch, seps, cache, world, T, modes,
                               'two_windows_nfft%d_crop%d_T%d_w%d' % (n_fft, cropsize, T, world))
        _tta_refused(monkeypatch, seps, world, T, 'sharded')
        _tta_refused(monkeypatch, seps, world, T, 'sharded', 'host')
    assert not failed, '\n'.join(failed)


@pytest.mark.parametrize('variant', ['late_read_span', 'halo_skipped'])
def test_wrong_orchestrations_fail_the_bitwise_check(rig, monkeypatch, variant):
    """Two wrong orchestrations of 7 windows over 3 ranks (n_fft 2048, hop 1024, cropsize 256, batch 4, the halo
    frame of rank 1 the track's last frame) must give stems that differ from the single-GPU stems: the interior
    rank's spectrogram span [a, b) starting one frame late (its first window then reads a frame no rank computed), and
    the halo frame never received (the receive buffer left at zero)."""
    from lib import distributed
    seps, cache = rig(2048, 1024, 256, 4)
    world = 3
    T = _frames(256, seps[0].offset, 'halo')
    halo = 'exchange'
    if variant == 'late_read_span':
        plan = distributed.shard_plan

        def late(n_frames, cropsize, offset, world_, rank):
            p = list(plan(n_frames, cropsize, offset, world_, rank))
            if 0 < rank < world_ - 1:
                assert p[5] > 0, 'the interior rank must start inside the track'
                p[5] += 1
            return tuple(p)
        monkeypatch.setattr(distributed, 'shard_plan', late)
    else:
        halo = 'skip'
    waves = _tracks(1024, T)
    refs = _references(cache, seps[0], waves, False)
    records, _ = _separate(monkeypatch, seps, world, waves, 'device', 'sharded', False, halo)
    differing = []
    for rec, ref in zip(records, refs):
        assert rec['path'] == '_separate_wave_sharded'
        differing.append(sum(int((got != want).sum()) for got, want in zip(rec['stems'], ref['stems'])))
    record_parity('sharded_wrong_variant_%s_samples_differing' % variant, min(differing))
    assert min(differing) > 0, ('%s: the stems equal the single-GPU stems; the bitwise check would not catch it'
                                % variant)


def _children(pid):
    """pids of the processes whose parent is `pid` (read from /proc)"""
    out = []
    for entry in os.listdir('/proc'):
        if not entry.isdigit():
            continue
        try:
            with open('/proc/%s/stat' % entry) as f:
                stat = f.read()
        except OSError:
            continue
        if int(stat.rsplit(')', 1)[1].split()[1]) == pid:
            out.append(int(entry))
    return out


def _runs(pid, script):
    """whether process `pid` still exists and runs `script`"""
    try:
        with open('/proc/%d/cmdline' % pid, 'rb') as f:
            return script.encode() in f.read()
    except OSError:
        return False


def _torchrun(script, nproc, log, timeout):
    """`python -m torch.distributed.run --standalone --nproc-per-node nproc script`, its output in the file `log` (a
    pipe would stay open in any worker that outlived torchrun).  Returns torchrun's exit code, or None when it did
    not finish within `timeout` seconds.  Then it gets SIGTERM, on which its agent stops every worker (each worker
    runs in a session of its own, so signalling torchrun's process group would not reach them); whatever is still
    running a minute later, workers first, is killed."""
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', str(nproc), script]
    with open(log, 'w') as out:
        proc = subprocess.Popen(cmd, cwd=ROOT, stdout=out, stderr=subprocess.STDOUT, stdin=subprocess.DEVNULL)
    try:
        return proc.wait(timeout=timeout)
    except subprocess.TimeoutExpired:
        pass
    workers = set(_children(proc.pid))
    proc.terminate()
    try:
        proc.wait(timeout=60)
    except subprocess.TimeoutExpired:
        workers.update(_children(proc.pid))   # and any worker started since
    for pid in sorted(workers):
        if _runs(pid, script):
            try:
                os.killpg(pid, signal.SIGKILL)   # the worker leads its own session and process group
            except OSError:
                pass
    if proc.poll() is None:
        proc.kill()
        proc.wait(timeout=60)
    return None


def test_two_gpus_run_mgpu_check(tmp_path):
    """tests/mgpu_check.py under torchrun on two GPUs: every exchange mode over real NCCL, CUDA IPC and NVLink
    reproduces the single-GPU stems exactly.  A run that does not finish in 900 s is stopped, workers included."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs (%d visible): the one-GPU emulation above covers the orchestration, not IPC, '
                    'NVLink or NCCL' % torch.cuda.device_count())
    log = str(tmp_path / 'mgpu_check.log')
    rc = _torchrun(os.path.join(ROOT, 'tests', 'mgpu_check.py'), 2, log, 900)
    with open(log) as f:
        out = f.read()
    print(out)
    assert rc is not None, 'mgpu_check did not finish in 900 s:\n' + out[-4000:]
    assert rc == 0 and 'MGPU_CHECK PASS' in out, out[-4000:]
