"""H100-native mirror of the reference's lib/nets.py model-load API.

``CascadedNet(n_fft, hop_length, nout=32, nout_lstm=128)`` keeps the constructor, attributes
(``offset``, ``n_fft``, ``hop_length``, ``max_bin``, ``output_bin``), the 689-key ``state_dict`` format
and the ``predict_mask`` / ``predict`` / ``forward`` calls of lib/nets.py:44-141, but holds no
torch layers: the forward runs in libvr_b200.so (hand-written sm_90a kernels) on a CUDA device.
There is no CPU execution path; calling the model before ``.to(cuda)`` raises.
"""
import os
from collections import OrderedDict

import numpy as np
import torch
from torch import nn

from . import _native
from . import synth


class CascadedNet(nn.Module):

    def __init__(self, n_fft, hop_length, nout=32, nout_lstm=128, is_complex=False):
        super(CascadedNet, self).__init__()
        if is_complex:
            # never enabled by any reference caller (inference.py:130, train.py:208, pseudo.py:32)
            raise NotImplementedError('is_complex=True is outside the H100 inference hot path')
        self.n_fft = n_fft
        self.hop_length = hop_length
        self.is_complex = False
        self.nout = nout
        self.nout_lstm = nout_lstm
        self.max_bin = n_fft // 2
        self.output_bin = n_fft // 2 + 1
        self.nin_lstm = self.max_bin // 2
        self.offset = 64
        self._spec = synth.state_dict_spec(n_fft, nout, nout_lstm)
        # Default-constructed weights are zeros (the reference's are torch default inits); a checkpoint is
        # expected to be loaded, exactly as inference.py:130-131 does.
        self._tensors = OrderedDict(
            (k, torch.zeros(s, dtype=torch.int64 if kind == 'bn_count' else torch.float32))
            for k, s, kind in self._spec)
        self._device = torch.device('cpu')
        self._ctxs = {}
        # 0: wgmma tensor-core convolutions where the tile fits (default); 1: CUDA-core kernel everywhere.
        # VR_CONV_MODE=1 is a validation switch (same device, same library), not a backend.
        self.conv_mode = int(os.environ.get('VR_CONV_MODE', '0'))

    # ---- nn.Module surface used by the reference callers -------------------------------------------
    def state_dict(self, *args, **kwargs):
        return OrderedDict((k, v.clone()) for k, v in self._tensors.items())

    def load_state_dict(self, state_dict, strict=True):
        missing = [k for k in self._tensors if k not in state_dict]
        unexpected = [k for k in state_dict if k not in self._tensors]
        errors = []
        for k, v in state_dict.items():
            if k in self._tensors and tuple(v.shape) != tuple(self._tensors[k].shape):
                errors.append('size mismatch for {}: copying a param with shape {} from checkpoint, the shape in '
                              'current model is {}.'.format(k, tuple(v.shape), tuple(self._tensors[k].shape)))
        if strict and (missing or unexpected):
            if unexpected:
                errors.insert(0, 'Unexpected key(s) in state_dict: {}. '.format(', '.join(map(repr, unexpected))))
            if missing:
                errors.insert(0, 'Missing key(s) in state_dict: {}. '.format(', '.join(map(repr, missing))))
        if errors:
            raise RuntimeError('Error(s) in loading state_dict for CascadedNet:\n\t' + '\n\t'.join(errors))
        for k in self._tensors:
            if k in state_dict:
                v = state_dict[k]
                v = v.detach().cpu() if torch.is_tensor(v) else torch.from_numpy(np.asarray(v))
                self._tensors[k] = v.to(self._tensors[k].dtype).clone()
        self._drop_contexts()
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def parameters(self, recurse=True):
        for (k, _, kind) in self._spec:
            if not kind.startswith('bn_mean') and kind not in ('bn_var', 'bn_count'):
                yield self._tensors[k]

    def to(self, *args, **kwargs):
        device = kwargs.get('device', args[0] if args else None)
        if device is not None and not isinstance(device, torch.dtype):
            device = torch.device(device)
            if device.type == 'cuda' and device.index is None:
                device = torch.device('cuda', torch.cuda.current_device())
            if device != self._device:
                self._drop_contexts()
            self._device = device
        return self

    def cuda(self, device=None):
        return self.to(torch.device('cuda', 0 if device is None else device))

    def _drop_contexts(self):
        for ctx in self._ctxs.values():
            ctx.close()
        self._ctxs = {}

    # ---- native contexts ----------------------------------------------------------------------------
    def native_context(self, cropsize, max_batch):
        """The vr_ctx for (cropsize, max_batch) on this model's CUDA device, with weights loaded."""
        if self._device.type != 'cuda':
            raise RuntimeError('CascadedNet (H100) has no CPU execution path: call model.to(torch.device("cuda:N")) '
                               'first (the reference default --gpu -1 is not available here)')
        key = (int(cropsize), int(max_batch), int(self.conv_mode))
        ctx = self._ctxs.get(key)
        if ctx is None:
            for k in [k for k in self._ctxs if k[0] == key[0] and k[2] == key[2] and k[1] < key[1]]:
                self._ctxs.pop(k).close()
            ctx = _native.Context(self._device.index, self.n_fft, self.hop_length, self.nout, self.nout_lstm,
                                  cropsize, max_batch, self.conv_mode)
            ctx.load_state_dict(self._tensors)
            self._ctxs[key] = ctx
        return ctx

    def _run(self, x, cropped):
        if not torch.is_tensor(x):
            raise TypeError('expected a torch tensor')
        if x.dim() != 4 or x.size(1) != 2 or x.size(2) != self.output_bin:
            raise ValueError('expected input of shape (N, 2, {}, W), got {}'.format(self.output_bin, tuple(x.shape)))
        if x.device.type != 'cuda':
            raise RuntimeError('CascadedNet (H100) input must be a CUDA tensor; there is no CPU path')
        N, W = x.size(0), x.size(3)
        out_w = W - 2 * self.offset if cropped else W
        assert out_w > 0   # lib/nets.py:129
        ctx = self.native_context(W, max(1, min(N, 16)))
        x = x.contiguous().float()
        with torch.cuda.device(x.device):
            mask = torch.empty((N, 2, self.output_bin, out_w), dtype=torch.float32, device=x.device)
            fn = ctx.lib.vr_predict_mask if cropped else ctx.lib.vr_forward
            ctx.check(fn(ctx.handle, _native.ptr(x), N, _native.ptr(mask), _native.stream_ptr()),
                      'vr_predict_mask' if cropped else 'vr_forward')
        return mask

    def forward(self, x):
        """lib/nets.py:82-117: float32 (N, 2, n_fft//2+1, W) magnitudes -> mask of the same shape."""
        return self._run(x, cropped=False)

    def predict_mask(self, x):
        """lib/nets.py:124-131: mask cropped by ``offset`` frames on both sides of the time axis."""
        if self.offset > 0:
            return self._run(x, cropped=True)
        return self._run(x, cropped=False)

    def predict(self, x):
        """lib/nets.py:133-141."""
        pred = x * self.forward(x)
        if self.offset > 0:
            pred = pred[:, :, :, self.offset:-self.offset]
            assert pred.size()[3] > 0
        return pred


# older releases of the reference (and BASELINE.json) call the class CascadedASPPNet
CascadedASPPNet = CascadedNet
