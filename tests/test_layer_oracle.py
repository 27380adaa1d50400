"""The per-layer gates of tests/test_gpu_layer_parity.py rehearsed on the CPU (oracle/layer_oracle.py).

The small net (CascadedNet(512, 256, 16, 32), one 192-frame window) runs through the oracle with every convolution
replaced by the CPU emulation of the product's arithmetic (oracle/precision_oracle.py's default scheme: split-bf16
operands, three products, fp32 accumulation, split-bf16 output).  Each convolution's input and emulated output then go
through the helper the GPU test uses: the three-product scheme must pass the gate, and dropping either correction
product must fail it by 8x.  The LSTM branch's gates are rehearsed the same way on fp32 CPU arithmetic.
"""
import numpy as np
import pytest
import torch

from oracle import layer_oracle as lo
from oracle import precision_oracle as po

N_FFT, HOP, NOUT, NOUT_LSTM, CROP = 512, 256, 16, 32, 192


@pytest.fixture(scope='module')
def captured():
    """(prefix, x, y, conv kwargs) of every convolution of one emulated forward, and the float64 state dict"""
    from lib import synth
    from oracle import net_oracle, stft_oracle
    sd = synth.to_torch_state_dict(synth.make_state_dict(N_FFT, NOUT, NOUT_LSTM))
    X = stft_oracle.wave_to_spectrogram(synth.sine_mix(3.0), HOP, N_FFT)
    x = torch.from_numpy(np.abs(X[None, :, :, :CROP]) / np.abs(X).max()).float()
    convs = []

    def conv(sd_, p, x_, stride=1, pad=1, dil=1, act='relu'):
        y = po.Scheme().conv_bn_act(sd_, p, x_, stride, pad, dil, act)
        convs.append((p, x_, y, dict(stride=stride, pad=pad, dil=dil, act=act)))
        return y

    with torch.no_grad():
        net_oracle.forward(sd, x, n_fft=N_FFT, conv=conv)
    return convs, lo.state_dict64(sd, 'cpu')


def test_gate_accepts_three_products_and_rejects_two(captured):
    convs, sd64 = captured
    checked = 0
    worst = [0.0, np.inf, np.inf]
    for p, x, y, kw in convs:
        if p.endswith('.lstm_dec2.conv'):   # the LSTM's 1x1 input convolution is fp32 (test_lstm_gates_on_cpu)
            continue
        r, r_wlo, r_xlo, _, _ = lo.conv_ratios(sd64, p, x.double(), y.double(), **kw)
        assert r <= lo.CONV_GATE, (p, r)
        assert min(r_wlo, r_xlo) >= lo.nonvacuous_factor(sd64, p) * lo.CONV_GATE, (p, r_wlo, r_xlo)
        worst = [max(worst[0], r), min(worst[1], r_wlo), min(worst[2], r_xlo)]
        checked += 1
    assert checked == 5 * 19 + 2   # 19 per BaseNet and the two bridges
    print('three products: max r = %.3g; no_wlo: min r = %.3g; no_xlo: min r = %.3g (gate %.3g)'
          % (worst[0], worst[1], worst[2], lo.CONV_GATE))


def test_upsample_gate_on_cpu(captured):
    """fp32 ATen interpolation (what the kernels reproduce) passes the upsample gate; align_corners=False fails it."""
    convs, _ = captured
    for p, _, y, _ in convs:
        if p.endswith('.aspp.bottleneck') or p.endswith('.dec4.conv1') or p.endswith('.dec3.conv1'):
            low = y.double()   # what the decoders up-sample
            got = torch.nn.functional.interpolate(y, scale_factor=2, mode='bilinear', align_corners=True).double()
            r, r_wrong = lo.upsample_ratios(low, got)
            assert r <= lo.UPSAMPLE_GATE and r_wrong >= lo.NONVACUOUS * lo.UPSAMPLE_GATE, (p, r, r_wrong)


def test_lstm_gates_on_cpu(captured):
    """The branch computed in fp32 on the CPU from the emulated dec2 output passes the LSTM gates, and the reverse
    direction run forwards in time fails the recurrence's."""
    import torch.nn.functional as F
    from oracle import net_oracle
    convs, sd64 = captured
    for p, x, _, _ in convs:
        if not p.endswith('.lstm_dec2.conv'):
            continue
        q = p[:-len('.conv')]
        sd32 = {k: (v.float() if v.is_floating_point() else v) for k, v in sd64.items()}
        scale, shift = po.fold_bn(sd64, q + '.conv.conv.1')
        w = (net_oracle._t(sd64, q + '.conv.conv.0.weight')[0, :, 0, 0] * scale[0]).float()
        l0 = torch.einsum('nchw,c->nhw', x, w)
        a = F.relu(l0 + float(shift[0])).permute(0, 2, 1)
        wih = torch.cat([sd32[f'{q}.lstm.weight_ih_l0{s}'] for s in ('', '_reverse')])
        b = torch.cat([sd32[f'{q}.lstm.bias_ih_l0{s}'] + sd32[f'{q}.lstm.bias_hh_l0{s}'] for s in ('', '_reverse')])
        xp = a @ wih.t() + b
        hs = lo.bilstm(sd32, q, xp)
        n, T, K = hs.shape
        y = net_oracle.lstm_dense(sd32, q, hs.reshape(n * T, K)).reshape(n, T, -1).permute(0, 2, 1)
        r = lo.lstm_ratios(sd64, p[:-len('.lstm_dec2.conv')], x.double(), l0.double(), xp.double(), hs.double(),
                           y.double())
        for k in ('l0', 'xp', 'y'):
            assert r[k] <= lo.FP32_SUM_GATE, (q, k, r[k])
        assert r['hs'] <= lo.LSTM_H_GATE, (q, r['hs'])
        assert r['hs_reverse_forwards'] >= lo.NONVACUOUS * lo.LSTM_H_GATE, (q, r['hs_reverse_forwards'])
