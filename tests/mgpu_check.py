"""Multi-GPU correctness check (run under torchrun on >= 2 GPUs; not collected by pytest, which starts it from
tests/test_gpu_sharded_separation.py when two GPUs are visible): every exchange mode of lib/distributed.py must
reproduce the single-GPU stems bit for bit (the one-GPU emulation of every rank in that file shows why they are
equal)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'vocal-remover_b200'))
import inference  # noqa: E402
from lib import distributed as vr_dist  # noqa: E402
from lib import nets, synth  # noqa: E402


def main():
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    dist.init_process_group('nccl', device_id=dev)
    model = nets.CascadedNet(2048, 1024, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    model.to(dev)
    sp = inference.Separator(model, dev, 4, 256, False)
    wave = synth.sine_mix(31.0)
    d_wave = torch.from_numpy(wave).to(dev)
    ref_inst, ref_voc = sp.separate_wave(d_wave)          # single-GPU fused path on every rank
    ok = True
    for mode in ('sharded', 'p2p', 'nccl'):
        os.environ['VR_GATHER'] = mode
        for rep in range(2):                              # twice: cached buffers / barriers must be reusable
            inst, voc = vr_dist.separate_wave(sp, d_wave, world=world, rank=rank)
        if rank == 0:
            e = max((inst - ref_inst).abs().max().item(), (voc - ref_voc).abs().max().item())
            print('mode %-8s device-resident max |diff| vs single GPU: %.3g' % (mode, e), flush=True)
            ok = ok and e == 0.0
    os.environ['VR_GATHER'] = 'sharded'
    # --tta (inference.py:83-98): both passes sharded by the same frame spans, combined locally
    ref_inst_t, ref_voc_t = sp.separate_wave(d_wave, tta=True)
    for rep in range(2):
        inst, voc = vr_dist.separate_wave(sp, d_wave, tta=True, world=world, rank=rank)
    if rank == 0:
        e = max((inst - ref_inst_t).abs().max().item(), (voc - ref_voc_t).abs().max().item())
        print('mode sharded+tta device-resident max |diff| vs single GPU: %.3g' % e, flush=True)
        ok = ok and e == 0.0
    h_wave = torch.from_numpy(wave).pin_memory()
    Lo = ref_inst.shape[1]
    h_inst = torch.zeros((2, Lo)).pin_memory()
    h_voc = torch.zeros((2, Lo)).pin_memory()
    s0, s1 = vr_dist.separate_wave_host(sp, h_wave, h_inst, h_voc, world=world, rank=rank)
    e = 0.0
    if s1 > s0:
        e = max((h_inst[:, s0:s1] - ref_inst[:, s0:s1].cpu()).abs().max().item(),
                (h_voc[:, s0:s1] - ref_voc[:, s0:s1].cpu()).abs().max().item())
    spans = [None] * world
    dist.all_gather_object(spans, (s0, s1, e))
    if rank == 0:
        print('host-sharded slices:', spans, flush=True)
        ok = ok and spans[0][0] == 0 and spans[-1][1] == Lo and all(x[1] == y[0] for x, y in zip(spans, spans[1:]))
        ok = ok and all(x[2] == 0.0 for x in spans)
        print('MGPU_CHECK', 'PASS' if ok else 'FAIL', flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
