"""Times BSS Eval on the GPU (csrc/bsseval.cu through lib/bsseval.py) on a 4-minute stereo pair.

Input: instruments ``0.5 * synth.sine_mix(240)``, vocals the same sines an octave down, the mixture their sum, and the
two stems of separating the mixture with the seeded checkpoint (synth.make_state_dict) as the estimates: K = C = 2,
N = 10.6 M samples, 1 s frames, 512-tap filters.  Reported: the three phases of ``vr_bss_eval`` (correlations,
assembly + Cholesky + solves, projections + frame sums) and the whole call on the GPU, from its CUDA events, as the
median of --runs after warm-up; the wall time of one ``bss_eval`` call; the float64 oracle's time on the host CPU in
the same run and its largest difference from the GPU; the ``separate_wave`` time of the same track; and the fp64 FLOP/s
of each phase from the op counts below.  The card's name and power limit are read in the same run (read-only
``nvidia-smi --query-gpu``).

Op counts (one multiply-add = 2 flops), M = K * C, Lc = L rounded up to 128, Lp = L rounded up to 16, n = M * L:
  correlations  M * 2M * Lc * N multiply-adds (every lag of every reference against every reference and estimate)
  solves        n^3 / 3 + K (C L)^3 / 3 flops of Cholesky, 2 n^2 M + K 2 (C L)^2 C of triangular solves
  projections   M * (M + C) * Lp multiply-adds per frame sample (the P_all and P_j FIRs of every estimate channel)

With --framewise the same pair is scored with framewise filters (BSS Eval v3: every frame its own systems) instead,
and the track-filter call is timed in the same run.  Op counts then (nwin frames of ``window`` samples, T = the
projection timeline window + L - 1):
  correlations  nwin * M * 2M * Lc * window multiply-adds
  Cholesky      nwin * (n^3 / 3 + K (C L)^3 / 3) flops, and nwin * 128 KB * (Tn^3 + K Tb^3) / 6 bytes of tile traffic:
                each 64 x 64 trailing-tile update reads two panel tiles and reads and writes its own (Tn, Tb: the
                tiles along a full and a block system)
  projections   nwin * M * (M + C) * Lp * T multiply-adds
The oracle then runs on an excerpt (the first --excerpt seconds; each frame only depends on its own samples, so these
are the track's first frames), and --long MINUTES times one call on a synthetic noise pair of that length with the
batch chosen by the default workspace budget.

Usage: python profiles/bsseval.py [--seconds 240] [--runs 20] [--no-oracle] [--out bsseval.json]
       python profiles/bsseval.py --framewise [--excerpt 10] [--long 40]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'vocal-remover_b200')
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def _gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # the numbers stay valid; the card is then named by torch only
        return dict(gpu=None, nvidia_smi_error=str(e))


def op_counts(K, C, N, L, window, hop):
    from lib import bsseval
    M = K * C
    Lc, Lp = -(-L // 128) * 128, -(-L // 16) * 16
    n, nb = M * L, C * L
    nwin = bsseval.frame_count(N, window, hop)
    covered = min(N, (nwin - 1) * hop + window) if hop <= window else nwin * window
    return dict(correlation=2.0 * M * 2 * M * Lc * N,
                solve=n ** 3 / 3.0 + K * nb ** 3 / 3.0 + 2.0 * n * n * M + K * 2.0 * nb * nb * C,
                projection=2.0 * M * (M + C) * Lp * covered)


FP64_FMA_PEAK = 33.5e12   # H100 SXM, fp64 without the tensor cores (data sheet, 700 W)
HBM_PEAK = 3.35e12


def framewise_op_counts(K, C, N, L, window, hop):
    from lib import bsseval
    M = K * C
    Lc, Lp = -(-L // 128) * 128, -(-L // 16) * 16
    n, nb = M * L, C * L
    Tn, Tb = -(-n // 64), -(-nb // 64)
    nwin = bsseval.frame_count(N, window, hop)
    return dict(correlation=2.0 * nwin * M * 2 * M * Lc * window,
                cholesky=nwin * (n ** 3 / 3.0 + K * nb ** 3 / 3.0),
                cholesky_bytes=nwin * 128 * 1024 * (Tn ** 3 + K * Tb ** 3) / 6.0,
                projection=2.0 * nwin * M * (M + C) * Lp * (window + L - 1))


def framewise(args, refs, ests, sep_ms, sr):
    import torch
    from lib import bsseval
    K, C, N = (int(v) for v in refs.shape)
    L, window, hop = args.filters_len, sr, sr
    runs = {'v3': [], 'v4': []}
    for i in range(2 + args.runs):   # the two modes alternate
        for mode in ('v3', 'v4'):
            out = bsseval.frame_sums(refs, ests, window, hop, L, timings=True, framewise=mode == 'v3')
            if i >= 2:
                runs[mode].append(out['phase_ms'])
            if mode == 'v3':
                v3 = out
    ph3, ph4 = (np.median(np.asarray(runs[m]), axis=0) for m in ('v3', 'v4'))
    ops = framewise_op_counts(K, C, N, L, window, hop)
    bound = dict(correlation_min_ms=ops['correlation'] / FP64_FMA_PEAK * 1e3,
                 cholesky_flop_min_ms=ops['cholesky'] / FP64_FMA_PEAK * 1e3,
                 cholesky_byte_min_ms=ops['cholesky_bytes'] / HBM_PEAK * 1e3,
                 projection_min_ms=ops['projection'] / FP64_FMA_PEAK * 1e3)
    got = bsseval.metrics(v3['sums'])
    res = dict(_gpu_info(), torch_device=torch.cuda.get_device_name(refs.device), mode='framewise (v3)', K=K, C=C,
               N=N, filters_len=L, window=window, hop=hop, runs=args.runs,
               frames_per_batch=v3['frames_per_batch'],
               correlation_ms=float(ph3[0]), solve_ms=float(ph3[1]), projection_ms=float(ph3[2]),
               bss_eval_framewise_gpu_ms=float(ph3[3]), bss_eval_v4_gpu_ms=float(ph4[3]),
               v4_phase_ms=ph4.tolist(), separate_wave_ms=float(np.median(sep_ms)),
               correlation_tflops=ops['correlation'] / ph3[0] * 1e-9,
               solve_tflops=ops['cholesky'] / ph3[1] * 1e-9,
               solve_tile_gbytes_per_s=ops['cholesky_bytes'] / ph3[1] * 1e-6,
               projection_tflops=ops['projection'] / ph3[2] * 1e-9,
               op_counts=ops, least_time=bound,
               track_medians={m: bsseval.track_medians(got)[m].tolist() for m in bsseval.METRICS})
    if not args.no_oracle:
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        import bsseval_framewise_oracle as fo
        n = int(args.excerpt * sr)
        s_host, e_host = refs[:, :, :n].cpu().numpy(), ests[:, :, :n].cpu().numpy()
        t = time.perf_counter()
        want = fo.bss_eval_framewise(s_host, e_host, window, hop, L)
        res['oracle_excerpt_s'] = args.excerpt
        res['oracle_excerpt_cpu_s'] = time.perf_counter() - t
        res['oracle_cpu_threads'] = os.cpu_count()
        nw = want['sdr'].shape[1]
        res['excerpt_max_abs_db_vs_oracle'] = max(float(np.nanmax(np.abs(got[m][:, :nw] - want[m])))
                                                 for m in bsseval.METRICS)
    if args.long:
        rng = np.random.default_rng(7)
        n = int(args.long * 60 * sr)
        s = torch.from_numpy(rng.standard_normal((2, 2, n), dtype=np.float32)).to(refs.device)
        e = s + 0.3 * s.flip(0) + 0.1 * torch.randn(s.shape, generator=torch.Generator(device=refs.device).manual_seed(8),
                                                    device=refs.device)
        free, _ = torch.cuda.mem_get_info(refs.device)
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = bsseval.frame_sums(s, e, window, hop, L, framewise=True, timings=True)
        res['long'] = dict(minutes=args.long, N=n, frames=int(out['sums'].shape[1]),
                           frames_per_batch=out['frames_per_batch'], budget_bytes=min(free // 4, bsseval.WORKSPACE_CAP),
                           wall_s=time.perf_counter() - t, gpu_ms=float(out['phase_ms'][3]),
                           max_allocated_bytes=torch.cuda.max_memory_allocated(refs.device))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=240.0)
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--filters_len', type=int, default=512)
    ap.add_argument('--no-oracle', action='store_true')
    ap.add_argument('--framewise', action='store_true', help='time BSS Eval v3 (framewise filters) and v4 together')
    ap.add_argument('--excerpt', type=float, default=10.0, help='--framewise: seconds the oracle scores')
    ap.add_argument('--long', type=float, default=0.0, help='--framewise: minutes of a synthetic pair scored once')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    import inference
    from lib import bsseval, nets, synth
    dev = torch.device('cuda:0')
    sr = 44100
    inst = 0.5 * synth.sine_mix(args.seconds, seed=1)
    voc = 0.5 * synth.sine_mix(args.seconds / 2, sr=2 * sr, seed=2)[:, :inst.shape[1]]
    X = (inst + voc).astype(np.float32)
    model = nets.CascadedNet(2048, 1024, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    model.to(dev)
    sp = inference.Separator(model, dev, 4, 256, False)
    d_x = torch.from_numpy(X).to(dev)
    d_inst = torch.from_numpy(np.ascontiguousarray(inst, dtype=np.float32)).to(dev)

    def separate():
        return sp.separate_wave(d_x)

    est_i, est_v = separate()
    n = est_i.shape[1]
    refs = torch.stack([d_inst[:, :n], (d_x - d_inst)[:, :n]]).contiguous()
    ests = torch.stack([est_i, est_v]).contiguous()
    K, C, N = refs.shape
    L, window, hop = args.filters_len, sr, sr

    sep_ms = []
    for i in range(3 + args.runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        separate()
        b.record()
        b.synchronize()
        if i >= 3:
            sep_ms.append(a.elapsed_time(b))

    if args.framewise:
        res = framewise(args, refs, ests, sep_ms, sr)
        print(json.dumps(res, indent=1))
        if args.out:
            with open(args.out, 'w') as f:
                json.dump(res, f, indent=1)
        return

    phases, walls = [], []
    for i in range(3 + args.runs):
        t = time.perf_counter()
        out = bsseval.frame_sums(refs, ests, window, hop, L, timings=True)
        wall = time.perf_counter() - t
        if i >= 3:
            phases.append(out['phase_ms'])
            walls.append(wall * 1e3)
    phases = np.median(np.asarray(phases), axis=0)
    got = bsseval.metrics(out['sums'])

    ops = op_counts(K, C, N, L, window, hop)
    res = dict(_gpu_info(), torch_device=torch.cuda.get_device_name(dev), K=int(K), C=int(C), N=int(N),
               filters_len=L, window=window, hop=hop, runs=args.runs,
               correlation_ms=float(phases[0]), solve_ms=float(phases[1]), projection_ms=float(phases[2]),
               bss_eval_gpu_ms=float(phases[3]), bss_eval_wall_ms=float(np.median(walls)),
               separate_wave_ms=float(np.median(sep_ms)),
               correlation_tflops=ops['correlation'] / phases[0] * 1e-9,
               solve_tflops=ops['solve'] / phases[1] * 1e-9,
               projection_tflops=ops['projection'] / phases[2] * 1e-9,
               op_counts=ops, track_medians={m: bsseval.track_medians(got)[m].tolist() for m in bsseval.METRICS})
    if not args.no_oracle:
        from oracle import bsseval_oracle
        s_host, e_host = refs.cpu().numpy(), ests.cpu().numpy()
        t = time.perf_counter()
        want = bsseval_oracle.bss_eval(s_host, e_host, window, hop, L)
        res['oracle_cpu_s'] = time.perf_counter() - t
        res['oracle_cpu_threads'] = os.cpu_count()
        res['max_abs_db_vs_oracle'] = max(float(np.nanmax(np.abs(got[m] - want[m]))) for m in bsseval.METRICS)
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
