"""The deterministic training mode against the default mode (DESIGN 4.7), one JSON line.

    python tools/bench_deterministic.py [--configs C1,C2,C3,C4] [--rows 20000] [--steps 50] [--runs 3]

For each bench.py configuration (C1 UCI / strategy none, C2 batch_all, C3 batch_hard, C4 F = 50 000 / H = 1000 batch_all; B = 800,
the configuration's data maker, --rows articles):
  * step_ms: one engine per mode, each with its replayed CUDA graph of the whole step; the two modes' windows of --steps replays
    alternate --runs times, each window timed with CUDA events; median and range per mode;
  * kernels_us: three eager steps on ONE stream under torch.profiler, mean device time per step of every kernel whose time differs
    between the modes or that only one mode runs (the deterministic mode's new kernels: bucketing, dbh levels, gather, sparse add,
    stream-K fixups, loss-slot sum);
  * workspace_mb: the deterministic mode's extra device buffers (3 GEMM workspaces, decode loss partials, loss slots, encode-backward
    workspace).
The card name and its power limit go into the JSON line.  Nothing is written to the source tree.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _power_limit_w():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:   # noqa: BLE001 -- no nvidia-smi: the limit is reported as unknown
        return None


def _engine(w, x, labels, det, dev):
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    import bench
    eng = TrainEngine(w['F'], w['H'], enc_act_func=w['enc'], dec_act_func=w['dec'], loss_func=w['loss'], opt=w['opt'],
                      learning_rate=w['lr'], alpha=w['alpha'], triplet_strategy=w['strategy'], device=dev, deterministic=det)
    eng.set_parameters(bench.xavier(w['F'], w['H'], 0))
    eng.set_data(DeviceCSR(x, dev), None, torch.from_numpy(labels).to(dev))
    eng.corrupt_masking(w['corr_frac'], seed=1234, epoch=0)
    g = torch.Generator(device=dev)
    g.manual_seed(4321)
    perm = torch.randperm(x.shape[0], device=dev, dtype=torch.int32, generator=g)
    return eng, perm


def _window(eng, K, steps_per_epoch):
    """K replays from a cursor at 0, back to 0 after every steps_per_epoch (the permutation's end), as bench.py's epochs do."""
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(20_000_000)      # the K replays are enqueued behind a spin: device time, not host launch gaps
    a.record()
    for i in range(K):
        if i % steps_per_epoch == 0:
            eng.set_step_cursor(0, 0)
        eng.replay_step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / K


def _kernels(eng, perm, B, n=3):
    """Mean device microseconds per step of every kernel, n eager single-stream steps under torch.profiler."""
    from torch.profiler import profile, ProfilerActivity
    eng.fork_branches = False
    eng.step(perm, 0, B)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(n):
            eng.step(perm, s * B, B)
        torch.cuda.synchronize()
    eng.fork_branches = True
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            out[ev.key[:90]] = out.get(ev.key[:90], 0.0) + t / n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='C1,C2,C3,C4')
    ap.add_argument('--rows', type=int, default=20000)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--runs', type=int, default=3)
    args = ap.parse_args()
    import bench
    dev = torch.device('cuda', 0)
    res = {'device': torch.cuda.get_device_name(dev), 'power_limit_w': _power_limit_w(), 'rows': args.rows, 'steps': args.steps,
           'runs': args.runs, 'configs': {}}
    for name in args.configs.split(','):
        w = bench.CONFIGS[name]
        B = w['B']
        x, labels = bench.make_data(w, min(args.rows, w['rows']), seed=1000)
        spe = x.shape[0] // B
        engines = {}
        for det in (False, True):
            eng, perm = _engine(w, x, labels, det, dev)
            eng.capture_step_graph(perm, B, None)
            engines[det] = (eng, perm)
        times = {False: [], True: []}
        for _ in range(args.runs):
            for det in (False, True):
                times[det].append(_window(engines[det][0], args.steps, spe))
        kern = {det: _kernels(engines[det][0], engines[det][1], B) for det in (False, True)}
        e = engines[True][0]
        ws = {'gemm': sum(t.numel() for t in e.gemm_ws) / 1e6, 'decode_loss_parts': e.loss_parts.numel() * 4 / 1e6,
              'loss_slots': e.loss_slots.numel() * 8 / 1e6, 'encode_backward': e.enc_det_ws.numel() / 1e6}
        diff = {}
        for k in sorted(set(kern[False]) | set(kern[True])):
            a, b = kern[False].get(k, 0.0), kern[True].get(k, 0.0)
            if abs(a - b) > max(1.0, 0.05 * a):   # the kernels one mode adds, or whose time the mode changes
                diff[k] = [round(a, 1), round(b, 1)]
        res['configs'][name] = {
            'workload': w['name'],
            'step_ms': {m: {'median': float(np.median(times[det])), 'min': float(np.min(times[det])), 'max': float(np.max(times[det]))}
                        for m, det in (('default', False), ('deterministic', True))},
            'kernels_us_default_vs_deterministic': diff,
            'workspace_mb': {k: round(v, 2) for k, v in ws.items()},
        }
        del engines, e
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
