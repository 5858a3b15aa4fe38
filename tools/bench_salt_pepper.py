"""Salt-and-pepper corruption on the device (dae_salt_pepper_csr) at the bench.py shapes, one JSON line.

    python tools/bench_salt_pepper.py [--configs C1,C2,C4] [--fit C1,C2] [--reps 5]

For each configuration (bench.py's data maker and its rows; v = round(0.3 F)):
  * corrupt_ms: TrainEngine.corrupt_salt_pepper over the whole set, CUDA-event median of --reps calls, in Philox mode (device) and in
    host-draw mode (upload of N x v uint32 draws + kernels, host clock around a synchronised call; the draws are random numbers of the
    right shape, not the reference's stream);
  * host_function_s: utils.salt_and_pepper_noise on a row sample, EXTRAPOLATED linearly to all rows;
  * numpy_draws_s: utils.salt_and_pepper_draws (the rng_mode='numpy' draws) on a row sample, EXTRAPOLATED linearly to all rows;
  * buffers_gb: the corrupted-CSR buffers (capacity x 8 B + indptr) and the entries stored per row.
For each --fit configuration, DenoisingAutoencoder.fit (3 epochs, B = 800, rng_mode 'device') with corr_type 'masking' and
'salt_and_pepper': the last epoch's time, the replayed step (CUDA events over one epoch of replays of the captured graph) and the encode
forward / backward kernels' device time (events around each launch, 5 eager steps).
The card name and its power limit go into the JSON line.  Nothing is written to the source tree.
"""
import argparse
import functools
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                           timeout=20)
        return r.stdout.strip()
    except Exception as e:   # noqa: BLE001 -- no nvidia-smi: reported as such
        return 'nvidia-smi failed: %s' % e


@functools.lru_cache(maxsize=1)
def _data(cfg):
    import bench
    w = bench.CONFIGS[cfg]
    x, labels = bench.make_data(w, w['rows'], 0)
    x = x.tocsr().astype(np.float32)
    x.sort_indices()
    return w, x, labels


def corruption(cfg, reps):
    from dae_rnn_news_recommendation_b200.autoencoder import utils
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    w, x, _ = _data(cfg)
    N, F = x.shape
    v = int(round(0.3 * F))
    lo, hi = float(x.min()), float(x.max())
    eng = TrainEngine(F, 16, device='cuda:0', triplet_strategy='none')
    eng.set_data(DeviceCSR(x, eng.device), None, None)
    out = {'rows': N, 'F': F, 'v': v, 'clean_nnz_per_row': x.nnz / N}
    ev = []
    for e in range(reps + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.corrupt_salt_pepper(v, lo, hi, seed=1, epoch=e)
        b.record()
        ev.append((a, b))
    torch.cuda.synchronize()
    t = [a.elapsed_time(b) for a, b in ev[2:]]
    out['corrupt_ms_philox'] = {'median': float(np.median(t)), 'min': min(t), 'max': max(t)}
    sp_ = eng.salt_pepper_buffers(v)
    stored = int(eng.csr_c.indptr[-1].item())
    out['capacity_entries'] = sp_['cap']
    out['buffers_gb'] = (sp_['cap'] * 8 + (N + 1) * 8) / 1e9
    out['stored_per_row'] = stored / N
    draws = np.random.default_rng(0).integers(0, F, N * v, dtype=np.uint32)
    draws[1::2] |= np.uint32(1 << 31)
    t = []
    for e in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.corrupt_salt_pepper(v, lo, hi, draws_host=draws)
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    out['corrupt_ms_host_draws'] = {'median': float(np.median(t[1:])), 'min': min(t[1:]), 'max': max(t[1:]), 'draw_bytes': N * v * 4}
    eng.check_corruption()
    del draws, eng
    torch.cuda.empty_cache()
    sample = 100 if F <= 10000 else 20
    xs = x[:sample]
    t0 = time.perf_counter()
    utils.salt_and_pepper_noise(xs, v)
    out['host_function_s_extrapolated'] = (time.perf_counter() - t0) * N / sample
    out['host_function_sample_rows'] = sample
    ns = min(N, 2000)
    t0 = time.perf_counter()
    utils.salt_and_pepper_draws(x[:ns], v)
    out['numpy_draws_s_extrapolated'] = (time.perf_counter() - t0) * N / ns
    out['numpy_draws_sample_rows'] = ns
    return out


def fit(cfg, corr):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder
    import bench
    w, x, labels = _data(cfg)
    strategy = w['strategy']
    with tempfile.TemporaryDirectory() as d:
        cwd = os.getcwd()
        os.chdir(d)
        try:
            m = DenoisingAutoencoder(model_name='b', main_dir='b', compress_factor=w['F'] // w['H'], enc_act_func=w['enc'],
                                     dec_act_func=w['dec'], loss_func=w['loss'], num_epochs=3, batch_size=w['B'], opt=w['opt'],
                                     learning_rate=w['lr'], corr_type=corr, corr_frac=w['corr_frac'], verbose=False, verbose_step=100,
                                     seed=0, triplet_strategy=strategy, W_init=bench.xavier(w['F'], w['H'], 0))
            m.fit(x, train_set_label=labels if strategy != 'none' else None)
        finally:
            os.chdir(cwd)
    eng = m.engine
    assert eng._graph is not None, 'the fit did not replay a captured graph'
    out = {'epoch_ms_last': m.train_time * 1e3}
    N, B = x.shape[0], w['B']
    steps = N // B
    torch.cuda.synchronize()
    eng.set_step_cursor(0, 0)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        eng.replay_step()
    b.record()
    torch.cuda.synchronize()
    out['replayed_step_ms'] = a.elapsed_time(b) / steps
    perm = torch.arange(N, dtype=torch.int32, device=eng.device)
    names = ['dae_encode_csr_fwd', 'dae_encode_csr_bwd']
    eng.time_kernels(names)
    for s in range(5):
        eng.step(perm, s * B, B)
    kt = eng.kernel_times_ms()
    eng.time_kernels(None)
    out['encode_fwd_us'] = float(np.median(kt[names[0]])) * 1e3
    out['encode_bwd_us'] = float(np.median(kt[names[1]])) * 1e3
    out['corrupted_nnz_per_row'] = float(eng.csr_c.indptr[-1].item()) / N
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='C1,C2,C4')
    ap.add_argument('--fit', default='C1,C2')
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_salt_pepper: no CUDA device (this measures the GPU)')
    res = {'card': _card(), 'device_name': torch.cuda.get_device_name(0), 'corruption': {}, 'fit': {}}
    for cfg in [c for c in a.configs.split(',') if c]:
        res['corruption'][cfg] = corruption(cfg, a.reps)
        torch.cuda.empty_cache()
        print(cfg, json.dumps(res['corruption'][cfg]), file=sys.stderr, flush=True)
    for cfg in [c for c in a.fit.split(',') if c]:
        res['fit'][cfg] = {corr: fit(cfg, corr) for corr in ('masking', 'salt_and_pepper')}
        torch.cuda.empty_cache()
        print(cfg, json.dumps(res['fit'][cfg]), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
