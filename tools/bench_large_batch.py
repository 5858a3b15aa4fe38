"""Training steps with large triplet batches on the C2 data (100 000 synthetic tf-idf rows, F = 10 000, H = 500), one JSON line.

    python tools/bench_large_batch.py [--batch-sizes 800,4096,9800,16384,32768] [--strategies batch_all,batch_hard]
                                      [--steps 3] [--warmup 1] [--ab-rounds 5] [--mining-block-rows R] [--classes 4]

For each strategy and batch size B:
  * step_ms: a replayed CUDA graph of the whole step (the path `fit` takes), median of --steps CUDA-event timings, the same batch
    every replay; articles_per_s = B / step time;
  * kernels_ms: one eager step on a single stream with each launch bracketed by CUDA events -- batch preparation, Gram GEMM,
    mining sweep, (G + G^T).E GEMM and the fused decode (median of two steps);
  * peak_gb: torch's peak allocated device memory over the configuration.
With --mining-block-rows R the engines mine S in blocks of R anchor rows (batches up to 262 144 rows), and kernels_ms holds each
phase's total over one eager step (after a warm-up step): preparation, Gram blocks, rows kernels, G's hi / lo split (batch_hard),
dE2 GEMMs, batch_hard's finish and the fused decode.
For batch_all at B <= 4096 the in-shared-memory sweep and the tiled sweep (the kernel used above 4096, forced through
dae_triplet_config) are also timed alternately, kernel alone and as the replayed step.
The card name and its power limit go into the JSON line.  Nothing is written to the source tree.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KERNELS = ('dae_batch_prepare', 'gemm_gram', 'dae_triplet_batch_all', 'dae_triplet_batch_hard', 'gemm_dE_tri', 'gemm_decode_fwd')
PHASES_BLOCKED = ('dae_batch_prepare_blocked', 'gemm_gram', 'dae_triplet_batch_all_rows', 'dae_triplet_batch_hard_rows', 'dae_split_bf16',
                  'gemm_dE_tri', 'dae_triplet_batch_hard_finish', 'gemm_decode_fwd')


def _power_limit_w():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:   # noqa: BLE001 -- no nvidia-smi: the limit is reported as unknown
        return None


def _time_replays(graph, n):
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        graph.replay()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch-sizes', default='800,4096,9800,16384,32768')
    ap.add_argument('--strategies', default='batch_all,batch_hard')
    ap.add_argument('--rows', type=int, default=100000)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--ab-rounds', type=int, default=5)
    ap.add_argument('--mining-block-rows', type=int, default=0, help='R > 0: block mining (TrainEngine(mining_block_rows=R))')
    ap.add_argument('--classes', type=int, default=4)
    a = ap.parse_args()
    R = a.mining_block_rows or None
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200._cabi import call, ptr
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    F, H = 10000, 500
    dev = torch.device('cuda:0')
    x = make_sparse(a.rows, F, 100, 'tfidf', seed=0)
    labels = make_labels(a.rows, a.classes, seed=0)
    W0 = np.random.default_rng(1).uniform(-1, 1, (F, H)).astype(np.float32) * np.sqrt(6.0 / (F + H))
    csr = DeviceCSR(x, dev)
    lab_d = torch.from_numpy(labels).to(dev)
    out = {'workload': 'C2 data: %d synthetic tf-idf rows, F=%d, H=%d, %d classes, masking 0.3, SGD' % (a.rows, F, H, a.classes),
           'mining_block_rows': R, 'device': torch.cuda.get_device_name(dev), 'power_limit_w': _power_limit_w(), 'results': [],
           'sweep_ab': []}
    for strategy in a.strategies.split(','):
        for B in [int(b) for b in a.batch_sizes.split(',')]:
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats(dev)
            eng = TrainEngine(F, H, device=dev, triplet_strategy=strategy, opt='gradient_descent', learning_rate=0.1,
                              mining_block_rows=R)
            eng.set_parameters(W0)
            eng.set_data(csr, None, lab_d)
            eng.corrupt_masking(0.3, seed=1234)
            perm = torch.randperm(a.rows, device=dev, dtype=torch.int32)
            # per-kernel times: eager steps on one stream
            eng.fork_branches = False
            if R is None:
                eng.time_kernels(KERNELS)
                for _ in range(2):
                    eng.step(perm, 0, B)
                kt = {k: float(np.median(v)) for k, v in eng.kernel_times_ms().items() if v}
            else:   # one block loop launches each phase's kernels many times: their total over the second eager step
                eng.step(perm, 0, B)
                eng.time_kernels(PHASES_BLOCKED)
                eng.step(perm, 0, B)
                kt = {k: float(np.sum(v)) for k, v in eng.kernel_times_ms().items() if v}
            eng.time_kernels(None)
            eng.fork_branches = True
            g = eng.capture_step_graph(perm, B, None, row_stride=0)
            eng.set_step_cursor(0, 0)
            for _ in range(a.warmup):
                g.replay()
            ms = _time_replays(g, a.steps)
            torch.cuda.synchronize()
            stats = eng.read_stats()
            row = {'strategy': strategy, 'B': B, 'step_ms': ms, 'articles_per_s': B / ms * 1e3, 'kernels_ms': kt,
                   'peak_gb': torch.cuda.max_memory_allocated(dev) / 1e9, 'cost': stats['cost'], 'triplet_loss': stats['triplet_loss']}
            if strategy == 'batch_all' and B <= 4096 and R is None:
                g_tiled = None
                try:
                    call('dae_triplet_config', 1)
                    g_tiled = eng.capture_step_graph(perm, B, None, row_stride=0)
                finally:
                    call('dae_triplet_config', 0)
                eng.set_step_cursor(0, 0)
                st = torch.cuda.current_stream().cuda_stream
                args = (ptr(eng.S), B, B, ptr(eng.seg_lo), ptr(eng.seg_hi), ptr(eng.G), B, ptr(eng.stats), 0, ptr(eng.GG_hi),
                        ptr(eng.GG_lo), eng.GG_hi.stride(0), st)
                k_ms = {0: [], 1: []}
                s_ms = {0: [], 1: []}
                for _ in range(a.ab_rounds):
                    for tiled in (0, 1):
                        call('dae_triplet_config', tiled)
                        try:
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record()
                            call('dae_triplet_batch_all', *args)
                            e1.record()
                            e1.synchronize()
                            k_ms[tiled].append(e0.elapsed_time(e1))
                        finally:
                            call('dae_triplet_config', 0)
                        s_ms[tiled].append(_time_replays(g_tiled if tiled else g, 1))
                out['sweep_ab'].append({'B': B, 'sweep_ms_shared': float(np.median(k_ms[0])), 'sweep_ms_tiled': float(np.median(k_ms[1])),
                                        'sweep_ms_shared_all': k_ms[0], 'sweep_ms_tiled_all': k_ms[1],
                                        'step_ms_shared': float(np.median(s_ms[0])), 'step_ms_tiled': float(np.median(s_ms[1]))})
                del g_tiled
            out['results'].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            del g, eng
            torch.cuda.synchronize()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
