"""Near-duplicate pairs (every pair with similarity >= tau): helpers.similar_pairs against the alternatives a user has without it.
One JSON line.

    python tools/bench_similar_pairs.py [--dense_n 100000,1000000] [--h 500] [--reps 3] [--warmup 1] [--chunked_max_n 200000]

Workloads:
  dense   clustered embeddings (clusters of ~21 rows) on the device, cosine, self join, at two thresholds calibrated on a sample of
          rows to give about 10 and about 0.1 pairs per row
  c1      the UCI fixture's training articles (tests/golden/uci_c1.npz), binary, cosine, self join
  c2like  100 000 synthetic tf-idf rows (synth.make_sparse), linear kernel, self join
Paths, each from the operands on the device to device results, in rotating order after warm-up, CUDA events around one call:
  pairs     similar_pairs(to_host=False): the thresholded-pair kernel, the sort into (i, j) order included (sparse: from the
            device CSR, as topk10, so the host normalisation and upload are not timed)
  topk10    top_k_similar(k=10) (dense or sparse)
  chunked   pairwise_similarity's GEMM in row blocks of 4096 x N + (block >= tau).nonzero() (dense, up to --chunked_max_n rows)
Executed TFLOP/s count the three bf16 products of the bf16x3 scheme over the computed tiles (the lower triangle and the diagonal of
128 x 128 tiles, dim padded to the 64-wide k-blocks).  Peak memory is torch's allocator peak above what was allocated before the
call (the inputs).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dae_rnn_news_recommendation_b200 import helpers  # noqa: E402


def _gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi failed: %s' % e


def _time(paths, reps, warmup):
    """{name: (median ms, peak bytes above the inputs, result)} with the paths in rotating order."""
    names = list(paths)
    for _ in range(warmup):
        for nm in names:
            paths[nm]()
    times = {nm: [] for nm in names}
    peaks = {nm: 0 for nm in names}
    results = {}
    for r in range(reps):
        for nm in names[r % len(names):] + names[:r % len(names)]:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = paths[nm]()
            b.record()
            torch.cuda.synchronize()
            times[nm].append(a.elapsed_time(b))
            peaks[nm] = max(peaks[nm], torch.cuda.max_memory_allocated() - base)
            results[nm] = out
            del out
    return {nm: (float(np.median(times[nm])), int(peaks[nm]), results[nm]) for nm in names}


def _calibrate(hi, lo, n, h, per_row, sample=256):
    """tau giving about per_row pairs (i > j) per row: from the scores of `sample` rows against all rows (self match dropped)."""
    rows = torch.randperm(n, device=hi.device)[:sample]
    out = torch.empty(sample, n, dtype=torch.float32, device=hi.device)
    helpers._gemm_nt((hi[rows].contiguous(), lo[rows].contiguous()), (hi, lo), sample, n, h, out)
    out[torch.arange(sample, device=out.device), rows] = -2.0
    k = int(round(2 * per_row * sample))     # both orientations of a pair
    return float(torch.topk(out.flatten(), k).values[-1].item())


def dense_workload(n, h, reps, warmup, chunked_max_n):
    g = torch.Generator(device='cuda').manual_seed(n)
    centres = torch.randn(n // 21 + 1, h, device='cuda', generator=g)
    lab = torch.randint(0, centres.shape[0], (n,), device='cuda', generator=g)
    x = centres[lab] + 0.6 * torch.randn(n, h, device='cuda', generator=g)
    del centres, lab
    hi, lo, _ = helpers._normalised_operands(x, 2)
    out = []
    for per_row in (10.0, 0.1):
        tau = _calibrate(hi, lo, n, h, per_row)
        paths = {'pairs': lambda: helpers.similar_pairs(x, tau, to_host=False),
                 'topk10': lambda: helpers.top_k_similar(x, k=10, to_host=False)}
        if n <= chunked_max_n:
            def chunked():
                res = []
                blk = torch.empty(4096, n, dtype=torch.float32, device='cuda')
                for r0 in range(0, n, 4096):
                    r1 = min(n, r0 + 4096)
                    helpers._gemm_nt((hi[r0:r1], lo[r0:r1]), (hi, lo), r1 - r0, n, h, blk)
                    nz = (blk[:r1 - r0, :r0 + 4096] >= tau).nonzero()
                    nz = nz[nz[:, 0] + r0 > nz[:, 1]]
                    res.append((nz[:, 0] + r0, nz[:, 1], blk[nz[:, 0], nz[:, 1]]))
                return res
            paths['chunked'] = chunked
        t = _time(paths, reps, warmup)
        tm = (n + 127) // 128
        flops = tm * (tm + 1) / 2 * 128 * 128 * ((h + 63) // 64 * 64) * 2 * 3
        n_pairs = int(t['pairs'][2][0].shape[0])
        rec = {'workload': 'dense', 'n': n, 'h': h, 'metric': 'cosine', 'tau': tau, 'target_pairs_per_row': per_row,
               'pairs': n_pairs, 'pairs_per_row': n_pairs / n, 'executed_tflops': flops / (t['pairs'][0] * 1e-3) / 1e12}
        for nm, (ms, peak, _) in t.items():
            rec[nm + '_ms'] = ms
            rec[nm + '_peak_mb'] = peak / 1e6
        if 'chunked' in t:
            rec['chunked_pairs'] = int(sum(r[0].shape[0] for r in t['chunked'][2]))
        out.append(rec)
        print(json.dumps(rec), file=sys.stderr, flush=True)
    return out


def sparse_workload(name, x, metric, tau, reps, warmup):
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    d = DeviceCSR(helpers._csr_operand(x, metric), torch.device('cuda:0'))
    paths = {'pairs': lambda: helpers._csr_similarity_pairs(d, d, True, float(np.float32(tau)), 1 << 28, tau),
             'topk10': lambda: helpers._csr_similarity_topk(d, d, 10, exclude=True)}
    t = _time(paths, reps, warmup)
    rec = {'workload': name, 'n': x.shape[0], 'features': x.shape[1], 'nnz': int(x.nnz), 'metric': metric, 'tau': tau,
           'pairs': int(t['pairs'][2][0].shape[0])}
    for nm, (ms, peak, _) in t.items():
        rec[nm + '_ms'] = ms
        rec[nm + '_peak_mb'] = peak / 1e6
    print(json.dumps(rec), file=sys.stderr, flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dense_n', default='100000,1000000')
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--chunked_max_n', type=int, default=200000)
    ap.add_argument('--c2_n', type=int, default=100000)
    args = ap.parse_args()
    import scipy.sparse as sp
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    res = {'gpu': _gpu_info(), 'runs': []}
    for n in (int(v) for v in args.dense_n.split(',') if v):
        res['runs'] += dense_workload(n, args.h, args.reps, args.warmup, args.chunked_max_n)
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'uci_c1.npz'))
    c1 = sp.csr_matrix((np.ones(z['train_indices'].shape[0], np.float32), z['train_indices'].astype(np.int32), z['train_indptr']),
                       shape=tuple(int(v) for v in z['train_shape']))
    res['runs'].append(sparse_workload('c1', c1, 'cosine', 0.8, args.reps, args.warmup))
    c2 = make_sparse(args.c2_n, 10000, 100, 'tfidf', seed=0)
    res['runs'].append(sparse_workload('c2like', c2, 'linear kernel', 0.3, args.reps, args.warmup))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
