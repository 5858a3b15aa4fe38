"""Related-vs-unrelated AUROC without the similarity matrix (helpers.similarity_auroc) against the sort path
(pairwise_similarity + visualize_pairwise_similarity), with the dense top-k as the main-loop reference point.  One JSON line.

    python tools/bench_auroc.py [--n 1000000] [--h 500] [--bins 2097152] [--reps 3]

Workloads:
  dense   clustered embeddings (4 labels, generated like tools/bench_topk.py's) at N = 8 000 and 100 000 (and --n), cosine:
          the pair-histogram kernel alone (_pair_histograms, device buffers in and out) and the whole similarity_auroc call (with
          the host evaluation of the histograms); top_k_similar(k = 10) at the same N -- the histogram kernel computes half of
          top-k's tiles, so about half its time means the histogram adds hide behind the tensor-core main loop; the sort path at
          8 000 and 20 000 rows (it forms the N x N matrix).
  sparse  the C1 UCI articles (8 000 x 10 000 binary, cosine, category labels) and a C2-like set (100 000 x 10 000 tf-idf, linear
          kernel, 4 labels): the sparse pair-histogram kernel and the whole call; the sort path at C1.
Times are CUDA-event medians of --reps calls after one warm-up call; memory is the peak above the inputs during one call.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402
import torch  # noqa: E402
from dae_rnn_news_recommendation_b200 import helpers  # noqa: E402


def _gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi failed: %s' % e


def _measure(fn, reps):
    """(median ms, all ms, peak bytes above the allocation before the first call, result of the first call)"""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), [round(t, 3) for t in times], int(peak), out


def _summary(res):
    return {'auroc': res['auroc'], 'auroc_error_bound': res['auroc_error_bound'], 'bin_width': res['bin_width'],
            'related_median': res['related'].get('median'), 'unrelated_median': res['unrelated'].get('median')}


def _case(data, labels, metric, bins, reps, sort_data=None):
    r = {}
    ms, all_ms, peak, _ = _measure(lambda: helpers._pair_histograms(data, labels, metric, bins), reps)
    r['kernel'] = {'ms_median': ms, 'ms_all': all_ms, 'peak_above_inputs_bytes': peak}
    ms, all_ms, peak, out = _measure(lambda: helpers.similarity_auroc(data, labels, metric=metric, bins=bins), reps)
    r['similarity_auroc'] = {'ms_median': ms, 'ms_all': all_ms, 'peak_above_inputs_bytes': peak, **_summary(out)}
    if sort_data is not None:   # pairwise_similarity takes host arrays (dense) or scipy sparse
        def sort():
            return helpers.visualize_pairwise_similarity(labels, helpers.pairwise_similarity(sort_data, metric=metric, to_host=False))
        ms, all_ms, peak, out = _measure(sort, reps)
        r['sort_path'] = {'ms_median': ms, 'ms_all': all_ms, 'peak_above_inputs_bytes': peak, 'auroc': out['auroc'],
                          'auroc_grid_minus_sort': r['similarity_auroc']['auroc'] - out['auroc']}
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=0, help='one more dense size (e.g. 1000000)')
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--bins', type=int, default=1 << 21)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_auroc: no CUDA device')
    res = {'bins': args.bins, 'reps': args.reps, 'H': args.h, 'dense': {}, 'sparse': {}}
    dev = torch.device('cuda:0')
    sizes = [8000, 20000, 100000] + ([args.n] if args.n else [])
    for n in sizes:
        rng = np.random.RandomState(0)
        labels = rng.randint(0, 4, n)
        emb = (rng.randn(4, args.h)[labels] * 0.15 + rng.randn(n, args.h)).astype(np.float32)
        x = torch.from_numpy(emb).to(dev)
        if n == 20000:   # the sort path's largest default size: only the comparison
            r = _case(x, labels, 'cosine', args.bins, args.reps, emb)
        else:
            r = _case(x, labels, 'cosine', args.bins, args.reps, emb if n == 8000 else None)
            ms, all_ms, peak, _ = _measure(lambda: helpers.top_k_similar(x, k=10, to_host=False), args.reps)
            r['top_k_similar_k10'] = {'ms_median': ms, 'ms_all': all_ms, 'peak_above_inputs_bytes': peak}
            r['kernel_over_topk'] = r['kernel']['ms_median'] / ms
        res['dense'][str(n)] = r
        del x, emb
    from dae_rnn_news_recommendation_b200.synth import make_labels, make_sparse
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'uci_c1.npz'))
    c1 = sp.csr_matrix((np.ones(z['train_indices'].shape[0], np.float32), z['train_indices'], z['train_indptr']),
                       shape=tuple(int(v) for v in z['train_shape']))
    res['sparse']['c1_uci_binary_cosine'] = _case(c1, z['train_label_category_publish_name'], 'cosine', args.bins, args.reps, c1)
    c2 = make_sparse(100000, 10000, 100, 'tfidf', seed=0)
    res['sparse']['c2_like_tfidf_linear'] = _case(c2, make_labels(100000, 4), 'linear kernel', args.bins, args.reps)
    res['gpu'] = _gpu_info()
    res['device_name'] = torch.cuda.get_device_name(0)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
