"""Recommending unread articles to users (helpers.recommend) and what its exclusion lists cost.  One JSON line.

    python tools/bench_recommend.py [--n 100000] [--h 500] [--users 100000,1000000] [--k 10] [--reps 5] [--warmup 2]

Clustered articles (device-resident, as tools/bench_topk.py) and synth.make_histories users (mean length --mean_len, capped at
2 000).  Paths, from the device embeddings and the device history CSR (host preparation excluded) to (index, score) on the device:
  a  recommend's device half: profiles (dae_encode_csr_fwd) + the top-k with the histories as exclusion lists; also split into
     a_profiles and a_topk_lists (the top-k alone, on the same profiles)
  b  the same top-k on the same profiles without exclusion lists (dae_similarity_topk_bf16x3): b vs a_topk_lists is the lists' cost
  c  (first user count only) chunked GEMM into a chunk x N fp32 block, -inf at the history entries, torch.topk
Sparse: dae_csr_similarity_topk on synth.make_sparse tf-idf rows (self search), without and with lists of ~--sparse_list rows.
Paths run in rotating order after warm-up; times are CUDA-event medians around one call; peaks are above the inputs.
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
from dae_rnn_news_recommendation_b200.engine import DeviceCSR  # noqa: E402
from dae_rnn_news_recommendation_b200.synth import make_histories, make_sparse  # noqa: E402


def _gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi failed: %s' % e


def _run(paths, reps, warmup):
    names = list(paths)
    mem, out = {}, {}
    for name in names:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out[name] = paths[name]()
        torch.cuda.synchronize()
        mem[name] = torch.cuda.max_memory_allocated() - base
        for _ in range(warmup - 1):
            paths[name]()
    torch.cuda.synchronize()
    times = {n: [] for n in names}
    for rep in range(reps):
        for name in names[rep % len(names):] + names[:rep % len(names)]:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            paths[name]()
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b))
    res = {n: {'ms_median': float(np.median(times[n])), 'ms_min': float(min(times[n])), 'ms_all': [round(t, 3) for t in times[n]],
               'peak_above_inputs_bytes': int(mem[n])} for n in names}
    return res, out


def dense_part(args, emb, labels, n_users, with_c):
    N, H, K = emb.shape[0], emb.shape[1], args.k
    h, _ = make_histories(n_users, labels, mean_len=args.mean_len, seed=1, max_len=2000, holdout=False)
    w, _ = helpers._history_weights(h, N, 'bench')
    hist = DeviceCSR(w, emb.device)
    lists = helpers._DeviceLists(hist.indptr, hist.indices, hist.nnz)
    prof = helpers._profiles(hist, emb)
    paths = {'a_recommend_device': lambda: helpers._recommend_topk(helpers._profiles(hist, emb), emb, K, 'cosine', lists),
             'a_profiles': lambda: helpers._profiles(hist, emb),
             'a_topk_lists': lambda: helpers._recommend_topk(prof, emb, K, 'cosine', lists),
             'b_topk_no_lists': lambda: helpers._recommend_topk(prof, emb, K, 'cosine', None)}
    if with_c:
        rows = torch.repeat_interleave(torch.arange(n_users, device=emb.device), hist.indptr[1:] - hist.indptr[:-1])
        indptr_h = w.indptr

        def path_c():
            q = helpers._normalised_operands(prof, 2)[:2]
            c = helpers._normalised_operands(emb, 2)[:2]
            idx = torch.empty(n_users, K, dtype=torch.int64, device=emb.device)
            val = torch.empty(n_users, K, dtype=torch.float32, device=emb.device)
            buf = torch.empty(min(args.chunk, n_users), N, dtype=torch.float32, device=emb.device)
            for r0 in range(0, n_users, args.chunk):
                r1 = min(n_users, r0 + args.chunk)
                helpers._gemm_nt((q[0][r0:r1], q[1][r0:r1]), c, r1 - r0, N, H, buf)
                b = buf[:r1 - r0]
                p0, p1 = int(indptr_h[r0]), int(indptr_h[r1])
                b[rows[p0:p1] - r0, hist.indices[p0:p1].long()] = float('-inf')
                torch.topk(b, K, dim=1, out=(val[r0:r1], idx[r0:r1]))
            return idx, val
        paths['c_chunked_gemm_mask_torch_topk'] = path_c
    res, out = _run(paths, args.reps, args.warmup)
    info = {'users': n_users, 'history_entries': int(hist.nnz), 'mean_len': hist.nnz / n_users,
            'max_len': int(np.diff(w.indptr).max()), 'inputs_bytes': int(emb.numel() * 4 + hist.h2d_bytes), 'paths': res}
    a, b = res['a_topk_lists']['ms_median'], res['b_topk_no_lists']['ms_median']
    info['lists_cost_over_topk'] = a / b - 1.0
    ia, va = (t.cpu().numpy() for t in out['a_topk_lists'])
    sample = np.random.default_rng(0).choice(n_users, min(n_users, 500), replace=False)
    hs = (h[sample] > 0).toarray()
    info['read_articles_returned_in_500_sampled_users'] = int(np.take_along_axis(hs, np.maximum(ia[sample], 0), 1)[ia[sample] >= 0].sum())
    if with_c:
        ic, vc = (t.cpu().numpy() for t in out['c_chunked_gemm_mask_torch_topk'])
        info['a_vs_c_same_index_sets'] = float((np.sort(ia, 1) == np.sort(ic, 1)).all(1).mean())
        info['a_vs_c_max_abs_score_diff'] = float(np.abs(va - vc).max())
    return info


def sparse_part(args):
    x = make_sparse(args.sparse_n, args.sparse_f, 100, 'tfidf', seed=0)
    op = helpers._csr_operand(x, 'linear kernel')
    dev = torch.device('cuda:0')
    d = DeviceCSR(op, dev)
    n = op.shape[0]
    rng = np.random.default_rng(2)
    cnt = rng.poisson(args.sparse_list, n)
    ex = sp.csr_matrix((np.ones(cnt.sum(), np.float32), (np.repeat(np.arange(n), cnt), rng.integers(0, n, cnt.sum()))), shape=(n, n))
    indptr, indices, _ = helpers._stored_positions(ex, (n, n), 'exclude', 'bench')
    lists = helpers._DeviceLists.from_host(indptr, indices, torch.device('cuda:0'))
    paths = {'sparse_topk_no_lists': lambda: helpers._csr_similarity_topk(d, d, args.k, exclude=True),
             'sparse_topk_lists': lambda: helpers._csr_similarity_topk(d, d, args.k, exclude=True, lists=lists)}
    res, _ = _run(paths, args.reps, args.warmup)
    return {'rows': n, 'features': op.shape[1], 'nnz': int(op.nnz), 'list_entries': int(lists.nnz), 'paths': res,
            'lists_cost': res['sparse_topk_lists']['ms_median'] / res['sparse_topk_no_lists']['ms_median'] - 1.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=100000)
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--users', default='100000,1000000')
    ap.add_argument('--mean_len', type=float, default=20.0)
    ap.add_argument('--k', type=int, default=10)
    ap.add_argument('--chunk', type=int, default=8192)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--sparse_n', type=int, default=100000)
    ap.add_argument('--sparse_f', type=int, default=10000)
    ap.add_argument('--sparse_list', type=float, default=20.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_recommend: no CUDA device')
    rng = np.random.RandomState(0)
    labels = rng.randint(0, 4, args.n)
    emb = torch.from_numpy((rng.randn(4, args.h)[labels] * 0.15 + rng.randn(args.n, args.h)).astype(np.float32)).cuda()
    res = {'N': args.n, 'H': args.h, 'k': args.k, 'reps': args.reps, 'gpu': _gpu_info(), 'device_name': torch.cuda.get_device_name(0)}
    res['dense'] = [dense_part(args, emb, labels, int(u), i == 0) for i, u in enumerate(args.users.split(','))]
    res['sparse'] = sparse_part(args)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
