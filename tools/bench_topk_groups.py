"""What one-per-group top-k (top_k_similar(groups=...), recommend(groups=...)) costs, and why a host filter is no substitute.
One JSON line.

    python tools/bench_topk_groups.py [--n 100000] [--big 1000000] [--h 500] [--k 10] [--reps 3] [--warmup 1]

Articles: --n rows in stories of ~21 near-duplicates (row = story centre + small noise; stories drawn around 50 topic centres),
device-resident, cosine.  Groups: helpers.similar_pairs(emb, --tau) + duplicate_groups, as main_autoencoder.py --top_k_dedup
does.  Dense paths, from the bf16 hi / lo operands on the device to (index, score) on the device:
  plain          dae_similarity_topk_bf16x3, k
  grouped        dae_similarity_topk_groups_bf16x3, k
  filter32       the plain call at k = 32, copied to the host, and a NumPy filter keeping each group's first entry, then k of them
                 (rows_short: how many rows come back with fewer than k entries -- the reason the selection is in the kernel)
at --n rows (self search) and with --n queries against --big corpus rows (the corpus is the same construction at --big rows).
Sparse: dae_csr_similarity_topk vs _groups on --n C2-like tf-idf rows (synth.make_sparse, 10 000 columns), self search, groups
of ~21 random rows.  recommend: the device half at 10^5 and 10^6 users (synth.make_histories over the --n articles): top-k with
the read lists vs the read-group lists (built on the device by helpers._read_group_lists, timed separately) and groups.
Paths run in rotating order after warm-up; times are CUDA-event medians (host clock around a synchronise for filter32).
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
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


def _time(paths, reps, warmup, host=()):
    names = list(paths)
    out = {n: paths[n]() for n in names}
    for _ in range(warmup - 1):
        for n in names:
            paths[n]()
    torch.cuda.synchronize()
    times = {n: [] for n in names}
    for rep in range(reps):
        for n in names[rep % len(names):] + names[:rep % len(names)]:
            if n in host:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                paths[n]()
                torch.cuda.synchronize()
                times[n].append((time.perf_counter() - t0) * 1e3)
                continue
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            paths[n]()
            b.record()
            torch.cuda.synchronize()
            times[n].append(a.elapsed_time(b))
    return {n: {'ms_median': float(np.median(times[n])), 'ms_all': [round(t, 3) for t in times[n]]} for n in names}, out


def _articles(n, h, seed):
    rng = np.random.default_rng(seed)
    topics = rng.standard_normal((50, h))
    n_st = max(1, n // 21)
    story = topics[rng.integers(0, 50, n_st)] + 0.8 * rng.standard_normal((n_st, h))
    lab = rng.integers(0, n_st, n)
    x = torch.from_numpy(story[lab].astype(np.float32)).cuda()
    x += 0.12 * torch.randn(n, h, device='cuda', generator=torch.Generator('cuda').manual_seed(seed))
    return x


def _groups(x, tau):
    i, j, _ = helpers.similar_pairs(x, tau, to_host=True)
    return helpers.duplicate_groups(i, j, x.shape[0])


def _host_filter(idx32, val32, g, k):
    """Keep each group's first entry of the k = 32 lists, then the first k: (index, score, rows with fewer than k)."""
    idx = idx32.cpu().numpy()
    val = val32.cpu().numpy()
    G = np.where(idx >= 0, g[np.maximum(idx, 0)], -1)
    keep = idx >= 0
    for j in range(1, idx.shape[1]):
        keep[:, j] &= ~(G[:, :j] == G[:, j:j + 1]).any(1)
    rank = np.cumsum(keep, 1) - 1
    sel = keep & (rank < k)
    out_i = np.full((idx.shape[0], k), -1, np.int32)
    out_v = np.full((idx.shape[0], k), -np.inf, np.float32)
    r, c = np.nonzero(sel)
    out_i[r, rank[r, c]] = idx[r, c]
    out_v[r, rank[r, c]] = val[r, c]
    return out_i, out_v, int((sel.sum(1) < k).sum())


def dense_part(args, q_x, c_x, g, self_mode):
    nq, nc, h, k = q_x.shape[0], c_x.shape[0], q_x.shape[1], args.k
    q = helpers._normalised_operands(q_x, 2)[:2]
    c = q if self_mode else helpers._normalised_operands(c_x, 2)[:2]
    g_dev = torch.from_numpy(g.astype(np.int32)).cuda()
    filt = {}

    def filter32():
        i, v = helpers._similarity_topk(q, c, nq, nc, h, 32, exclude=self_mode)
        filt['res'] = _host_filter(i, v, g, k)
        return filt['res']
    paths = {'plain': lambda: helpers._similarity_topk(q, c, nq, nc, h, k, exclude=self_mode),
             'grouped': lambda: helpers._similarity_topk(q, c, nq, nc, h, k, exclude=self_mode, groups=g_dev),
             'filter32': filter32}
    res, out = _time(paths, args.reps, args.warmup, host=('filter32',))
    gi, gv = (t.cpu().numpy() for t in out['grouped'])
    fi, fv, short = filt['res']
    pi = out['plain'][0].cpu().numpy()
    gp = g[np.maximum(pi, 0)]
    dup_rows = int(sum(np.unique(r).size < k for r in gp))
    full = (fi >= 0).all(1)
    return {'queries': nq, 'corpus': nc, 'self': self_mode, 'groups': int(np.unique(g).size), 'paths': res,
            'grouped_over_plain': res['grouped']['ms_median'] / res['plain']['ms_median'] - 1.0,
            'plain_rows_with_a_repeated_group': dup_rows,
            'filter32_rows_short': short,
            'filter32_equals_grouped_on_full_rows': bool(np.array_equal(fi[full], gi[full]) and np.array_equal(fv[full], gv[full]))}


def sparse_part(args):
    x = make_sparse(args.n, 10000, 100, 'tfidf', seed=0)
    d = DeviceCSR(helpers._csr_operand(x, 'linear kernel'), torch.device('cuda:0'))
    g = np.random.default_rng(1).integers(0, max(1, args.n // 21), args.n)
    g_dev = torch.from_numpy(g.astype(np.int32)).cuda()
    paths = {'sparse_plain': lambda: helpers._csr_similarity_topk(d, d, args.k, exclude=True),
             'sparse_grouped': lambda: helpers._csr_similarity_topk(d, d, args.k, exclude=True, groups=g_dev)}
    res, _ = _time(paths, args.reps, args.warmup)
    return {'rows': args.n, 'nnz': int(d.nnz), 'paths': res,
            'grouped_over_plain': res['sparse_grouped']['ms_median'] / res['sparse_plain']['ms_median'] - 1.0}


def recommend_part(args, emb, g, n_users):
    n, k = emb.shape[0], args.k
    h, _ = make_histories(n_users, g % 20, mean_len=20, seed=2, max_len=2000, holdout=False)
    w, _ = helpers._history_weights(h, n, 'bench')
    hist = DeviceCSR(w, emb.device)
    prof = helpers._profiles(hist, emb)
    g_dev = torch.from_numpy(g.astype(np.int32)).cuda()
    lists = helpers._DeviceLists(hist.indptr, hist.indices, hist.nnz)
    ptr, ind = helpers._read_group_lists(hist.indptr, hist.indices, g_dev, g_dev)
    glists = helpers._DeviceLists(ptr, ind, ind.numel())
    paths = {'topk_read_lists': lambda: helpers._recommend_topk(prof, emb, k, 'cosine', lists),
             'topk_group_lists_groups': lambda: helpers._recommend_topk(prof, emb, k, 'cosine', glists, groups=g_dev),
             'build_group_lists': lambda: helpers._read_group_lists(hist.indptr, hist.indices, g_dev, g_dev)}
    res, _ = _time(paths, args.reps, args.warmup)
    return {'users': n_users, 'read_entries': int(hist.nnz), 'group_list_entries': int(glists.nnz), 'paths': res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=100000)
    ap.add_argument('--big', type=int, default=1000000)
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--k', type=int, default=10)
    ap.add_argument('--tau', type=float, default=0.9)
    ap.add_argument('--users', default='100000,1000000')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_topk_groups: no CUDA device')
    res = {'N': args.n, 'big': args.big, 'H': args.h, 'k': args.k, 'tau': args.tau, 'reps': args.reps, 'gpu': _gpu_info(),
           'device_name': torch.cuda.get_device_name(0)}
    x = _articles(args.n, args.h, 0)
    g = _groups(x, args.tau)
    res['dense'] = [dense_part(args, x, x, g, True)]
    res['recommend'] = [recommend_part(args, x, g, int(u)) for u in args.users.split(',')]
    if args.big:
        xb = _articles(args.big, args.h, 0)
        gb = _groups(xb, args.tau)
        res['dense'].append(dense_part(args, xb[:args.n], xb, gb, False))
        del xb
    res['sparse'] = sparse_part(args)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
