"""Bag-of-words user profiles (DESIGN 4.20): the profile build, recommend_sparse and impression_metrics_sparse against their
alternatives, and the bag-of-words baseline's quality on the C1 UCI articles.  One JSON line.

    python tools/bench_user_input.py [--users 100000,1000000] [--reps 5] [--imps 1000000] [--quality_users 2000] [--epochs 50]

Workload: 100 000 C2-like tf-idf articles (synth.make_sparse, F = 10 000) and synth.make_histories users (mean 20 reads before the
held-out one).  Reported, on the card named in the output:
  build[U]      : dae_csr_profiles_count + dae_csr_profiles for all U users (CUDA events, median of --reps after a warm-up), mean /
                  max profile nnz, the peak device memory above the inputs; torch.sparse.mm of the same device CSR operands (cuSPARSE
                  SpGEMM) in alternation with it, and its largest difference from the kernels' values relative to the largest value
                  over the first 10 000 users; scipy's W @ X on the host (one call, wall clock).
  recommend     : recommend_sparse(k = 10, linear kernel) at the first size as a whole (synchronised wall clock, median of --reps) and
                  its two device phases (CUDA events): the profile build and the top-k of the profiles; the chunk count at every
                  size; helpers.recommend at H = 500 on random embeddings for the same users, for context.
  impressions   : --imps impressions of 20-54 shown articles (mean 37, the README's workload) scored against the first --imps
                  profiles of the largest size: dae_csr_impression_metrics alone (CUDA events) next to dae_impression_metrics at
                  H = 500 on the same impressions, alternating.
  quality       : the DAE trained at C1 (tests/golden/uci_c1.npz, --epochs) and --quality_users make_histories users over its
                  categories with one held-out read each: hit@10 / recall@10 of recommend_sparse (binary, cosine) and of the mean
                  profile of the embeddings (recommend, cosine).  Both are reported; neither is expected to win.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402
import torch  # noqa: E402
from dae_rnn_news_recommendation_b200 import _cabi, helpers  # noqa: E402
from dae_rnn_news_recommendation_b200.engine import DeviceCSR  # noqa: E402
from dae_rnn_news_recommendation_b200.synth import make_histories, make_labels, make_sparse  # noqa: E402


def _gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi failed: %s' % e


def _events(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def _torch_csr(m, dev):
    return torch.sparse_csr_tensor(torch.from_numpy(m.indptr.astype(np.int64)), torch.from_numpy(m.indices.astype(np.int64)),
                                   torch.from_numpy(m.data.astype(np.float32)), size=m.shape).to(dev)


def build_arm(args, H, X, dev):
    w, _ = helpers._history_weights(H, X.shape[0], 'bench')
    hist, x = DeviceCSR(w, dev), DeviceCSR(X, dev)
    out = {'users': w.shape[0], 'reads': int(w.nnz)}

    def ours():
        p = helpers._profile_structure(hist, x)
        return p, helpers._profile_rows(hist, x, p, np.asarray(p.cpu()), 0, w.shape[0], False)

    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    p, P = ours()
    torch.cuda.synchronize()
    out['peak_mem_above_inputs_mb'] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    counts = np.diff(np.asarray(p.cpu()))
    out.update({'profile_nnz': int(counts.sum()), 'mean_nnz': float(counts.mean()), 'max_nnz': int(counts.max()),
                'chunks': len(helpers._profile_chunks(np.asarray(p.cpu()), helpers.SPARSE_PROFILE_CHUNK_NNZ))})
    head = min(10000, w.shape[0])
    ours_head = sp.csr_matrix((P.values[:int(p[head])].cpu().numpy(), P.indices[:int(p[head])].cpu().numpy(), p[:head + 1].cpu().numpy()),
                              shape=(head, X.shape[1]))
    del P, p
    wt, xt = _torch_csr(w, dev), _torch_csr(X, dev)

    def cusparse():
        return torch.sparse.mm(wt, xt)

    t = {'kernels': [], 'cusparse': []}
    try:
        r = cusparse()
        crow, col, val = r.crow_indices().cpu().numpy(), r.col_indices().cpu().numpy(), r.values().cpu().numpy()
        del r
        ref = sp.csr_matrix((val[:crow[head]], col[:crow[head]], crow[:head + 1]), shape=(head, X.shape[1]))
        out['cusparse_max_rel_diff'] = float(abs(ours_head - ref).max() / abs(ref).max())
        ok = True
    except RuntimeError as e:   # cuSPARSE's SpGEMM buffers may not fit at the largest size
        out['cusparse_error'] = str(e).splitlines()[0][:200]
        ok = False
        torch.cuda.empty_cache()
    _events(ours)
    for rep in range(args.reps):
        arms = ['kernels', 'cusparse'] if ok else ['kernels']
        for name in (arms if rep % 2 == 0 else arms[::-1]):
            t[name].append(_events(ours if name == 'kernels' else cusparse))
            torch.cuda.empty_cache()
    out['ms'] = {k: float(np.median(v)) for k, v in t.items() if v}
    out['ms_all'] = t
    if w.shape[0] <= args.scipy_max_users:
        t0 = time.perf_counter()
        ref = w @ X
        out['scipy_ms'] = (time.perf_counter() - t0) * 1e3
        out['scipy_nnz'] = int(ref.nnz)
    del wt, xt
    torch.cuda.empty_cache()
    return out


def recommend_arm(args, H, X, dev):
    out = {}
    w, _ = helpers._history_weights(H, X.shape[0], 'bench')
    hist, x = DeviceCSR(w, dev), DeviceCSR(X, dev)
    lists = helpers._DeviceLists(hist.indptr, hist.indices, hist.nnz)
    state = {}

    def build():
        p = helpers._profile_structure(hist, x)
        state['q'] = helpers._profile_rows(hist, x, p, np.asarray(p.cpu()), 0, w.shape[0], False)

    def topk():
        helpers._csr_similarity_topk(state['q'], x, 10, lists=lists)

    whole = lambda: helpers.recommend_sparse(H, X, k=10, metric='linear kernel', to_host=False)   # noqa: E731
    emb = torch.randn(X.shape[0], 500, device=dev)
    dense = lambda: helpers.recommend(H, emb, k=10, metric='cosine', to_host=False)   # noqa: E731
    build(), topk(), whole(), dense()
    t = {'recommend_sparse': [], 'profiles': [], 'topk': [], 'recommend_dense_h500': []}
    for rep in range(args.reps):
        names = list(t)
        for name in names[rep % 4:] + names[:rep % 4]:
            fn = {'recommend_sparse': lambda: _wall(whole), 'profiles': lambda: _events(build), 'topk': lambda: _events(topk),
                  'recommend_dense_h500': lambda: _wall(dense)}[name]
            t[name].append(fn())
    out['ms'] = {k: float(np.median(v)) for k, v in t.items()}
    out['ms_all'] = t
    return out


def impressions_arm(args, Q, X, dev, rng):
    n_imp, N = args.imps, X.shape[0]
    lens = rng.integers(20, 55, n_imp)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    row = np.repeat(np.arange(n_imp), lens)
    pos = np.arange(int(indptr[-1])) - np.repeat(indptr[:-1], lens)
    items = ((rng.integers(0, N, n_imp)[row] + pos * (2 * rng.integers(1, 1000, n_imp)[row] + 1)) % N).astype(np.int32)
    clicked = (rng.random(items.size) < 0.1).astype(np.uint8)
    clicked[indptr[:-1]] = 1
    imp = {'indptr': indptr, 'items': items, 'clicked': clicked}
    x = DeviceCSR(X, dev)
    q = DeviceCSR.from_tensors(Q.indptr[:n_imp + 1], Q.indices[:int(Q.indptr[n_imp])], Q.values[:int(Q.indptr[n_imp])],
                               (n_imp, X.shape[1]))
    d = {k: torch.from_numpy(v).to(dev) for k, v in imp.items()}
    H = 500
    qd = torch.randn(n_imp, H, device=dev) / np.sqrt(H)
    emb = torch.randn(N, H, device=dev) / np.sqrt(H)
    scores = torch.empty(items.size, dtype=torch.float32, device=dev)
    met = torch.empty(n_imp, 4, dtype=torch.float64, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def sparse_k():
        _cabi.call('dae_csr_impression_metrics', q.indptr.data_ptr(), q.indices.data_ptr(), q.values.data_ptr(), x.indptr.data_ptr(),
                   x.indices.data_ptr(), x.values.data_ptr(), N, X.shape[1], 0, d['indptr'].data_ptr(), d['items'].data_ptr(),
                   d['clicked'].data_ptr(), n_imp, scores.data_ptr(), met.data_ptr(), st)

    def dense_k():
        _cabi.call('dae_impression_metrics', qd.data_ptr(), H, emb.data_ptr(), H, H, 0, d['indptr'].data_ptr(), d['items'].data_ptr(),
                   d['clicked'].data_ptr(), n_imp, scores.data_ptr(), met.data_ptr(), st)

    sparse_k(), dense_k()
    t = {'csr_impression_metrics': [], 'impression_metrics_h500': []}
    for rep in range(args.reps):
        for name in (list(t) if rep % 2 == 0 else list(t)[::-1]):
            t[name].append(_events(sparse_k if name == 'csr_impression_metrics' else dense_k))
    q_nnz = np.diff(q.indptr.cpu().numpy())
    return {'impressions': n_imp, 'shown': int(items.size), 'query_mean_nnz': float(q_nnz.mean()),
            'ms': {k: float(np.median(v)) for k, v in t.items()}, 'ms_all': t}


def quality_arm(args):
    from helpers import load_uci_c1
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder, utils
    os.chdir(os.environ.get('TMPDIR', '/tmp'))
    d = load_uci_c1()
    X, lab = d['train'], d['train_label_category_publish_name']
    m = DenoisingAutoencoder(model_name='bow_q', main_dir='bow_q', compress_factor=20, enc_act_func='sigmoid', dec_act_func='sigmoid',
                             loss_func='cross_entropy', corr_type='masking', corr_frac=0.3, opt='gradient_descent', learning_rate=0.1,
                             num_epochs=args.epochs, batch_size=0.1, alpha=1, triplet_strategy='none', seed=0, verbose=False)
    m.fit(X, None, lab)
    enc = m.transform(utils.decay_noise(X, 0.3), name='bow_q', save=False)
    H, T = make_histories(args.quality_users, lab, seed=1)
    out = {'users': args.quality_users, 'epochs': args.epochs}
    for name, idx in (('bag_of_words', helpers.recommend_sparse(H, X, k=10, metric='cosine')[0]),
                      ('dae_mean_profile', helpers.recommend(H, enc, k=10, metric='cosine')[0])):
        r = helpers.recommendation_recall(idx, T)
        out[name] = {'hit@10': r['hit_rate'], 'recall@10': r['recall']}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--users', default='100000,1000000')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--imps', type=int, default=1000000)
    ap.add_argument('--scipy_max_users', type=int, default=1000000)
    ap.add_argument('--quality_users', type=int, default=2000)
    ap.add_argument('--epochs', type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_user_input: no GPU')
    dev = torch.device('cuda:0')
    res = {'gpu': _gpu_info(), 'articles': 100000, 'features': 10000, 'build': {}}
    X = make_sparse(100000, 10000, kind='tfidf', seed=0)
    labels = make_labels(100000)
    sizes = [int(u) for u in args.users.split(',')]
    for U in sizes:
        H, _ = make_histories(U, labels, seed=2)
        res['build'][str(U)] = build_arm(args, H, X, dev)
        if U == sizes[0]:
            res['recommend'] = recommend_arm(args, H, X, dev)
        if U == sizes[-1]:
            w, _ = helpers._history_weights(H, X.shape[0], 'bench')
            hist, x = DeviceCSR(w, dev), DeviceCSR(X, dev)
            p = helpers._profile_structure(hist, x)
            n_q = min(args.imps, U)
            Q = helpers._profile_rows(hist, x, p, np.asarray(p.cpu()), 0, n_q, False)
            del hist, x
            args.imps = n_q
            res['impressions'] = impressions_arm(args, Q, X, dev, np.random.default_rng(3))
            del Q
            torch.cuda.empty_cache()
    res['quality'] = quality_arm(args)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
