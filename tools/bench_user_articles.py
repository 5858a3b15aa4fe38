"""The article encoder fine-tuned through the user encoders' losses (user_model.ArticleEncoder, DESIGN 4.19): training speed frozen
against joint, the per-batch breakdown of a joint batch, its memory, the encode regimes at the measured touched count T, and the
cold-start learning check.  One JSON line.

    python tools/bench_user_articles.py [--n 100000] [--f 10000] [--h 500] [--users 32768] [--batch_users 1024,4096] [--rounds 2]
                                        [--learning_lrs 1e-4,1e-3,1e-2] [--skip_speed]

Reported:
  train[B]: positions/s of one epoch of --users make_sequences users over --n tf-idf articles (synth.make_sparse, C2-like: 100
            words per article), GRU at H = --h, batch_users B, frozen (the encoder's vectors as embeddings) and joint, after a
            warm-up epoch of each, over --rounds alternating rounds;
  phases[B]: per joint batch, the mean touched count T and the mean time of each phase (CUDA events between the phase marks);
  memory[B]: peak device bytes of a joint epoch above what the inputs and the model hold;
  regimes[B]: at the measured T, dae_encode_csr_fwd_groups with 1 and 4 groups, and dae_encode_csr_bwd against
            dae_encode_csr_bwd_gather (CUDA events, 20 calls each);
  learning: learning_workload (click preference follows word groups; 20 % of the articles held out of training, the test
            impressions show only those): test-impression AUC of a GRU on the frozen encoder and jointly trained at each
            --learning_lrs, every one scored with art.vectors(X_held_out).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402
import torch  # noqa: E402
from bench_user_model import _gpu_info  # noqa: E402
from dae_rnn_news_recommendation_b200 import _cabi, helpers  # noqa: E402
from dae_rnn_news_recommendation_b200.synth import make_labels, make_sequences, make_sparse  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import ArticleEncoder, Packed, UserGRU  # noqa: E402

PHASES = ('start', 'compact', 'encode', 'input_projection', 'forward_recurrence', 'loss', 'backward_recurrence', 'weight_gradients',
          'input_gradient', 'article_backward', 'optimizer', 'article_step')


def _params(F, H, seed):
    rng = np.random.default_rng(seed)
    k = np.sqrt(6.0 / (F + H))
    return {'enc_w': rng.uniform(-k, k, (F, H)).astype(np.float32), 'enc_b': np.zeros(H, np.float32)}


def _epoch(m, indptr, items, emb, art, epoch, packs):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for bi, pk in enumerate(packs):
        m._forward_backward(pk, emb, epoch, bi, None, art)
        m._optimizer_step()
        if art is not None:
            art.step()
            m._mark('article_step')
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _events_ms(fn, reps=20):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def regimes(art, T, seed=0):
    """ms per call at T random distinct rows: the forward with 1 and 4 groups, the plain and the gathered backward."""
    d, F, H = art.device, art.F, art.dim
    rows = torch.from_numpy(np.sort(np.random.default_rng(seed).choice(art.n, T, replace=False)).astype(np.int32)).to(d)
    E = torch.empty(T, H, device=d)
    cc = torch.empty(F, dtype=torch.int32, device=d)
    out = {}
    for g in (1, 4):
        out['fwd_groups%d_ms' % g] = _events_ms(lambda: _cabi.call(
            'dae_encode_csr_fwd_groups', art.csr.indptr.data_ptr(), art.csr.indices.data_ptr(), art.csr.values.data_ptr(),
            rows.data_ptr(), T, F, H, art.in_scale, art.W.data_ptr(), art.bh.data_ptr(), _cabi.act_code(art.enc_act_func),
            E.data_ptr(), H, cc.data_ptr(), None, None, 0, g, torch.cuda.current_stream().cuda_stream))
    dE = torch.randn(T, H, device=d) * 1e-3
    dE0 = dE.clone()

    def plain():
        dE.copy_(dE0)
        _cabi.call('dae_encode_csr_bwd', art.csr.indptr.data_ptr(), art.csr.indices.data_ptr(), art.csr.values.data_ptr(),
                   rows.data_ptr(), T, F, H, art.in_scale, E.data_ptr(), art.bh.data_ptr(), _cabi.act_code(art.enc_act_func),
                   dE.data_ptr(), None, H, art.grad.data_ptr(), art.grad[F * H:].data_ptr(), 0,
                   torch.cuda.current_stream().cuda_stream)

    def gathered():
        dE.copy_(dE0)
        art.backward(rows, T, E, dE, cc)
    copy_ms = _events_ms(lambda: dE.copy_(dE0))
    out['bwd_plain_ms'] = _events_ms(plain) - copy_ms
    out['bwd_gather_ms'] = _events_ms(gathered) - copy_ms   # includes zeroing dW, as in training
    return out


def speed(args):
    d = torch.device('cuda:0')
    X = make_sparse(args.n, args.f, mean_nnz=100, kind='tfidf', seed=1)
    labels = make_labels(args.n, seed=2)
    indptr, items, _ = make_sequences(args.users, labels, mean_len=20, seed=3, holdout=False)
    out = {}
    for B in args.batch_users:
        art = ArticleEncoder(X, _params(args.f, args.h, 0), enc_act_func='sigmoid', in_scale=0.7, device=d)
        emb = art.vectors(to_host=False)
        ms = {'frozen': UserGRU(args.h, batch_users=B, seed=0), 'joint': UserGRU(args.h, batch_users=B, seed=0)}
        if args.deterministic:   # DESIGN 4.21: both paths in the deterministic mode too, timed in the same alternation
            ms.update(frozen_det=UserGRU(args.h, batch_users=B, seed=0, deterministic=True),
                      joint_det=UserGRU(args.h, batch_users=B, seed=0, deterministic=True))
        packs = [Packed(indptr, items, u, 50) for u in ms['frozen'].batches(indptr, 0)]
        P = sum(p.P for p in packs)
        joint = lambda name: name.startswith('joint')   # noqa: E731
        for name, m in ms.items():   # warm-up
            _epoch(m, indptr, items, None if joint(name) else emb, art if joint(name) else None, 0, packs)
        rates = {name: [] for name in ms}
        for _ in range(args.rounds):
            for name, m in ms.items():
                s = _epoch(m, indptr, items, None if joint(name) else emb, art if joint(name) else None, 0, packs)
                rates[name].append(P / s)
        out[str(B)] = {'positions': P, 'batches': len(packs), 'frozen_positions_per_s': rates['frozen'],
                       'joint_positions_per_s': rates['joint']}
        if args.deterministic:
            out[str(B)].update(frozen_det_positions_per_s=rates['frozen_det'], joint_det_positions_per_s=rates['joint_det'])
        for name in ('joint', 'joint_det') if args.deterministic else ('joint',):
            out[str(B)].update(_joint_phases(ms[name], art, packs, '' if name == 'joint' else '_det'))
    return out


def _joint_phases(m, art, packs, sfx):
    """One epoch of the joint model with phase events: the per-batch phase times, the touched-article counts and the peak memory."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m.phase_events, Ts = [], []
    for bi, pk in enumerate(packs):
        m._forward_backward(pk, None, 0, bi, None, art)
        Ts.append(int(m.article_batch['rows'].numel()))
        m._optimizer_step()
        art.step()
        m._mark('article_step')
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ph = {}
    ev = m.phase_events
    for (n0, e0), (n1, e1) in zip(ev[:-1], ev[1:]):
        if n1 != 'start':
            ph[n1] = ph.get(n1, 0.0) + e0.elapsed_time(e1)
    m.phase_events = None
    r = {'T_mean': float(np.mean(Ts)), 'T_max': int(np.max(Ts)), 'phase_ms_per_batch': {k: v / len(packs) for k, v in ph.items()},
         'peak_bytes_above_inputs': int(peak)}
    if sfx:
        r['article_backward_workspace_bytes'] = int(art.det_workspace_bytes)
    else:
        r['regimes_at_T_mean'] = regimes(art, int(np.mean(Ts)))
    return {k + sfx: v for k, v in r.items()}


# ---- the cold-start learning check ---------------------------------------------------------------------------------------
def learning_workload(n=3000, F=2000, users=1500, seq_len=20, shown=5, seed=0):
    """Articles of two topics: each carries 6 of its topic's 100 words among ~40 Zipf background words (tf-idf-like values), so a
    random encoder spreads the topic over many directions.  Users prefer one topic; they read their topic's articles, and each
    impression shows one article of their topic (the click) and shown - 1 of the other.  The last 20 % of the articles are held
    out of every sequence and training impression; the test impressions, one per user after the last read, show only those.
    Returns a dict of X_train, X_all (held-out rows from n_train on), the sequences, train / test impressions and W, bh."""
    rng = np.random.default_rng(seed)
    topic = rng.integers(0, 2, n)
    bg = make_sparse(n, F - 200, mean_nnz=40, kind='tfidf', seed=seed + 1)
    rows, cols, vals = [], [], []
    for a in range(n):
        w = rng.choice(100, 6, replace=False) + 100 * topic[a]
        rows += [a] * 6
        cols += list(w)
        vals += list(rng.uniform(0.1, 0.3, 6))
    tw = sp.csr_matrix((np.array(vals, np.float32), (rows, cols)), shape=(n, 200))
    X = sp.hstack([tw, bg]).tocsr().astype(np.float32)
    n_tr = int(0.8 * n)
    tr = [np.flatnonzero(topic[:n_tr] == c) for c in (0, 1)]
    ho = [np.flatnonzero(topic[n_tr:] == c) + n_tr for c in (0, 1)]
    pref = rng.integers(0, 2, users)
    items = np.concatenate([rng.choice(tr[pref[u]], seq_len) for u in range(users)]).astype(np.int32)
    indptr = np.arange(users + 1, dtype=np.int64) * seq_len

    def imps(pool, times):
        it, ck, us, tm = [], [], [], []
        for u in range(users):
            for t in times:
                it.append(np.concatenate([rng.choice(pool[pref[u]], 1), rng.choice(pool[1 - pref[u]], shown - 1, replace=False)]))
                ck.append(np.r_[1, np.zeros(shown - 1)])
                us.append(u)
                tm.append(t)
        return {'user': np.array(us, np.int64), 'time': np.array(tm, np.int64), 'indptr': np.arange(len(it) + 1, dtype=np.int64) * shown,
                'items': np.concatenate(it).astype(np.int32), 'clicked': np.concatenate(ck).astype(np.uint8)}
    p = _params(F, 32, seed + 7)
    return {'X_train': X[:n_tr], 'X_all': X, 'seqs': (indptr, items), 'train': imps(tr, range(2, seq_len + 1, 3)),
            'test': imps(ho, [seq_len]), 'params': p, 'H': 32}


def learning_auc(data, art_lr=None, cell=UserGRU, epochs=12, seed=0):
    """Test-impression AUC of a user encoder trained on the frozen encoder (art_lr None) or jointly with it (art_lr), scored with
    art.vectors(X_all), whose held-out rows only the test impressions show."""
    art = ArticleEncoder(data['X_train'], data['params'], enc_act_func='sigmoid', learning_rate=art_lr or 0.0)
    m = cell(data['H'], max_len=50, batch_users=128, num_epochs=epochs, seed=seed, learning_rate=1e-2)
    m.fit(data['seqs'], art if art_lr is not None else art.vectors(), impressions=data['train'])
    test = dict(data['test'])
    states = m.impression_states(data['seqs'], art, dict(test, items=np.tile(np.arange(5, dtype=np.int32), len(test['user']))))
    return helpers.impression_metrics(states, art.vectors(data['X_all']), test)['auc']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=100000)
    ap.add_argument('--f', type=int, default=10000)
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--users', type=int, default=32768)
    ap.add_argument('--batch_users', default='1024,4096')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--learning_lrs', default='1e-4,1e-3,1e-2')
    ap.add_argument('--skip_speed', action='store_true')
    ap.add_argument('--skip_learning', action='store_true')
    ap.add_argument('--deterministic', action='store_true',
                    help='also time the frozen and joint paths in the deterministic mode (DESIGN 4.21)')
    args = ap.parse_args()
    args.batch_users = [int(x) for x in args.batch_users.split(',')]
    out = {'gpu': _gpu_info()}
    if not args.skip_speed:
        out['train'] = speed(args)
    if args.skip_learning:
        print(json.dumps(out))
        return
    data = learning_workload()
    out['learning'] = {'frozen': learning_auc(data)}
    for lr in [float(x) for x in args.learning_lrs.split(',') if x]:
        out['learning']['joint_%g' % lr] = learning_auc(data, lr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
