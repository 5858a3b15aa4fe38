"""The long-term user vectors of the GRU / LSTM user encoders (user_model, long_term_users; DESIGN 4.18): training speed with and
without the table, the row update's kernel time, the table's memory, transform time and the learning check.  One JSON line.

    python tools/bench_user_long_term.py [--cell gru|lstm] [--n 100000] [--h 500] [--users 32768] [--batch_users 1024,4096]
                                         [--table_users 100000,1000000] [--rounds 3] [--learning_lrs 0.01,0.03,0.1]

Reported:
  train[B]: positions/s over one epoch of --users make_sequences users (bench_user_model.py's workload) at batch_users B, plain
            and with a table of --users rows (mask 0.5), after a warm-up epoch of each, over --rounds alternating rounds;
  rows_step[U]: CUDA-event time per call of dae_rows_optimizer_step (Adam, B = 1024 and 4096 distinct random rows of a [U, H]
            table) next to dae_optimizer_step (Adam) over a theta of U x H floats, 50 calls per timing, alternating rounds;
  memory[U]: device bytes of the table, its Adam slots and row counts (the allocation growth when the model is built);
  transform[U]: transform of U users (batch_users 16384) plain and with a table of U rows, alternating rounds;
  learning: synth.make_long_term_impressions (the signal lies before the window of the last max_len reads): test-impression
            AUC of the same GRU trained plain and with the table at each --learning_lrs learning rate.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from bench_user_model import _epoch, _gpu_info  # noqa: E402
from dae_rnn_news_recommendation_b200 import _cabi, helpers  # noqa: E402
from dae_rnn_news_recommendation_b200.synth import make_long_term_impressions, make_sequences  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import Packed, UserGRU, UserLSTM  # noqa: E402

CELLS = {'gru': UserGRU, 'lstm': UserLSTM}


def _events_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def train_arm(args, B, indptr, items, emb):
    U = len(indptr) - 1
    ms = {'plain': args.cls(args.h, max_len=50, batch_users=B, seed=0),
          'long_term': args.cls(args.h, max_len=50, batch_users=B, seed=0, long_term_users=U)}
    packs = [Packed(indptr, items, u, 50) for u in ms['plain'].batches(indptr, 1)]
    for m in ms.values():
        _epoch(m, indptr, items, emb, 0)                      # warm-up
    out = {k: [] for k in ms}
    for r in range(args.rounds):
        for k, m in ms.items():
            sec, pos, _, _ = _epoch(m, indptr, items, emb, 1 + r, packs)
            out[k].append(pos / sec)
    return {'batch_users': B, 'positions': sum(p.P for p in packs),
            **{k + '_positions_per_s': float(np.median(v)) for k, v in out.items()}, 'rounds': out}


def rows_step_arm(args, U):
    H, d = args.h, 'cuda:0'
    table, s1, s2 = (torch.zeros(U + 1, H, device=d) for _ in range(3))
    counts = torch.zeros(U + 1, dtype=torch.int32, device=d)
    theta = torch.zeros(U * H, device=d)
    g_theta, t1, t2 = torch.randn(U * H, device=d), torch.zeros(U * H, device=d), torch.zeros(U * H, device=d)
    st = torch.cuda.current_stream().cuda_stream
    res = {'users': U}
    for B in (1024, 4096):
        rows = torch.from_numpy(np.random.default_rng(B).choice(U, B, replace=False).astype(np.int32)).to(d)
        grad = torch.randn(B, H, device=d)
        rows_fn = lambda: _cabi.call('dae_rows_optimizer_step', table.data_ptr(), H, H, rows.data_ptr(), B, grad.data_ptr(), H,  # noqa: E731
                                     s1.data_ptr(), s2.data_ptr(), counts.data_ptr(), _cabi.OPT['adam'], 1e-2, 0.5, st)
        _events_ms(rows_fn, 5)
        t = [_events_ms(rows_fn, 50) for _ in range(args.rounds)]
        res['rows_step_ms_B%d' % B] = float(np.median(t))
    full_fn = lambda: _cabi.call('dae_optimizer_step', theta.data_ptr(), g_theta.data_ptr(), t1.data_ptr(), t2.data_ptr(), U * H,  # noqa: E731
                                 _cabi.OPT['adam'], 1e-3, 0.5, 1.0, 1, None, None, None, 0, 0, 0, st)
    _events_ms(full_fn, 3)
    res['dense_optimizer_step_ms'] = float(np.median([_events_ms(full_fn, 20) for _ in range(args.rounds)]))
    del table, s1, s2, counts, theta, g_theta, t1, t2
    torch.cuda.empty_cache()
    return res


def memory_arm(args, U):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    a = torch.cuda.memory_allocated()
    plain = args.cls(args.h, seed=0)
    b = torch.cuda.memory_allocated()
    m = args.cls(args.h, seed=0, long_term_users=U)
    c = torch.cuda.memory_allocated()
    out = {'users': U, 'table_and_adam_slots_bytes': int((c - b) - (b - a)),
           'table_bytes': int(m._lt.numel() * 4), 'per_user_bytes': float(((c - b) - (b - a)) / U)}
    del plain, m
    torch.cuda.empty_cache()
    return out


def transform_arm(args, labels, emb, U):
    indptr, items, _ = make_sequences(U, labels, mean_len=20, seed=7, holdout=False)
    ms = {'plain': args.cls(args.h, max_len=50, batch_users=16384, seed=0),
          'long_term': args.cls(args.h, max_len=50, batch_users=16384, seed=0, long_term_users=U)}
    for m in ms.values():
        m.transform((indptr[:1001], items[:indptr[1000]]), emb, to_host=False)   # warm-up
    t = {k: [] for k in ms}
    for _ in range(args.rounds):
        for k, m in ms.items():
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            m.transform((indptr, items), emb, to_host=False)
            b.record()
            torch.cuda.synchronize()
            t[k].append(a.elapsed_time(b) / 1e3)
    del ms
    torch.cuda.empty_cache()
    return {'users': U, **{k + '_s': float(np.median(v)) for k, v in t.items()}, 'rounds': t}


LEARNING = dict(N=3000, H=64, classes=8, users=4000, max_len=5, epochs=10, batch_users=512, lr=3e-3)


def learning_workload(seed=0):
    """(indptr, items, train, test, emb) of the learning check: LEARNING's sizes, clustered article vectors."""
    c = LEARNING
    rng = np.random.default_rng(seed + 11)
    labels = rng.integers(0, c['classes'], c['N'])
    emb = ((rng.standard_normal((c['classes'], c['H']))[labels] + 0.6 * rng.standard_normal((c['N'], c['H']))) /
           np.sqrt(c['H'])).astype(np.float32)
    indptr, items, train, test = make_long_term_impressions(c['users'], labels, window=c['max_len'], seed=seed + 12)
    return indptr, items, train, test, emb


def learning_auc(cls, data, long_term_lr=None):
    """Test-impression AUC of cls trained on the learning workload: plain (long_term_lr None) or with the table at long_term_lr."""
    indptr, items, train, test, emb = data
    c = LEARNING
    kw = {} if long_term_lr is None else dict(long_term_users=len(indptr) - 1, long_term_learning_rate=long_term_lr)
    m = cls(c['H'], max_len=c['max_len'], batch_users=c['batch_users'], num_epochs=c['epochs'], learning_rate=c['lr'], seed=0, **kw)
    m.fit((indptr, items), emb, impressions=train)
    q = m.impression_states((indptr, items), emb, test)
    return helpers.impression_metrics(q, emb, test, metric='linear kernel')['auc']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cell', default='gru', choices=sorted(CELLS))
    ap.add_argument('--n', type=int, default=100000)
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--users', type=int, default=32768)
    ap.add_argument('--batch_users', default='1024,4096')
    ap.add_argument('--table_users', default='100000,1000000')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--learning_lrs', default='0.01,0.03,0.1')
    ap.add_argument('--skip', default='', help='comma-separated parts to skip: train, rows, memory, transform, learning')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_user_long_term: no CUDA device')
    args.cls = CELLS[args.cell]
    skip = set(args.skip.split(','))
    res = {'cell': args.cell, 'N': args.n, 'H': args.h, 'gpu': _gpu_info(), 'device_name': torch.cuda.get_device_name(0)}
    rng = np.random.RandomState(0)
    labels = rng.randint(0, 16, args.n)
    emb = torch.from_numpy(((rng.randn(16, args.h)[labels] + 0.6 * rng.randn(args.n, args.h)) / np.sqrt(args.h)).astype(np.float32)).cuda()
    table_users = [int(u) for u in args.table_users.split(',')]
    if 'train' not in skip:
        indptr, items, _ = make_sequences(args.users, labels, mean_len=20, seed=1, holdout=False)
        res['train'] = [train_arm(args, int(B), indptr, items, emb) for B in args.batch_users.split(',')]
    if 'rows' not in skip:
        res['rows_step'] = [rows_step_arm(args, U) for U in table_users]
    if 'memory' not in skip:
        res['memory'] = [memory_arm(args, U) for U in table_users]
    if 'transform' not in skip:
        res['transform'] = [transform_arm(args, labels, emb, U) for U in table_users]
    if 'learning' not in skip:
        data = learning_workload()
        res['learning'] = {'plain_auc': learning_auc(args.cls, data),
                           **{'long_term_auc_lr%s' % lr: learning_auc(args.cls, data, float(lr)) for lr in args.learning_lrs.split(',')},
                           'config': LEARNING}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
