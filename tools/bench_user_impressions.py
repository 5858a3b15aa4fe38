"""Impression logs: GRU training on impressions (the pairwise loss, and the sampled softmax at K = 4 and K = 0) against random
negatives, and the per-impression ranking metrics against a padded torch arm.  One JSON line.

    python tools/bench_user_impressions.py [--n 100000] [--h 500] [--users 32768] [--batch_users 1024,4096] [--imps 1000000] [--reps 3]

Workload: --n clustered articles of width --h (device resident), synth.make_sequences users (mean length 20, the last 50 reads
trained) and synth.make_impressions (shown = 20: one impression per read after the first).  Reported:
  train[B]: one epoch at batch_users B per arm -- impressions with the pairwise loss, with the softmax loss at K = 4 and at K = 0,
            and random negatives -- (host packing and the impression batches built outside the timed span, the arms in rotating
            order, medians of --reps epochs after a warm-up epoch of each): positions/s, impressions/s, clicks/s, and the loss
            kernel's device time per epoch (dae_impression_rank_loss, dae_impression_softmax_loss or dae_seq_rank_loss, CUDA
            events around the kernel in a separate epoch);
  metrics: --imps impressions of 20-54 shown articles (mean 37) with random queries: dae_impression_metrics alone (inputs on
           the device, CUDA events), helpers.impression_metrics as a whole (host checks, uploads, the means; synchronised
           wall clock), and a torch arm on the same device (padded gather + bmm, the ranks and the four metrics by padded torch
           ops, in chunks of 50 000 impressions), each the median of --reps calls in rotating order; the two arms' metrics
           compared on the same scores; the peak device memory of impression_metrics above its inputs.
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
from dae_rnn_news_recommendation_b200 import _cabi, helpers  # noqa: E402
from dae_rnn_news_recommendation_b200.synth import make_impressions, make_sequences  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import (ImpressionBatch, Packed, UserGRU, check_impressions,  # noqa: E402
                                                         usable_impressions)


def _gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi failed: %s' % e


def _epoch(m, batches, emb, epoch):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for bi, (pk, ib) in enumerate(batches):
        m._forward_backward(pk, emb, epoch, bi, ib)
        m._optimizer_step()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _loss_ms(m, batches, emb, epoch):
    m.phase_events = []
    _epoch(m, batches, emb, epoch)
    torch.cuda.synchronize()
    ev, ms = m.phase_events, 0.0
    for (_, a), (name, b) in zip(ev[:-1], ev[1:]):
        if name == 'loss':
            ms += a.elapsed_time(b)
    m.phase_events = None
    return ms


ARMS = {'impressions': {}, 'softmax K=4': dict(impression_loss='softmax', impression_negatives=4),
        'softmax K=0': dict(impression_loss='softmax', impression_negatives=0), 'random negatives': {}}


def train_arm(args, B, indptr, items, emb, imp):
    res = {'batch_users': B}
    use = usable_impressions(imp, indptr, 50)
    active = np.unique(imp['user'][use])
    arms = {}
    names = list(ARMS)
    for name in names:
        m = UserGRU(args.h, max_len=50, batch_users=B, seed=0, **ARMS[name])
        if name != 'random negatives':
            b = []
            for u in m.batches(indptr, 0, active):
                pk = Packed(indptr, items, u, 50)
                b.append((pk, ImpressionBatch(pk, imp, use, indptr)))
        else:
            b = [(Packed(indptr, items, u, 50), None) for u in m.batches(indptr, 0)]
        _epoch(m, b, emb, 0)                                        # warm-up
        arms[name] = (m, b, [])
    for r in range(args.reps):
        for name in names[r % len(names):] + names[:r % len(names)]:
            m, b, t = arms[name]
            t.append(_epoch(m, b, emb, 1 + r))
    for name, (m, b, t) in arms.items():
        sec = float(np.median(t))
        pos = sum(pk.P for pk, _ in b)
        out = {'epoch_s': sec, 'epochs_s': t, 'positions_per_s': pos / sec, 'positions': pos, 'batches': len(b),
               'loss_kernel_ms_per_epoch': _loss_ms(m, b, emb, 99)}
        if name != 'random negatives':
            n, c = sum(ib.n for _, ib in b), sum(ib.clicks for _, ib in b)
            out.update({'impressions': n, 'impressions_per_s': n / sec, 'clicks': c, 'clicks_per_s': c / sec})
        res[name] = out
    return res


def torch_metrics(q, emb, indptr_d, items_d, clicked_d, m_max, chunk=50000, scores=None):
    """The padded torch arm: [I, 4] AUC, MRR, nDCG@5, nDCG@10 with the same tie rule (scores: use these instead of bmm's)."""
    n_imp = q.shape[0]
    out = torch.empty(n_imp, 4, dtype=torch.float64, device=q.device)
    ar = torch.arange(m_max, device=q.device)
    disc = 1.0 / torch.log2(ar.double() + 2.0)
    for a in range(0, n_imp, chunk):
        b = min(n_imp, a + chunk)
        lo, ln = indptr_d[a:b], indptr_d[a + 1:b + 1] - indptr_d[a:b]
        valid = ar[None, :] < ln[:, None]
        idx = torch.where(valid, lo[:, None] + ar[None, :], torch.zeros_like(lo)[:, None])
        if scores is None:
            E = emb[items_d[idx].long()]                                  # [c, m, H]
            s = torch.bmm(E, q[a:b, :, None])[:, :, 0]
        else:
            s = scores[idx]
        c = (clicked_d[idx] != 0) & valid
        n = (~c) & valid
        gt = (s[:, None, :] > s[:, :, None]) & valid[:, None, :]          # [c, j, k]: s_k > s_j
        tb = (s[:, None, :] == s[:, :, None]) & valid[:, None, :] & (ar[None, :] < ar[:, None])[None]
        rank = (gt.sum(2) + tb.sum(2)).double()
        below = ((s[:, None, :] < s[:, :, None]) & n[:, None, :]).sum(2)
        tie = ((s[:, None, :] == s[:, :, None]) & n[:, None, :]).sum(2)
        nc, nn = c.sum(1).double(), n.sum(1).double()
        auc = ((2 * below + tie) * c).sum(1).double() / (2 * nc * nn)
        mrr = (c / (rank + 1)).sum(1) / nc
        g = torch.where(rank < 10, 1.0 / torch.log2(rank + 2), torch.zeros_like(rank))
        g5 = (g * (rank < 5) * c).sum(1)
        g10 = (g * c).sum(1)
        cum = torch.cumsum(disc, 0)
        i5 = cum[(nc.clamp(max=5) - 1).clamp(min=0).long()]
        i10 = cum[(nc.clamp(max=10) - 1).clamp(min=0).long()]
        r = torch.stack([auc, mrr, g5 / i5, g10 / i10], 1)
        r[(nc == 0) | (nn == 0)] = float('nan')
        out[a:b] = r
    return out


def _events(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def metrics_arm(args, emb, rng):
    n_imp, N, H = args.imps, emb.shape[0], args.h
    lens = rng.integers(20, 55, n_imp)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    row = np.repeat(np.arange(n_imp), lens)
    # distinct articles per impression: a random start and a random odd stride modulo N
    pos = np.arange(int(indptr[-1])) - np.repeat(indptr[:-1], lens)
    items = ((rng.integers(0, N, n_imp)[row] + pos * (2 * rng.integers(1, 1000, n_imp)[row] + 1)) % N).astype(np.int32)
    clicked = (rng.random(items.size) < 0.1).astype(np.uint8)
    clicked[indptr[:-1]] = 1
    imp = {'indptr': indptr, 'items': items, 'clicked': clicked}
    check_impressions(imp, N, 'bench')
    q = torch.randn(n_imp, H, device='cuda') / np.sqrt(H)
    d = {k: torch.from_numpy(v).cuda() for k, v in imp.items()}
    scores = torch.empty(items.size, dtype=torch.float32, device='cuda')
    met = torch.empty(n_imp, 4, dtype=torch.float64, device='cuda')
    st = torch.cuda.current_stream().cuda_stream

    def kernel():
        _cabi.call('dae_impression_metrics', q.data_ptr(), H, emb.data_ptr(), H, H, 0, d['indptr'].data_ptr(), d['items'].data_ptr(),
                   d['clicked'].data_ptr(), n_imp, scores.data_ptr(), met.data_ptr(), st)

    def whole():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        helpers.impression_metrics(q, emb, imp)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    m_max = int(lens.max())
    kernel(), whole(), torch_metrics(q, emb, d['indptr'], d['items'], d['clicked'], m_max)   # warm-up
    t = {'kernel': [], 'impression_metrics': [], 'torch': []}
    for r in range(args.reps):
        order = ['kernel', 'impression_metrics', 'torch']
        for name in order[r % 3:] + order[:r % 3]:
            if name == 'kernel':
                t[name].append(_events(kernel))
            elif name == 'impression_metrics':
                t[name].append(whole())
            else:
                t[name].append(_events(lambda: torch_metrics(q, emb, d['indptr'], d['items'], d['clicked'], m_max)))
    kernel()
    torch.cuda.synchronize()
    ref = torch_metrics(q, emb, d['indptr'], d['items'], d['clicked'], m_max, scores=scores)   # the torch arm on the kernel's scores
    own = torch_metrics(q, emb, d['indptr'], d['items'], d['clicked'], m_max)
    km, rm, om = met.cpu().numpy(), ref.cpu().numpy(), own.cpu().numpy()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    res = helpers.impression_metrics(q, emb, imp)
    peak = torch.cuda.max_memory_allocated() - base
    return {'impressions': n_imp, 'shown': int(items.size), 'mean_shown': float(lens.mean()),
            'ms': {k: float(np.median(v)) for k, v in t.items()}, 'ms_all': t,
            'impressions_per_s_kernel': n_imp / (np.median(t['kernel']) / 1e3),
            'same_scores_auc_equal': bool(np.array_equal(km[:, 0], rm[:, 0])),
            'same_scores_max_abs_diff': float(np.abs(km - rm).max()),
            'bmm_scores_mean_abs_diff': [float(x) for x in np.abs(km.mean(0) - om.mean(0))],
            'means': {k: res[k] for k in ('auc', 'mrr', 'ndcg@5', 'ndcg@10')}, 'peak_mem_above_inputs_mb': peak / 2 ** 20}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=100000)
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--users', type=int, default=32768)
    ap.add_argument('--batch_users', default='1024,4096')
    ap.add_argument('--imps', type=int, default=1000000)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_user_impressions: no CUDA device')
    rng = np.random.default_rng(0)
    labels = rng.integers(0, 50, args.n)
    emb = ((rng.standard_normal((50, args.h))[labels] + 0.6 * rng.standard_normal((args.n, args.h))) / np.sqrt(args.h)).astype(np.float32)
    emb_d = torch.from_numpy(emb).cuda()
    indptr, items, _ = make_sequences(args.users, labels, mean_len=20, seed=1, holdout=False)
    train, _ = make_impressions(indptr, items, labels, shown=20, seed=2)
    imp = check_impressions(train, args.n, 'bench', indptr)
    out = {'tool': 'bench_user_impressions', 'gpu': _gpu_info(), 'device_name': torch.cuda.get_device_name(0),
           'n': args.n, 'h': args.h, 'users': args.users, 'train_impressions': int(imp['user'].size), 'train': []}
    for B in [int(x) for x in args.batch_users.split(',') if x]:
        out['train'].append(train_arm(args, B, indptr, items, emb_d, imp))
    out['metrics'] = metrics_arm(args, emb_d, rng)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
