"""Impression logs on the GPU: dae_impression_rank_loss and dae_impression_metrics against the fp64 restatements of
tests/impression_oracle.py, one packed batch's gradients against autograd, the equivalence of one-pair impressions with the
random-negative loss, UserGRU.impression_states, the learning check and the CLI's impression flags."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import impression_oracle as io  # noqa: E402
from gru_kernel_oracle import philox_first_word  # noqa: E402
from helpers import rel_err  # noqa: E402
from user_gru_oracle import NAMES  # noqa: E402

from dae_rnn_news_recommendation_b200 import _cabi, helpers  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import (ImpressionBatch, Packed, UserGRU, check_impressions,  # noqa: E402
                                                         negatives_from_draws, usable_impressions)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _csr(lists, clicks):
    indptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return indptr, np.concatenate(lists).astype(np.int32), np.concatenate(clicks).astype(np.uint8)


def _random_lists(rng, N, sizes, p_click=0.3):
    lists, clicks = [], []
    for m in sizes:
        lists.append(rng.choice(N, m, replace=False))
        c = (rng.random(m) < p_click).astype(np.uint8)
        if m > 1:                                       # at least one click and one non-click
            j = rng.integers(0, m)
            c[j], c[(j + 1) % m] = 1, 0
        clicks.append(c)
    return lists, clicks


def _loss_call(h, emb, pos_indptr, indptr, items, clicked, scale):
    P, H = h.shape
    d = {k: _cuda(v) for k, v in (('h', h), ('emb', emb), ('pi', pos_indptr), ('ip', indptr), ('it', items), ('c', clicked))}
    dh = torch.full((P, H), float('nan'), dtype=torch.float32, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    _cabi.call('dae_impression_rank_loss', d['h'].data_ptr(), H, d['emb'].data_ptr(), H, H, d['pi'].data_ptr(), P, d['ip'].data_ptr(),
               d['it'].data_ptr(), d['c'].data_ptr(), scale, dh.data_ptr(), H, loss.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return float(loss.item()), dh.cpu().numpy()


@pytest.mark.parametrize('H', [37, 500])
def test_loss_kernel_against_oracle(H):
    rng = np.random.default_rng(H)
    N, P = 6000, 40
    emb = (rng.standard_normal((N, H)) / np.sqrt(H)).astype(np.float32)
    h = (rng.standard_normal((P, H)) * 2).astype(np.float32)
    sizes = list(rng.integers(2, 40, 60)) + [5000, 257, 2, 1]
    lists, clicks = _random_lists(rng, N, sizes)
    clicks[3][:] = 0                                    # skipped: no click
    clicks[4][:] = 1                                    # skipped: no non-click
    clicks[60][rng.choice(5000, 700, replace=False)] = 1  # |C| > 1 across the 256-score chunks
    indptr, items, clicked = _csr(lists, clicks)
    n_imp = len(sizes)
    # positions: several impressions at some, none at others (p % 3 == 1)
    pos = np.sort(rng.choice([p for p in range(P) if p % 3 != 1], n_imp))
    pos_indptr = np.zeros(P + 1, np.int64)
    np.cumsum(np.bincount(pos, minlength=P), out=pos_indptr[1:])
    assert (np.diff(pos_indptr) > 1).any()
    scale = 1.0 / 17
    loss, dh = _loss_call(h, emb, pos_indptr, indptr, items, clicked, scale)
    o_loss, o_dh = io.impression_loss(h, emb, pos_indptr, indptr, items, clicked, float(np.float32(scale)))
    empty = np.diff(pos_indptr) == 0
    assert (dh[empty] == 0).all() and not np.isnan(dh).any()
    assert rel_err(dh, o_dh) < 1e-4, rel_err(dh, o_dh)
    big = pos[60]                                       # the 5 000-article impression's row on its own scale
    assert rel_err(dh[big], o_dh[big]) < 1e-4
    assert rel_err(loss, o_loss) < 1e-4, (loss, o_loss)
    # deterministic: no atomics on dH
    _, dh2 = _loss_call(h, emb, pos_indptr, indptr, items, clicked, scale)
    assert np.array_equal(dh.view(np.uint32), dh2.view(np.uint32))


def _data(U, H, N, max_len, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 4, U)
    lens[:6] = [1, 2, max_len, max_len + 3, 2 * max_len, 1]
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N, int(indptr[-1])).astype(np.int32)
    emb = (rng.standard_normal((N, H)) * 0.5).astype(np.float32)
    return indptr, items, emb


def _random_impressions(rng, indptr, N, per_user=3, shown=(2, 12)):
    user, time, lists, clicks = [], [], [], []
    lens = np.diff(indptr)
    for u in range(lens.size):
        for _ in range(per_user):
            user.append(u)
            time.append(rng.integers(0, lens[u] + 1))
            m = int(rng.integers(*shown))
            lists.append(rng.choice(N, m, replace=False))
            c = (rng.random(m) < 0.3).astype(np.uint8)
            c[0] = 1
            clicks.append(c)
    indptr_i, items_i, clicked = _csr(lists, clicks)
    return {'user': np.array(user, np.int64), 'time': np.array(time, np.int64), 'indptr': indptr_i, 'items': items_i, 'clicked': clicked}


def _grads(m):
    H, g = m.dim, m.grad.cpu().double().numpy()
    hh, ih = g[:m.nW].reshape(3 * H, H + 1), g[m.nW:].reshape(3 * H, H + 1)
    return {'weight_ih_l0': ih[:, :H], 'weight_hh_l0': hh[:, :H], 'bias_ih_l0': ih[:, H], 'bias_hh_l0': hh[:, H]}


@pytest.mark.parametrize('H,U,max_len', [(37, 200, 10), (500, 100, 8)])
def test_batch_gradients_against_autograd(H, U, max_len):
    N = 900
    indptr, items, emb = _data(U, H, N, max_len, seed=H + 1)
    rng = np.random.default_rng(H)
    imp = check_impressions(_random_impressions(rng, indptr, N), N, 'test', indptr)
    use = usable_impressions(imp, indptr, max_len)
    m = UserGRU(H, max_len=max_len, batch_users=U, seed=1)
    pk = Packed(indptr, items, np.arange(U), max_len)
    ib = ImpressionBatch(pk, imp, use, indptr)
    assert 0 < ib.n < use.size
    m.stats.zero_()
    m._forward_backward(pk, torch.from_numpy(emb).cuda(), 0, 0, ib)
    torch.cuda.synchronize()
    loss = float(m.stats.item()) / ib.n
    seqs = [pk.items[[pk.position(i, t) for t in range(int(pk.L[i]))]] for i in range(pk.B)]
    row = {int(u): i for i, u in enumerate(pk.order)}
    imps = []
    for q, iid in enumerate(ib.ids):
        u = int(imp['user'][iid])
        i = row[u]
        t = int(imp['time'][iid]) - 1 - (int(indptr[u + 1] - indptr[u]) - int(pk.L[i]))
        a, b = ib.indptr[q], ib.indptr[q + 1]
        imps.append((i, t, ib.items[a:b], ib.clicked[a:b]))
    params = {k: v.double().numpy() for k, v in m.state_dict().items()}
    o_loss, o_g = io.impression_loss_and_grads(params, seqs, emb, imps)
    assert rel_err(loss, o_loss) < 1e-4, (loss, o_loss)
    g = _grads(m)
    for k in NAMES:
        assert rel_err(g[k], o_g[k]) < 1e-4, (k, rel_err(g[k], o_g[k]))


def test_one_pair_impressions_equal_random_negatives():
    """Epoch 0's Philox negatives, rebuilt on the host, as one-click / one-non-click impressions: one epoch of fit(impressions=)
    is fit()."""
    H, U, N, max_len = 37, 500, 800, 12
    indptr, items, emb = _data(U, H, N, max_len, seed=3)
    kw = dict(max_len=max_len, batch_users=128, num_epochs=1, seed=5, learning_rate=3e-3)
    a = UserGRU(H, **kw)
    user, time, lists = [], [], []
    lens = np.diff(indptr)
    for bi, users in enumerate(a.batches(indptr, 0)):
        pk = Packed(indptr, items, users, max_len)
        has = np.flatnonzero(pk.nxt >= 0)
        neg = negatives_from_draws(pk.nxt[has], philox_first_word(has, bi, 0, 5), N)
        for p, ng in zip(has, neg):
            t = int(np.searchsorted(pk.off, p, side='right') - 1)
            i = int(p - pk.off[t])
            u = int(pk.order[i])
            user.append(u)
            time.append(int(lens[u] - pk.L[i]) + t + 1)
            lists.append([pk.nxt[p], ng])
    imp = {'user': np.array(user), 'time': np.array(time), 'indptr': np.arange(0, 2 * len(lists) + 1, 2),
           'items': np.array(lists, np.int32).reshape(-1), 'clicked': np.tile(np.array([1, 0], np.uint8), len(lists))}
    a.fit((indptr, items), emb)
    b = UserGRU(H, **kw).fit((indptr, items), emb, impressions=imp)
    assert b.impression_counts == {'used': len(lists), 'skipped': 0}
    assert abs(a.train_loss[0] - b.train_loss[0]) <= 1e-6 * abs(a.train_loss[0]), (a.train_loss, b.train_loss)
    sa, sb = a.state_dict(), b.state_dict()
    for k in NAMES:
        assert rel_err(sb[k].numpy(), sa[k].numpy()) < 1e-5, (k, rel_err(sb[k].numpy(), sa[k].numpy()))


def _metrics_call(q, emb, indptr, items, clicked, cosine):
    s, m = helpers._impression_scores(_cuda(q.astype(np.float32)), _cuda(emb.astype(np.float32)),
                                      {'indptr': indptr, 'items': items, 'clicked': clicked}, 'cosine' if cosine else 'linear kernel')
    return s.cpu().numpy(), m.cpu().numpy()


def test_metrics_kernel_exact_with_ties():
    rng = np.random.default_rng(0)
    N, H = 6000, 16
    emb = rng.integers(-2, 3, (N, H)).astype(np.float32)
    sizes = list(rng.integers(1, 70, 300)) + [600, 5000, 1, 2]
    lists, clicks = _random_lists(rng, N, sizes)
    clicks[7][:] = 0
    clicks[8][:] = 1
    indptr, items, clicked = _csr(lists, clicks)
    q = rng.integers(-1, 2, (len(sizes), H)).astype(np.float32)
    q[5] = 0                                                      # every score 0: rank by position
    s, m = _metrics_call(q, emb, indptr, items, clicked, False)
    want_s = io.scores(q, emb, indptr, items, False)
    assert np.array_equal(s.astype(np.float64), want_s)          # integer scores are exact
    # ties across the click boundary
    row = np.repeat(np.arange(len(sizes)), np.diff(indptr))
    tie = sum(np.isin(s[(row == i) & (clicked == 1)], s[(row == i) & (clicked == 0)]).any() for i in range(len(sizes)))
    assert tie > 50
    want, _ = io.metrics(s, indptr, clicked)
    nan = np.isnan(want[:, 0])
    assert np.array_equal(np.isnan(m), np.repeat(nan[:, None], 4, 1))
    assert nan[7] and nan[8] and nan[len(sizes) - 2]            # no click, no non-click, a single candidate
    assert np.array_equal(m[~nan, 0], want[~nan, 0])
    np.testing.assert_allclose(m[~nan], want[~nan], rtol=1e-12, atol=0)


@pytest.mark.parametrize('cosine', [False, True])
def test_metrics_kernel_random(cosine):
    rng = np.random.default_rng(1 + cosine)
    N, H = 7000, 500
    emb = (rng.standard_normal((N, H)) / np.sqrt(H)).astype(np.float32)
    emb[3] = 0
    sizes = list(rng.integers(1, 80, 400)) + [5000]
    lists, clicks = _random_lists(rng, N, sizes)
    lists[0][0] = 3                                               # a zero article: cosine 0
    indptr, items, clicked = _csr(lists, clicks)
    q = rng.standard_normal((len(sizes), H)).astype(np.float32)
    q[1] = 0                                                      # a zero query
    s, m = _metrics_call(q, emb, indptr, items, clicked, cosine)
    want_s = io.scores(q, emb, indptr, items, cosine)
    assert np.abs(s - want_s).max() <= 1e-5 * np.abs(want_s).max()
    assert (s[indptr[1]:indptr[2]] == 0).all()
    if cosine:
        assert s[indptr[0]] == 0
    want, ints = io.metrics(s, indptr, clicked)                   # from the kernel's own scores
    nan = np.isnan(want[:, 0])
    assert np.array_equal(np.isnan(m[:, 0]), nan)
    n_c = np.add.reduceat(clicked.astype(np.int64), indptr[:-1])
    n_n = np.diff(indptr) - n_c
    ok = ~nan
    assert np.array_equal(np.rint(m[ok, 0] * 2 * n_c[ok] * n_n[ok]).astype(np.int64), ints[ok, 0])
    assert np.array_equal(m[ok, 0], want[ok, 0])
    np.testing.assert_allclose(m[ok], want[ok], rtol=1e-12, atol=0)
    # the public helper: means over the scored impressions
    r = helpers.impression_metrics(q, emb, {'indptr': indptr, 'items': items, 'clicked': clicked},
                                   metric='cosine' if cosine else 'linear kernel')
    assert r['impressions'] == ok.sum() and r['skipped'] == nan.sum()
    assert r['auc'] == pytest.approx(want[ok, 0].mean(), rel=1e-12) and r['ndcg@10'] == pytest.approx(want[ok, 3].mean(), rel=1e-12)
    with pytest.raises(ValueError, match='finite'):
        helpers.impression_metrics(np.where(np.arange(H) == 0, np.nan, q), emb, {'indptr': indptr, 'items': items, 'clicked': clicked})
    with pytest.raises(ValueError, match='shape'):
        helpers.impression_metrics(q[1:], emb, {'indptr': indptr, 'items': items, 'clicked': clicked})
    with pytest.raises(ValueError, match='metric'):
        helpers.impression_metrics(q, emb, {'indptr': indptr, 'items': items, 'clicked': clicked}, metric='dot')


def test_impression_states_against_oracle_windows():
    H, U, N, max_len = 37, 150, 700, 10
    indptr, items, emb = _data(U, H, N, max_len, seed=11)
    rng = np.random.default_rng(2)
    imp = _random_impressions(rng, indptr, N, per_user=4)
    lens = np.diff(indptr)
    imp['time'][:U] = lens                                        # time = len for every user's first impression
    imp['time'][U:U + 5] = 0
    imp = dict(imp, user=np.concatenate([np.arange(U), imp['user'][U:]]))
    m = UserGRU(H, max_len=max_len, batch_users=64, seed=4)
    got = m.impression_states((indptr, items), emb, imp)
    assert got.shape == (len(imp['user']), H)
    params = {k: v.double().numpy() for k, v in m.state_dict().items()}
    want = io.window_states(params, indptr, items, imp['user'], imp['time'], emb, max_len)
    assert (imp['time'] > max_len).sum() > 20
    assert not got[imp['time'] == 0].any()
    assert rel_err(got, want) < 1e-4, rel_err(got, want)
    tr = m.transform((indptr, items), emb)
    assert rel_err(got[:U], tr) < 1e-6


# test-impression AUC measured on an H100 80GB HBM3 at 700 W: impressions 0.9547, random negatives 0.9343, mean profile 0.7813
# (DESIGN 4.13); the asserted margin is half the gap to the mean profile.  The 0.020 lead over random negatives is one run and
# is printed, not asserted.
LEARNING_MARGIN = 0.087


def _learning_numbers():
    from dae_rnn_news_recommendation_b200.synth import make_impressions, make_sequences
    from dae_rnn_news_recommendation_b200.user_model import prefix_histories
    from test_gpu_user_gru import _clustered
    N, H = 3000, 64
    labels, emb = _clustered(N, H, 8, 11)
    indptr, items, targets = make_sequences(8000, labels, mean_len=20, session_len=5, seed=12)
    train, test = make_impressions(indptr, items, labels, targets, shown=20, seed=13)
    kw = dict(max_len=50, batch_users=512, num_epochs=8, learning_rate=3e-3, seed=0)
    g_imp = UserGRU(H, **kw).fit((indptr, items), emb, impressions=train)
    g_neg = UserGRU(H, **kw).fit((indptr, items), emb)
    auc = {}
    for name, g in (('impressions', g_imp), ('random negatives', g_neg)):
        auc[name] = helpers.impression_metrics(g.impression_states((indptr, items), emb, test), emb, test)['auc']
    prof = helpers.user_profiles(prefix_histories((indptr, items), test, N), emb)
    auc['mean profile'] = helpers.impression_metrics(prof, emb, test, metric='cosine')['auc']
    return auc, g_imp.train_loss, g_imp.impression_counts


def test_learning_beats_mean_profile():
    auc, losses, counts = _learning_numbers()
    print('test-impression AUC: %s; impression train loss %s; %s' % (
        ', '.join('%s %.4f' % kv for kv in auc.items()), ['%.4f' % x for x in losses], counts))
    assert losses[-1] < losses[0]
    assert auc['impressions'] > 0.5
    assert auc['impressions'] - auc['mean profile'] > LEARNING_MARGIN, auc


def test_cli_user_impressions(capsys, tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.synth import make_impressions, make_sequences
    argv = ['--model_name', 'synimp', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--top_k', '5']
    trX, _, trL, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    indptr, items, targets = make_sequences(300, trL, mean_len=8, seed=4)
    train, test = make_impressions(indptr, items, trL, targets, shown=10, seed=5)
    np.savez(tmp_path / 's.npz', indptr=indptr, items=items, targets=targets)
    np.savez(tmp_path / 'tr.npz', **train)
    np.savez(tmp_path / 'te.npz', **test)
    model = cli.main(argv + ['--user_sequences', str(tmp_path / 's.npz'), '--user_epochs', '2', '--user_impressions',
                             str(tmp_path / 'tr.npz'), '--user_test_impressions', str(tmp_path / 'te.npz')])
    printed = capsys.readouterr().out
    assert 'test impressions (GRU): AUC' in printed and 'impressions:' in printed
    for who in ('gru', 'mean'):
        for k in ('auc', 'mrr', 'ndcg5', 'ndcg10'):
            assert 0.0 <= model.evaluation['user_%s_imp_%s' % (who, k)] <= 1.0
