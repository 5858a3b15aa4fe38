"""Host side of impression logs: check_impressions, the impression -> packed position mapping, the metric oracle against sklearn
and a hand-worked example with ties, make_impressions, prefix_histories, the exports' argument checks and the CLI flags.  No
GPU needed."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import impression_oracle as io  # noqa: E402

from dae_rnn_news_recommendation_b200.user_model import (ImpressionBatch, Packed, check_impressions, prefix_histories,  # noqa: E402
                                                         usable_impressions)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _imp(user, time, lists, clicks):
    indptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return {'user': np.array(user, np.int64), 'time': np.array(time, np.int64), 'indptr': indptr,
            'items': np.concatenate([np.array(x, np.int32) for x in lists]) if lists else np.zeros(0, np.int32),
            'clicked': np.concatenate([np.array(c, np.uint8) for c in clicks]) if clicks else np.zeros(0, np.uint8)}


def test_check_impressions_errors_and_no_mutation():
    seq_indptr = np.array([0, 3, 3, 8], np.int64)
    good = _imp([0, 2], [1, 5], [[1, 2, 3], [4, 5]], [[1, 0, 0], [0, 1]])
    copy = {k: v.copy() for k, v in good.items()}
    out = check_impressions(good, 10, 'f', seq_indptr)
    assert out['clicked'].dtype == np.uint8 and out['items'].dtype == np.int32
    out['items'][0] = 9
    for k in good:
        assert np.array_equal(good[k], copy[k]) and good[k].dtype == copy[k].dtype
    bad = [
        (dict(indptr=np.array([0, 3, 4])), 'indptr'),                # does not end at len(items)
        (dict(indptr=np.array([0, 4, 3, 5][:3])), 'indptr'),         # decreasing
        (dict(user=np.array([0, 3])), 'user'),                       # no such user
        (dict(user=np.array([0, -1])), 'user'),
        (dict(time=np.array([4, 5])), 'time'),                       # user 0 read 3
        (dict(time=np.array([1, -1])), 'time'),
        (dict(items=np.array([1, 2, 3, 4, 10], np.int32)), 'outside'),
        (dict(items=np.array([1, 2, 1, 4, 5], np.int32)), 'twice'),
        (dict(clicked=np.array([1, 0, 0, 1], np.uint8)), 'clicked'),
        (dict(clicked=np.array([1, 0, 0, 1, 2], np.uint8)), 'clicked'),
        (dict(user=np.array([0])), 'user'),                          # wrong length
    ]
    for change, msg in bad:
        d = dict(good, **change)
        with pytest.raises(ValueError, match=msg):
            check_impressions(d, 10, 'f', seq_indptr)
    with pytest.raises(ValueError, match='map'):
        check_impressions({'indptr': good['indptr']}, 10, 'f')
    # the same article in two impressions is fine; user and time are not read without the sequences
    ok = check_impressions(_imp([9], [99], [[1, 2], [1, 2]][:1], [[1, 0]]), 10, 'f')
    assert 'user' not in ok
    # bool click masks are accepted
    check_impressions(dict(good, clicked=good['clicked'].astype(bool)), 10, 'f', seq_indptr)


def test_mapping_to_packed_positions():
    # users: 0 reads 7 (> max_len = 4), 1 reads 2, 2 reads 0, 3 reads 4
    lens = [7, 2, 0, 4]
    seq_indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = np.arange(int(seq_indptr[-1]), dtype=np.int32) % 20
    max_len = 4
    imp = _imp([0, 0, 0, 0, 1, 1, 1, 3, 3, 3, 0],
               [7, 3, 4, 5, 0, 2, 1, 4, 2, 2, 6],
               [[1, 2], [3, 4], [5, 6], [7, 8], [1, 2], [1, 2, 3], [4, 5], [1, 2], [3, 4], [5, 6], [7, 8, 9]],
               [[1, 0], [1, 0], [1, 0], [0, 1], [1, 0], [1, 1, 0], [0, 0], [0, 1], [1, 0], [1, 1], [1, 0, 1]])
    imp = check_impressions(imp, 20, 'f', seq_indptr)
    use = usable_impressions(imp, seq_indptr, max_len)
    # user 0: window = reads 3..6, so time in 4..7 is inside; time 3 is not.  time = 0 never.  imp 6: no click; imp 9: no non-click
    assert use.tolist() == [True, False, True, True, False, True, False, True, True, False, True]
    pk = Packed(seq_indptr, items, np.array([3, 0, 1]), max_len)
    assert pk.order.tolist() == [3, 0, 1] and pk.L.tolist() == [4, 4, 2]
    ib = ImpressionBatch(pk, imp, use, seq_indptr)
    # t' = time - 1 - (len - L); position = off[t'] + i
    want = {0: pk.off[3] + 1, 2: pk.off[0] + 1, 3: pk.off[1] + 1, 10: pk.off[2] + 1, 5: pk.off[1] + 2, 7: pk.off[3] + 0,
            8: pk.off[1] + 0}
    assert ib.n == len(want)
    got = dict(zip(ib.ids.tolist(), ib.p.tolist()))
    assert got == {k: int(v) for k, v in want.items()}
    # time = len is the user's last position
    assert got[0] == pk.position(1, int(pk.L[1]) - 1)
    assert (np.diff(ib.p) >= 0).all()
    assert ib.pos_indptr[-1] == ib.n and ib.pos_indptr.size == pk.P + 1
    for q, i in enumerate(ib.ids):
        a, b = imp['indptr'][i], imp['indptr'][i + 1]
        assert np.array_equal(ib.items[ib.indptr[q]:ib.indptr[q + 1]], imp['items'][a:b])
        assert np.array_equal(ib.clicked[ib.indptr[q]:ib.indptr[q + 1]], imp['clicked'][a:b])
        assert ib.pos_indptr[ib.p[q]] <= q < ib.pos_indptr[ib.p[q] + 1]
    # one packed buffer cut back into the four arrays
    import torch
    buf = torch.from_numpy(ib.buffer())
    v = ib.views(buf)
    for a, b in zip(v, (ib.pos_indptr, ib.indptr, ib.items, ib.clicked)):
        assert np.array_equal(a.numpy(), b)
    # a batch without user 3 maps none of its impressions
    ib2 = ImpressionBatch(Packed(seq_indptr, items, np.array([1]), max_len), imp, use, seq_indptr)
    assert sorted(ib2.ids.tolist()) == [5]


def test_metric_oracle_hand_example_with_ties():
    # scores 3, 1, 3, 2, 1 ; clicked at positions 2 and 4
    s = np.array([3.0, 1.0, 3.0, 2.0, 1.0], np.float32)
    c = np.array([0, 0, 1, 0, 1], np.uint8)
    m, ints = io.metrics(s, np.array([0, 5]), c)
    # ranks: pos0 -> 0, pos2 -> 1 (tie with the earlier pos0), pos3 -> 2, pos1 -> 3, pos4 -> 4 (tie with pos1)
    # AUC pairs: (3 vs 3) 0.5, (3 vs 1) 1, (3 vs 2) 1, (1 vs 3) 0, (1 vs 1) 0.5, (1 vs 2) 0 -> 3 / 6
    assert ints[0].tolist() == [6, 5]
    assert m[0, 0] == 0.5
    assert m[0, 1] == pytest.approx((1 / 2 + 1 / 5) / 2, rel=1e-15)
    idcg = 1 + 1 / np.log2(3)
    assert m[0, 2] == pytest.approx((1 / np.log2(3) + 1 / np.log2(6)) / idcg, rel=1e-15)
    assert m[0, 3] == m[0, 2]


def test_metric_oracle_against_sklearn():
    from sklearn.metrics import roc_auc_score
    rng = np.random.default_rng(0)
    lens = rng.integers(2, 40, 200)
    indptr = np.concatenate([[0], np.cumsum(lens)])
    s = rng.integers(-3, 4, int(indptr[-1])).astype(np.float32)   # many ties
    c = (rng.random(s.size) < 0.3).astype(np.uint8)
    c[indptr[:5]] = 1
    c[indptr[5]:indptr[6]] = 0                                       # no click
    c[indptr[6]:indptr[7]] = 1                                       # no non-click
    m, _ = io.metrics(s, indptr, c)
    assert np.isnan(m[5]).all() and np.isnan(m[6]).all()
    for i in range(200):
        ci = c[indptr[i]:indptr[i + 1]]
        if ci.all() or not ci.any():
            continue
        assert m[i, 0] == pytest.approx(roc_auc_score(ci, s[indptr[i]:indptr[i + 1]]), abs=1e-15)
        # MIND's mrr_score / ndcg_score with a stable descending order (ties to the earlier position)
        order = np.argsort(-s[indptr[i]:indptr[i + 1]], kind='stable')
        y = ci[order]
        assert m[i, 1] == pytest.approx(np.sum(y / (np.arange(y.size) + 1)) / y.sum(), rel=1e-14)
        for col, k in ((2, 5), (3, 10)):
            dcg = np.sum(y[:k] / np.log2(np.arange(min(k, y.size)) + 2))
            ideal = np.sort(ci)[::-1]
            idcg = np.sum(ideal[:k] / np.log2(np.arange(min(k, y.size)) + 2))
            assert m[i, col] == pytest.approx(dcg / idcg, rel=1e-14)


def test_loss_oracle_one_pair_is_the_random_negative_term():
    rng = np.random.default_rng(1)
    emb = rng.standard_normal((10, 4))
    h = rng.standard_normal((3, 4))
    # position 1: click 2, non-click 7
    loss, dh = io.impression_loss(h, emb, np.array([0, 0, 1, 1]), np.array([0, 2]), np.array([7, 2]), np.array([0, 1]), 0.5)
    x = h[1] @ emb[7] - h[1] @ emb[2]
    assert loss == pytest.approx(np.log1p(np.exp(x)), rel=1e-14)
    np.testing.assert_allclose(dh[1], 0.5 / (1 + np.exp(-x)) * (emb[7] - emb[2]), rtol=1e-14)
    assert not dh[0].any() and not dh[2].any()


def test_make_impressions_properties():
    from dae_rnn_news_recommendation_b200.synth import make_impressions, make_sequences
    labels = np.repeat(np.arange(8), 200)
    labels[:5] = -1
    indptr, items, targets = make_sequences(1500, labels, mean_len=15, seed=2)
    train, test = make_impressions(indptr, items, labels, targets, shown=20, seed=3)
    lens = np.diff(indptr)
    tr = check_impressions(train, labels.size, 'f', indptr)
    te = check_impressions(test, labels.size, 'f', indptr)                   # distinct articles within each impression
    assert tr['user'].size == int(np.maximum(lens - 1, 0).sum())
    assert te['user'].size == int(((targets >= 0) & (lens > 0)).sum())
    assert (te['time'] == lens[te['user']]).all()
    n_other = n_same_other = 0
    for d, kind in ((tr, 'train'), (te, 'test')):
        for i in range(min(d['user'].size, 3000)):
            a, b = d['indptr'][i], d['indptr'][i + 1]
            it, c = d['items'][a:b], d['clicked'][a:b].astype(bool)
            assert c.sum() == 1 and b - a >= 15
            u, t = d['user'][i], d['time'][i]
            click = it[c][0]
            want = items[indptr[u] + t] if kind == 'train' else targets[u]
            assert click == want                                              # the next read / the target
            assert (labels[it] >= 0).all()
            earlier = set(labels[items[indptr[u]:indptr[u] + t]].tolist()) - {labels[click]}
            if earlier:
                n_other += (~c).sum()
                n_same_other += np.isin(labels[it[~c]], list(earlier)).sum()
    # about half of the distractors come from the user's other earlier classes (plus the catalogue's share of those classes)
    frac = n_same_other / n_other
    assert 0.5 < frac < 0.75, frac
    # popularity: clicked and shown-not-clicked articles are about equally popular
    pop = np.bincount(items, minlength=labels.size)
    c = tr['clicked'].astype(bool)
    r = np.median(pop[tr['items'][c]]) / np.median(pop[tr['items'][~c]])
    assert 0.5 < r < 2.0, r
    again = make_impressions(indptr, items, labels, targets, shown=20, seed=3)
    assert all(np.array_equal(again[0][k], train[k]) for k in train)


def test_prefix_histories_by_hand():
    indptr = np.array([0, 4, 4, 6], np.int64)
    items = np.array([3, 1, 3, 0, 5, 2], np.int32)
    imp = _imp([0, 0, 2, 1, 2], [0, 3, 1, 0, 2], [[1, 2], [0, 4], [1, 3], [2, 6], [0, 1]], [[1, 0]] * 5)
    m = prefix_histories((indptr, items), imp, 7)
    assert m.shape == (5, 7)
    d = m.toarray()
    assert not d[0].any() and not d[3].any()
    assert np.flatnonzero(d[1]).tolist() == [1, 3] and (d[1][[1, 3]] == 1).all()        # reads 3, 1, 3: 3 counted once
    assert np.flatnonzero(d[2]).tolist() == [5] and np.flatnonzero(d[4]).tolist() == [2, 5]
    assert items.tolist() == [3, 1, 3, 0, 5, 2]


BAD_CALLS = [
    ('dae_impression_rank_loss', (None, 4, None, 4, 4, None, 1, None, None, None, 1.0, None, 4, None, None)),
    ('dae_impression_rank_loss', (8, 4, 8, 4, 4, 8, 0, 8, 8, 8, 1.0, 8, 4, 8, None)),       # no positions
    ('dae_impression_rank_loss', (8, 3, 8, 4, 4, 8, 1, 8, 8, 8, 1.0, 8, 4, 8, None)),       # ld_h < H
    ('dae_impression_metrics', (None, 4, None, 4, 4, 0, None, None, None, 1, None, None, None)),
    ('dae_impression_metrics', (8, 4, 8, 4, 4, 2, 8, 8, 8, 1, 8, 8, None)),                 # cosine flag not 0 / 1
    ('dae_impression_metrics', (8, 4, 8, 4, 0, 0, 8, 8, 8, 1, 8, 8, None)),                 # H = 0
]


@pytest.mark.parametrize('name,args', BAD_CALLS, ids=['%s_%d' % (b[0], i) for i, b in enumerate(BAD_CALLS)])
def test_export_argument_checks(name, args):
    """Fake non-NULL pointers: the checks reject the call before any CUDA call."""
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match=name):
        _cabi.call(name, *args)


def test_cli_flag_validation(tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    base = ['--model_name', 'x', '--synthetic', '100', '--top_k', '5']
    np.savez(tmp_path / 'i.npz', **_imp([0], [1], [[1, 2]], [[1, 0]]))
    for flag in ('--user_impressions', '--user_test_impressions'):
        with pytest.raises(AssertionError, match='needs --user_sequences'):
            cli.check_flags(cli.build_parser().parse_args(base + [flag, str(tmp_path / 'i.npz')]))
        with pytest.raises(AssertionError, match='no such file'):
            cli.check_flags(cli.build_parser().parse_args(base + ['--user_sequences', str(tmp_path / 'i.npz'), flag,
                                                                   str(tmp_path / 'nope.npz')]))
    F = cli.check_flags(cli.build_parser().parse_args(base + ['--user_sequences', str(tmp_path / 'i.npz'), '--user_test_impressions',
                                                               str(tmp_path / 'i.npz')]))
    seqs = (np.array([0, 3], np.int64), np.array([0, 1, 2], np.int32), None)
    train, test = cli.load_user_impressions(F, 10, seqs)
    assert train is None and test['user'].tolist() == [0]
    with pytest.raises(ValueError, match='outside'):
        cli.load_user_impressions(F, 2, seqs)
    with pytest.raises(ValueError, match='time'):
        cli.load_user_impressions(F, 10, (np.array([0, 0], np.int64), np.zeros(0, np.int32), None))
