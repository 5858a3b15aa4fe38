"""Exclusion lists in the dense and sparse top-k kernels (top_k_similar(exclude=...)), user_profiles, recommend and the CLI's
--user_histories, checked against NumPy on the host."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_topk import _check_fp64, _exact_top_k, _fp64_scores  # noqa: E402
from test_topk_sparse_host import f32_column_oracle  # noqa: E402


def _lists(nq, nc, seed, mean=6, extra=()):
    """Random exclusion lists plus the hand-picked positions `extra` ((row, col) pairs)."""
    rng = np.random.default_rng(seed)
    n = rng.poisson(mean, nq)
    r = np.repeat(np.arange(nq), n)
    c = rng.integers(0, nc, r.size)
    if extra:
        er, ec = zip(*extra)
        r, c = np.concatenate([r, er]), np.concatenate([c, ec])
    return sp.csr_matrix((np.ones(r.size, np.float32), (r, c)), shape=(nq, nc))


def _masked(s, ex):
    s = s.copy()
    coo = ex.tocoo()
    s[coo.row, coo.col] = -np.inf
    return s


def _boundary_extra(nq, nc, step):
    """Positions on and next to multiples of `step` (tile or range boundaries) for a spread of rows."""
    out = []
    for i in range(0, nq, 3):
        for b in range(step, nc, step):
            out += [(i, b - 1), (i, b)]
    return out


@pytest.mark.parametrize('k', [1, 10, 32])
def test_dense_exact_ties_and_lists(k):
    """Small-integer embeddings: every score is exact in bf16x3, so ties are real.  Lists hit tied columns and the columns on both
    sides of every 128-column tile boundary; the answer must equal the NumPy (score desc, index asc) order with the listed entries
    at -inf, bit for bit."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(1)
    q = rng.integers(-2, 3, (300, 24)).astype(np.float32)
    c = rng.integers(-2, 3, (777, 24)).astype(np.float32)
    c[100:140] = c[100]                                   # a block of tied corpus rows across the boundary at 128
    s = q.astype(np.float64) @ c.T.astype(np.float64)
    extra = _boundary_extra(300, 777, 128) + [(i, j) for i in range(0, 300, 2) for j in range(100, 140, 3)]
    ex = _lists(300, 777, 2, extra=extra)
    want = _exact_top_k(_masked(s, ex), k)
    for splits in (0, 1, 2, 7):
        idx, val = top_k_similar(q, k=k, corpus=c, metric='linear kernel', exclude=ex, splits=splits)
        assert np.array_equal(idx, want[0]) and np.array_equal(val, want[1])


@pytest.mark.parametrize('metric', ['cosine', 'linear kernel'])
def test_dense_random_against_fp64(metric):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(3)
    q = rng.standard_normal((700, 100)).astype(np.float32)
    c = rng.standard_normal((2100, 100)).astype(np.float32)
    ex = _lists(700, 2100, 4, mean=40)
    idx, val = top_k_similar(q, k=16, corpus=c, metric=metric, exclude=ex)
    _check_fp64(idx, val, _masked(_fp64_scores(q, c, metric), ex), 16)


def _sparse_data(n, f, seed):
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    return make_sparse(n, f, mean_nnz=20, kind='tfidf', seed=seed).astype(np.float32)


@pytest.mark.parametrize('k', [1, 10, 32])
def test_sparse_bit_exact_with_lists(k):
    """Corpus of 4 500 rows (ranges of 2048): lists on both sides of the range boundaries; bit-exact against the float32 column
    oracle with the lists applied, for every split count."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    c = _sparse_data(4500, 600, 5)
    q = _sparse_data(300, 600, 6)
    ex = _lists(300, 4500, 7, mean=30, extra=_boundary_extra(300, 4500, 2048))
    want = _exact_top_k(_masked(f32_column_oracle(q, c).astype(np.float64), ex), k)
    for splits in (0, 1, 2, 3):
        idx, val = top_k_similar(q, k=k, corpus=c, metric='linear kernel', exclude=ex, splits=splits)
        assert np.array_equal(idx, want[0]) and np.array_equal(val.view(np.int32), want[1].view(np.int32))


def test_empty_lists_are_bit_identical_to_no_exclusion():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(8)
    x = rng.standard_normal((1000, 64)).astype(np.float32)
    none = sp.csr_matrix((1000, 1000), dtype=np.float32)
    for corpus in (None, x[:700]):
        ex = none if corpus is None else sp.csr_matrix((1000, 700), dtype=np.float32)
        a = top_k_similar(x, k=10, corpus=corpus)
        b = top_k_similar(x, k=10, corpus=corpus, exclude=ex)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int32), b[1].view(np.int32))
    xs = _sparse_data(3000, 400, 9)
    a = top_k_similar(xs, k=10)
    b = top_k_similar(xs, k=10, exclude=sp.csr_matrix((3000, 3000), dtype=np.float32))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int32), b[1].view(np.int32))


def test_self_mode_combined_with_lists_and_split_invariance():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(10)
    x = rng.integers(-3, 4, (900, 16)).astype(np.float32)
    ex = _lists(900, 900, 11, mean=20, extra=_boundary_extra(900, 900, 128))
    s = x.astype(np.float64) @ x.T.astype(np.float64)
    np.fill_diagonal(s, -np.inf)
    want = _exact_top_k(_masked(s, ex), 12)
    for splits in (1, 2, 7, 0):
        idx, val = top_k_similar(x, k=12, metric='linear kernel', exclude=ex, splits=splits)
        assert np.array_equal(idx, want[0]) and np.array_equal(val, want[1])
    xs = _sparse_data(2500, 300, 12)
    ex = _lists(2500, 2500, 13, mean=10)
    s = f32_column_oracle(xs, xs).astype(np.float64)
    np.fill_diagonal(s, -np.inf)
    want = _exact_top_k(_masked(s, ex), 12)
    for splits in (1, 2, 7, 0):
        idx, val = top_k_similar(xs, k=12, metric='linear kernel', exclude=ex, splits=splits)
        assert np.array_equal(idx, want[0]) and np.array_equal(val.view(np.int32), want[1].view(np.int32))


def test_lists_that_leave_fewer_than_k_or_none_give_padding():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(14)
    q = rng.standard_normal((5, 32)).astype(np.float32)
    c = rng.standard_normal((300, 32)).astype(np.float32)
    rows = [np.arange(300), np.arange(296), np.array([5, 6]), np.arange(0, 300, 2), np.array([], int)]
    ex = sp.csr_matrix((np.ones(sum(map(len, rows))), (np.repeat(np.arange(5), list(map(len, rows))), np.concatenate(rows))),
                       shape=(5, 300))
    for data, corpus in ((q, c), (sp.csr_matrix(q), sp.csr_matrix(c))):
        idx, val = top_k_similar(data, k=10, corpus=corpus, metric='linear kernel', exclude=ex)
        assert (idx[0] == -1).all() and (val[0] == -np.inf).all()
        assert (idx[1, :4] >= 296).all() and (idx[1, 4:] == -1).all() and (val[1, 4:] == -np.inf).all()
        assert not np.isin(idx[2], [5, 6]).any() and (idx[3] % 2 == 1).all() and (idx[4] >= 0).all()


def test_a_user_with_5000_reads():
    from dae_rnn_news_recommendation_b200.helpers import recommend
    rng = np.random.default_rng(15)
    emb = rng.standard_normal((20000, 48)).astype(np.float32)
    read = np.sort(rng.choice(20000, 5000, replace=False))
    h = sp.csr_matrix((np.ones(5003), (np.r_[np.zeros(5000, int), 1, 1, 1], np.r_[read, 1, 2, 3])), shape=(2, 20000))
    idx, val = recommend(h, emb, k=32)
    prof = np.stack([emb[read].astype(np.float64).mean(0), emb[1:4].astype(np.float64).mean(0)])
    s = _fp64_scores(prof, emb, 'cosine')
    s[0, read] = -np.inf
    s[1, 1:4] = -np.inf
    _check_fp64(idx, val, s, 32)
    assert not np.isin(idx[0], read).any()


def test_user_profiles_against_fp64():
    from dae_rnn_news_recommendation_b200.helpers import user_profiles
    rng = np.random.default_rng(16)
    emb = rng.standard_normal((3000, 500)).astype(np.float32)
    h = sp.random(400, 3000, density=0.01, format='csr', random_state=17, dtype=np.float64)
    h.data = rng.random(h.nnz) + 0.1                     # recency-like weights
    c = h.tocoo()
    keep = (c.row != 5) & (c.row != 7)                   # user 5 reads nothing; user 7 one article with an explicit zero weight
    h = sp.coo_matrix((np.r_[c.data[keep], 0.0], (np.r_[c.row[keep], 7], np.r_[c.col[keep], 10])), shape=h.shape).tocsr()
    assert h.nnz == keep.sum() + 1
    got = user_profiles(h, emb)
    hd = h.toarray()
    tot = hd.sum(1, keepdims=True)
    want = np.where(tot > 0, hd / np.where(tot > 0, tot, 1.0), 0.0) @ emb.astype(np.float64)
    assert got.shape == (400, 500) and got.dtype == np.float32
    err = np.linalg.norm(got - want, axis=1)
    assert (err <= 1e-5 * np.maximum(np.linalg.norm(want, axis=1), 1e-30)).all()
    assert (got[5] == 0).all() and (got[7] == 0).all()


def test_recommend_never_returns_a_read_article():
    from dae_rnn_news_recommendation_b200.helpers import recommend
    from dae_rnn_news_recommendation_b200.synth import make_histories
    rng = np.random.default_rng(18)
    labels = rng.integers(0, 5, 6000)
    emb = (rng.standard_normal((5, 64))[labels] + 0.8 * rng.standard_normal((6000, 64))).astype(np.float32)
    h, _ = make_histories(2000, labels, mean_len=30, seed=19, holdout=False)
    h = sp.vstack([h, sp.csr_matrix((2, 6000), dtype=np.float32)]).tocsr()      # two users without reads
    hd = h.toarray() > 0
    idx, val = recommend(h, emb, k=10)
    assert (idx[-2:] == -1).all() and (val[-2:] == -np.inf).all()
    v = idx[:-2] >= 0
    assert v.all() and not np.take_along_axis(hd[:-2], idx[:-2], 1).any()
    cand = np.sort(rng.choice(6000, 1500, replace=False))
    idx, val = recommend(h, emb, k=10, candidates=cand)
    ok = idx[:-2] >= 0
    assert np.isin(idx[:-2][ok], cand).all()
    assert not np.take_along_axis(hd[:-2], np.where(ok, idx[:-2], 0), 1)[ok].any()
    # with candidates: the same as ranking the candidate rows directly with the remapped lists
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar, user_profiles
    prof = user_profiles(h, emb)
    ex = sp.csr_matrix(h[:, cand])
    i2, v2 = top_k_similar(prof, k=10, corpus=emb[cand], exclude=ex)
    i2 = np.where(i2 >= 0, cand[np.maximum(i2, 0)], -1)
    assert np.array_equal(idx[:-2], i2[:-2]) and np.array_equal(val[:-2], v2[:-2])
    idx_all, _ = recommend(h, emb, k=10, exclude_read=False)
    assert np.take_along_axis(hd[:-2], idx_all[:-2], 1).any()   # without exclusion the read articles do come back


def test_hit_rate_well_above_random():
    from dae_rnn_news_recommendation_b200.helpers import recommend, recommendation_recall
    from dae_rnn_news_recommendation_b200.synth import make_histories
    rng = np.random.default_rng(20)
    n, k = 20000, 10
    labels = rng.integers(0, 20, n)
    emb = (rng.standard_normal((20, 128))[labels] + 0.7 * rng.standard_normal((n, 128))).astype(np.float32)
    h, t = make_histories(5000, labels, mean_len=20, seed=21)
    idx, _ = recommend(h, emb, k=k)
    r = recommendation_recall(idx, t)
    assert r['users'] == 5000
    random_rate = k * 1 / n
    assert r['hit_rate'] > 5 * random_rate and r['recall'] == r['hit_rate']


def test_sampled_rows_at_100k_articles_and_100k_users():
    import torch
    from dae_rnn_news_recommendation_b200.helpers import recommend
    from dae_rnn_news_recommendation_b200.synth import make_histories
    rng = np.random.default_rng(22)
    n, h_dim = 100000, 500
    labels = rng.integers(0, 50, n)
    emb = (rng.standard_normal((50, h_dim))[labels] * 0.3 + rng.standard_normal((n, h_dim))).astype(np.float32)
    h, _ = make_histories(100000, labels, mean_len=20, seed=23, holdout=False)
    idx, val = recommend(h, torch.from_numpy(emb).cuda(), k=10)
    rows = rng.choice(100000, 64, replace=False)
    hs = h[rows]
    hd = hs.toarray()
    prof = (hd / np.maximum(hd.sum(1, keepdims=True), 1e-300)) @ emb.astype(np.float64)
    s = _fp64_scores(prof, emb, 'cosine')
    s[hd > 0] = -np.inf
    _check_fp64(idx[rows], val[rows], s, 10)


def test_cli_user_histories_on_synthetic(capsys, tmp_path):
    import re
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.helpers import recommendation_recall
    from dae_rnn_news_recommendation_b200.synth import make_histories
    argv = ['--model_name', 'synusers', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--top_k', '5']
    trX, _, trL, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    h, t = make_histories(300, trL, mean_len=8, seed=4)
    sp.save_npz(tmp_path / 'h.npz', h)
    sp.save_npz(tmp_path / 't.npz', t)
    model = cli.main(argv + ['--user_histories', str(tmp_path / 'h.npz'), '--user_targets', str(tmp_path / 't.npz')])
    printed = capsys.readouterr().out
    idx = np.load(model.data_dir + 'user_top_k_index.npy')
    score = np.load(model.data_dir + 'user_top_k_score.npy')
    assert idx.shape == score.shape == (300, 5) and idx.dtype == np.int32
    r = recommendation_recall(idx, t)
    ev = model.evaluation
    assert ev['user_hit_rate'] == r['hit_rate'] and ev['user_recall'] == r['recall']
    m = re.search(r'users: hit rate@5 ([0-9.]+) recall@5 ([0-9.]+) \((\d+) users with targets\)', printed)
    assert m and m.group(1) == '%.4f' % r['hit_rate'] and int(m.group(3)) == r['users']
    assert not np.take_along_axis(h.toarray() > 0, np.maximum(idx, 0), 1)[idx >= 0].any()
