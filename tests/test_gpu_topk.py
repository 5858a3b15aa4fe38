"""top_k_similar / dae_similarity_topk_bf16x3: the k most similar corpus rows per query, checked against fp64 NumPy on the host."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fp64_scores(q, c, metric):
    q, c = np.asarray(q, np.float64), np.asarray(c, np.float64)
    if metric == 'cosine':   # all-zero rows stay zero (sklearn.preprocessing.normalize)
        q = q / np.where((nq := np.linalg.norm(q, axis=1, keepdims=True)) > 0, nq, 1.0)
        c = c / np.where((nc := np.linalg.norm(c, axis=1, keepdims=True)) > 0, nc, 1.0)
    return q @ c.T


def _exclude(s, offset):
    s = s.copy()
    r = np.arange(s.shape[0])
    col = r + offset
    ok = (col >= 0) & (col < s.shape[1])
    s[r[ok], col[ok]] = -np.inf
    return s


def _exact_top_k(s, k):
    """(score desc, index asc) order of an exactly known score matrix; excluded entries are -inf."""
    nq, nc = s.shape
    order = np.lexsort((np.broadcast_to(np.arange(nc), s.shape), -s), axis=1)[:, :k]
    val = np.take_along_axis(s, order, 1)
    idx = np.where(np.isfinite(val), order, -1)
    if k > nc:
        idx = np.concatenate([idx, np.full((nq, k - nc), -1)], 1)
        val = np.concatenate([val, np.full((nq, k - nc), -np.inf)], 1)
    return idx.astype(np.int32), val.astype(np.float32)


def _check_fp64(idx, val, s, k, tol=2e-5, boundary=4e-5):
    """s: fp64 scores with excluded entries at -inf.  Scores within `tol` of fp64; the returned set is the fp64 top k except for
    entries within `boundary` of the fp64 k-th score; order non-increasing; padding -1 / -inf exactly where candidates run out."""
    nq, nc = s.shape
    assert idx.shape == (nq, k) and val.shape == (nq, k) and idx.dtype == np.int32 and val.dtype == np.float32
    finite = np.isfinite(s)
    scale = max(1.0, np.abs(s[finite]).max())
    tol, boundary = tol * scale, boundary * scale
    n_cand = finite.sum(1)
    valid = idx >= 0
    assert (valid.sum(1) == np.minimum(k, n_cand)).all()
    assert (valid[:, :-1] >= valid[:, 1:]).all()                           # padding only at the end
    assert (val[~valid] == -np.inf).all()
    got = np.take_along_axis(s, np.where(valid, idx, 0), 1)
    assert np.isfinite(got[valid]).all()                                   # no excluded column, no column >= Nc
    assert np.abs(val[valid] - got[valid]).max() <= tol
    for i in range(nq):
        assert len(set(idx[i][valid[i]].tolist())) == valid[i].sum()
    vv = np.where(valid, val, -np.inf)
    assert (vv[:, :-1] >= vv[:, 1:]).all()
    kk = np.minimum(k, n_cand)
    srt = -np.sort(-s, axis=1)
    kth = srt[np.arange(nq), np.maximum(kk - 1, 0)]
    rows = kk > 0
    assert (got[rows] >= np.where(valid[rows], kth[rows, None] - boundary, -np.inf)).all()
    must = (s > kth[:, None] + boundary).sum(1)
    have = ((got > kth[:, None] + boundary) & valid).sum(1)
    assert (must[rows] == have[rows]).all()


def _ops(x, metric='linear kernel'):
    import torch
    from dae_rnn_news_recommendation_b200 import helpers
    t = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    return helpers._normalised_operands(t, 2 if metric == 'cosine' else 0)[:2]


@pytest.mark.parametrize('k', [1, 7, 32])
def test_exact_ties_and_order(k):
    """Small integers: every bf16x3 product and fp32 sum is exact, so scores tie for real and the answer is known exactly."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(5)
    x = rng.integers(-2, 3, size=(700, 64)).astype(np.float32)
    y = rng.integers(-2, 3, size=(450, 64)).astype(np.float32)
    s = (x.astype(np.int64) @ x.T.astype(np.int64)).astype(np.float64)
    for got, want in ((top_k_similar(x, k=k, metric='linear kernel'), _exact_top_k(_exclude(s, 0), k)),
                      (top_k_similar(y, k=k, corpus=x, metric='linear kernel'),
                       _exact_top_k((y.astype(np.int64) @ x.T.astype(np.int64)).astype(np.float64), k))):
        assert np.array_equal(got[0], want[0])
        assert np.array_equal(got[1], want[1])


@pytest.mark.parametrize('metric', ['cosine', 'linear kernel'])
@pytest.mark.parametrize('k', [1, 10, 32])
@pytest.mark.parametrize('h', [37, 500, 1000])
def test_random_against_fp64(h, k, metric):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(h * 100 + k)
    c = (rng.random((1300, h)) - 0.4).astype(np.float32)
    q = (rng.random((333, h)) - 0.4).astype(np.float32)
    c[[3, 700, 1299]] = 0.0                         # all-zero rows in the corpus and among the queries
    q[[0, 200]] = 0.0
    idx, val = top_k_similar(c, k=k, metric=metric)
    _check_fp64(idx, val, _exclude(_fp64_scores(c, c, metric), 0), k)
    assert (idx != np.arange(1300)[:, None]).all()
    idx, val = top_k_similar(q, k=k, corpus=c, metric=metric)
    _check_fp64(idx, val, _fp64_scores(q, c, metric), k)


@pytest.mark.parametrize('k', [10, 32])
def test_splits_do_not_change_the_result(k):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(7)
    labels = rng.integers(0, 4, 3000)
    x = (rng.normal(size=(4, 200))[labels] * 0.3 + rng.normal(size=(3000, 200))).astype(np.float32)
    x[100:110] = x[90]                               # duplicate rows: exactly tied scores across column ranges
    for corpus, q in ((None, x), (x, x[:1000])):
        ref = top_k_similar(q, k=k, corpus=corpus, splits=1)
        for splits in (2, 7, 0):
            got = top_k_similar(q, k=k, corpus=corpus, splits=splits)
            assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), splits
        _check_fp64(ref[0], ref[1], _fp64_scores(q, x, 'cosine') if corpus is not None else _exclude(_fp64_scores(x, x, 'cosine'), 0), k)


def test_validation_against_training_corpus():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(11)
    train = rng.normal(size=(8000, 100)).astype(np.float32)
    val_set = rng.normal(size=(2000, 100)).astype(np.float32)
    idx, val = top_k_similar(val_set, k=10, corpus=train)
    _check_fp64(idx, val, _fp64_scores(val_set, train, 'cosine'), 10)


def test_row_window_excludes_the_diagonal_at_an_offset():
    import torch
    from dae_rnn_news_recommendation_b200 import helpers
    rng = np.random.default_rng(13)
    x = rng.normal(size=(2000, 96)).astype(np.float32)
    hi, lo = _ops(x, 'cosine')
    r0, r1 = 500, 1177
    idx, val = helpers._similarity_topk((hi[r0:r1], lo[r0:r1]), (hi, lo), r1 - r0, 2000, 96, 10, diag_offset=r0, exclude=True)
    torch.cuda.synchronize()
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    assert (idx != np.arange(r0, r1)[:, None]).all()
    _check_fp64(idx, val, _exclude(_fp64_scores(x[r0:r1], x, 'cosine'), r0), 10)


def test_fewer_candidates_than_k_are_padded():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(17)
    c = rng.normal(size=(5, 40)).astype(np.float32)
    q = rng.normal(size=(9, 40)).astype(np.float32)
    idx, val = top_k_similar(q, k=10, corpus=c)
    assert (idx[:, 5:] == -1).all() and (val[:, 5:] == -np.inf).all()
    _check_fp64(idx, val, _fp64_scores(q, c, 'cosine'), 10)
    idx, val = top_k_similar(c, k=10)                # self: 4 candidates per row
    assert (idx[:, 4:] == -1).all() and (val[:, 4:] == -np.inf).all()
    _check_fp64(idx, val, _exclude(_fp64_scores(c, c, 'cosine'), 0), 10)


def test_k1_agrees_with_nearest_neighbors():
    """The data and tolerance of test_gpu_similarity.test_sparse_matches_sklearn_and_nearest_neighbors."""
    from sklearn.metrics import pairwise
    from dae_rnn_news_recommendation_b200.helpers import nearest_neighbors, top_k_similar
    rng = np.random.default_rng(1)
    e = rng.normal(size=(1500, 64)).astype(np.float32)
    sim = pairwise.cosine_similarity(e.astype(np.float64))
    np.fill_diagonal(sim, -np.inf)
    idx, val = top_k_similar(e, k=1)
    assert idx.shape == (1500, 1)
    assert (idx[:, 0] == sim.argmax(1)).mean() > 0.999 and np.allclose(val[:, 0], sim.max(1), atol=2e-5)
    nn_idx, nn_val = nearest_neighbors(e, chunk=512)
    assert (idx[:, 0] == nn_idx).mean() > 0.999 and np.allclose(val[:, 0], nn_val, atol=2e-5)


def test_full_size_sampled_rows():
    """C2's 100 000 articles, H = 500, k = 10: 64 sampled query rows against fp64."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    n, h = 100000, 500
    rng = np.random.RandomState(0)
    labels = rng.randint(0, 4, n)
    emb = (rng.randn(4, h)[labels] * 0.15 + rng.randn(n, h)).astype(np.float32)
    idx, val = top_k_similar(emb, k=10)
    rows = np.sort(np.random.default_rng(3).choice(n, 64, replace=False))
    s = _fp64_scores(emb[rows], emb, 'cosine')
    s[np.arange(64), rows] = -np.inf
    _check_fp64(idx[rows], val[rows], s, 10)


def test_cli_top_k_on_synthetic():
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    model = cli.main(['--model_name', 'syntk', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size',
                      '200', '--seed', '3', '--top_k', '5'])
    ev = model.evaluation
    for split, n in (('', 960), ('_validate', 240)):
        idx = np.load(model.data_dir + 'article_top_k_index%s.npy' % split)
        score = np.load(model.data_dir + 'article_top_k_score%s.npy' % split)
        assert idx.shape == (n, 5) and score.shape == (n, 5) and idx.dtype == np.int32
        assert ((idx >= 0) & (idx < 960)).all() and (score <= 1.0 + 1e-5).all()
        assert np.array_equal(ev['top_k' + split][0], idx)
        assert 0.0 <= ev['top_k_precision' + split] <= 1.0
    assert (np.load(model.data_dir + 'article_top_k_index.npy') != np.arange(960)[:, None]).all()
