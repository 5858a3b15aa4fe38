"""Long top-k lists (k up to 1024: dae_similarity_topk_bound_bf16x3 / _collect_bf16x3 / _select, top_k_similar(long_lists=True),
recommend(long_lists=True)): bit for bit against the register kernels at k <= 32, against the exact lexsort oracle on integer
data, and against fp64 on random data."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from topk_groups_oracle import grouped_top_k
from test_gpu_topk import _check_fp64, _fp64_scores

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tks(x, k, **kw):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    kw.setdefault('metric', 'linear kernel')
    return top_k_similar(x, k=k, long_lists=True, **kw)


def _oracle(s, k, allowed=None, groups=None):
    return grouped_top_k(s, np.arange(s.shape[1]) if groups is None else groups, k, allowed)


def _ints(n, h, lo, hi, seed):
    return np.random.default_rng(seed).integers(lo, hi + 1, (n, h)).astype(np.float32)


def _lists(nq, nc, per_row, seed):
    rng = np.random.default_rng(seed)
    m = sp.random(nq, nc, density=per_row / nc, format='csr', random_state=rng)
    return m


@pytest.mark.parametrize('k', [1, 10, 32])
@pytest.mark.parametrize('mode', ['plain', 'excl', 'groups'])
@pytest.mark.parametrize('self_mode', [True, False])
def test_stages_equal_register_kernels(k, mode, self_mode, monkeypatch):
    from dae_rnn_news_recommendation_b200 import helpers
    x = _ints(700, 16, -2, 2, 1)          # many ties, across tiles and splits
    corpus = None if self_mode else _ints(900, 16, -2, 2, 2)
    nc = 700 if self_mode else 900
    kw = {}
    if mode in ('excl', 'groups'):
        kw['exclude'] = _lists(700, nc, 30, 3)
    if mode == 'groups':
        kw['groups'] = np.random.default_rng(4).integers(0, nc // 3, nc)
    ref = _tks(x, k, corpus=corpus, **kw)
    monkeypatch.setattr(helpers, 'TOPK_MAX_K', 0)   # every k through the three stages
    got = _tks(x, k, corpus=corpus, **kw)
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])


def test_prefix_property():
    x = np.random.default_rng(5).standard_normal((3000, 32)).astype(np.float32)
    i32, v32 = _tks(x, 32, metric='cosine')
    i100, v100 = _tks(x, 100, metric='cosine')
    i1024, v1024 = _tks(x, 1024, metric='cosine')
    assert np.array_equal(i1024[:, :32], i32) and np.array_equal(v1024[:, :32], v32)
    assert np.array_equal(i100[:, :32], i32) and np.array_equal(v100[:, :32], v32)
    assert np.array_equal(i1024[:, :100], i100) and np.array_equal(v1024[:, :100], v100)


@pytest.mark.parametrize('k', [33, 100, 1024])
@pytest.mark.parametrize('self_mode', [True, False])
def test_exact_scores_against_oracle(k, self_mode):
    x = _ints(600, 8, -2, 2, 6)
    c = x if self_mode else _ints(1500, 8, -2, 2, 7)
    s = x.astype(np.float64) @ c.astype(np.float64).T
    allowed = ~np.eye(600, dtype=bool) if self_mode else None
    idx, val = _tks(x, k, corpus=None if self_mode else c)
    ref = _oracle(s, k, allowed)
    assert np.array_equal(idx, ref[0]) and np.array_equal(val, ref[1])


@pytest.mark.parametrize('k', [100, 1000])
def test_random_against_fp64(k):
    rng = np.random.default_rng(8)
    q = rng.standard_normal((500, 64)).astype(np.float32)
    c = rng.standard_normal((5000, 64)).astype(np.float32)
    idx, val = _tks(q, k, corpus=c, metric='cosine')
    _check_fp64(idx, val, _fp64_scores(q, c, 'cosine'), k)


def test_exclusion_lists():
    nq, nc, k = 300, 6000, 100
    x = _ints(nq, 8, -2, 2, 9)
    c = _ints(nc, 8, -2, 2, 10)
    s = x.astype(np.float64) @ c.astype(np.float64).T
    rows, cols = [], []
    edges = [127, 128, 255, 256, 383, 384, 5999]
    for r in range(0, nq, 3):                      # tile-boundary columns
        rows += [r] * len(edges); cols += edges
    rows += [1] * 5000; cols += list(np.random.default_rng(11).choice(nc, 5000, replace=False))   # longer than k
    rows += [2] * nc; cols += list(range(nc))      # the whole corpus: all padding
    ex = sp.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(nq, nc))
    allowed = ~(ex.toarray() > 0)
    idx, val = _tks(x, k, corpus=c, exclude=ex)
    ref = _oracle(s, k, allowed)
    assert np.array_equal(idx, ref[0]) and np.array_equal(val, ref[1])
    assert (idx[2] == -1).all() and (val[2] == -np.inf).all()
    empty = _tks(x, k, corpus=c, exclude=sp.csr_matrix((nq, nc)))
    plain = _tks(x, k, corpus=c)
    assert np.array_equal(empty[0], plain[0]) and np.array_equal(empty[1], plain[1])


def test_groups():
    nq, nc, k = 300, 4000, 100
    x = _ints(nq, 8, -2, 2, 12)
    c = _ints(nc, 8, -2, 2, 13)
    s = x.astype(np.float64) @ c.astype(np.float64).T
    g = np.random.default_rng(14).permutation(np.arange(nc) // 21)   # stories of about 21 members
    idx, val = _tks(x, k, corpus=c, groups=g)
    ref = _oracle(s, k, groups=g)
    assert np.array_equal(idx, ref[0]) and np.array_equal(val, ref[1])
    same = _tks(x, k, corpus=c, groups=np.arange(nc))
    plain = _tks(x, k, corpus=c)
    assert np.array_equal(same[0], plain[0]) and np.array_equal(same[1], plain[1])
    ex = _lists(nq, nc, 200, 15)
    idx, val = _tks(x, k, corpus=c, groups=g, exclude=ex)
    ref = _oracle(s, k, ex.toarray() == 0, groups=g)
    assert np.array_equal(idx, ref[0]) and np.array_equal(val, ref[1])


def test_all_equal_scores_and_a_small_budget(monkeypatch):
    from dae_rnn_news_recommendation_b200 import helpers
    n, k = 2000, 100
    x = np.ones((n, 8), np.float32)                 # every column is a candidate of every row
    idx, val = _tks(x, k)
    ref = _oracle(np.full((n, n), 8.0), k, ~np.eye(n, dtype=bool))
    assert np.array_equal(idx, ref[0]) and np.array_equal(val, ref[1])
    calls = []
    real = helpers.call

    def spy(name, *args):
        calls.append(name)
        return real(name, *args)
    monkeypatch.setattr(helpers, 'call', spy)
    small = _tks(x, k, max_candidates=3 * n)       # 3 rows' candidates: every chunk overflows and is collected again
    assert np.array_equal(small[0], idx) and np.array_equal(small[1], val)
    assert calls.count('dae_similarity_topk_collect_bf16x3') > calls.count('dae_similarity_topk_bound_bf16x3') > 1
    y = np.random.default_rng(16).standard_normal((n, 16)).astype(np.float32)
    full = _tks(y, 300, metric='cosine')
    chunked = _tks(y, 300, metric='cosine', max_candidates=n)
    assert np.array_equal(full[0], chunked[0]) and np.array_equal(full[1], chunked[1])


def test_splits_do_not_change_the_result():
    x = _ints(800, 16, -2, 2, 17)
    ref = _tks(x, 200)
    for s in (1, 3, 32):
        got = _tks(x, 200, splits=s)
        assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])


def test_scale_sampled_rows_and_peak_memory():
    """100 000 x 100 000, H = 500, k = 1000: sampled rows against fp64; device memory above the inputs and the output stays under
    the budget's bound (36 B per candidate, the bound workspace, the sort's scratch)."""
    import torch
    from dae_rnn_news_recommendation_b200 import helpers
    n, h, k = 100000, 500, 1000
    rng = np.random.RandomState(0)
    labels = rng.randint(0, 4, n)
    emb = (rng.randn(4, h)[labels] * 0.15 + rng.randn(n, h)).astype(np.float32)
    x = torch.from_numpy(emb).cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    idx, val = helpers.top_k_similar(x, k=k, long_lists=True, to_host=False)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    budget = helpers.TOPK_LONG_MAX_CANDIDATES
    rows = budget // (2 * k)
    ld = (h + 7) // 8 * 8
    bound = (n * k * 8                 # the output
             + 2 * n * ld * 2          # the bf16 hi / lo operands
             + 36 * budget             # candidates and their sort
             + rows * (64 * 32 * 8 + 8) + (64 << 20))   # bound workspace, tau and counts, the sort's scratch
    assert peak <= bound, (peak, bound)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    sample = np.sort(np.random.default_rng(3).choice(n, 32, replace=False))
    s = _fp64_scores(emb[sample], emb, 'cosine')
    s[np.arange(32), sample] = -np.inf
    _check_fp64(idx[sample], val[sample], s, k)


def test_recommend_long_lists():
    from dae_rnn_news_recommendation_b200.helpers import recommend
    n_art, n_u, h = 3000, 200, 8
    emb = _ints(n_art, h, -2, 2, 18)
    prof = _ints(n_u, h, -3, 3, 19)
    rng = np.random.default_rng(20)
    hist = sp.random(n_u, n_art, density=10 / n_art, format='csr', random_state=rng)
    hist.data[:] = 1.0
    for k in (1, 20, 32):
        a = recommend(hist, emb, k=k, profiles=prof, metric='linear kernel')
        b = recommend(hist, emb, k=k, profiles=prof, metric='linear kernel', long_lists=True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    cand = np.sort(rng.choice(n_art, 2000, replace=False))
    g = rng.integers(0, 700, n_art)
    idx, val = recommend(hist, emb, k=100, profiles=prof, metric='linear kernel', candidates=cand, groups=g, long_lists=True)
    read_groups = [set(g[hist.indices[hist.indptr[u]:hist.indptr[u + 1]]].tolist()) for u in range(n_u)]
    allowed = np.array([[g[c] not in read_groups[u] for c in cand] for u in range(n_u)])
    s = prof.astype(np.float64) @ emb[cand].astype(np.float64).T
    ri, rv = _oracle(s, 100, allowed, g[cand])
    ri = np.where(ri >= 0, cand[np.maximum(ri, 0)], -1)
    empty = np.diff(hist.indptr) == 0
    ri[empty], rv[empty] = -1, -np.inf
    assert np.array_equal(idx, ri) and np.array_equal(val, rv)


def test_user_gru_recommend_passes_long_lists(monkeypatch):
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.user_model import UserGRU
    emb = np.random.default_rng(21).standard_normal((500, 16)).astype(np.float32)
    indptr = np.array([0, 3, 5], np.int64)
    items = np.array([1, 2, 3, 7, 9], np.int32)
    gru = UserGRU(16, num_epochs=1, seed=0)
    gru.fit((indptr, items), emb)
    seen = {}
    real = helpers.recommend

    def spy(*a, **kw):
        seen.update(kw)
        return real(*a, **kw)
    monkeypatch.setattr(helpers, 'recommend', spy)
    idx, val = gru.recommend((indptr, items), emb, k=100, long_lists=True)
    assert seen['long_lists'] is True and idx.shape == (2, 100)
    assert not np.isin(idx[0], [1, 2, 3]).any() and (np.diff(val, axis=1) <= 0).all()


def test_cli_long_lists_on_synthetic():
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    model = cli.main(['--model_name', 'syntkl', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size',
                      '200', '--seed', '3', '--top_k', '100', '--long_lists'])
    ev = model.evaluation
    for split, n in (('', 960), ('_validate', 240)):
        idx = np.load(model.data_dir + 'article_top_k_index%s.npy' % split)
        score = np.load(model.data_dir + 'article_top_k_score%s.npy' % split)
        assert idx.shape == (n, 100) and score.shape == (n, 100) and idx.dtype == np.int32
        assert ((idx >= 0) & (idx < 960)).all() and (np.diff(score, axis=1) <= 0).all()
        assert 0.0 <= ev['top_k_precision' + split] <= 1.0
    assert (np.load(model.data_dir + 'article_top_k_index.npy') != np.arange(960)[:, None]).all()
