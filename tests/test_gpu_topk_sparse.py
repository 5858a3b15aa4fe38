"""top_k_similar on scipy sparse inputs / dae_csr_similarity_topk: the k most similar corpus rows of bag-of-words vectors, checked
bit for bit against the float32 column-ordered oracle, exactly on integer overlaps, and against fp64."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from test_gpu_topk import _check_fp64, _exact_top_k, _exclude
from test_topk_sparse_host import f32_column_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _binary(n, f, density, seed):
    m = sp.random(n, f, density=density, format='csr', dtype=np.float32, random_state=seed)
    m.data[:] = 1.0
    return m


def _tfidf_like(n, f, seed):
    """synth.make_sparse rows (Zipf columns) plus hand-made ones: empty rows, a single-entry row, a column present in every row,
    a row with every column, negative values."""
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    m = make_sparse(n, f, mean_nnz=25, kind='tfidf', seed=seed).tolil()
    rng = np.random.default_rng(seed)
    m[:, 3] = rng.random((n, 1)).astype(np.float32) * 0.5 + 0.01                  # column 3 in every row
    m[7, :] = 0.0                                                                # empty rows (the every-row column too)
    m[n - 2, :] = 0.0
    m[11, :] = 0.0
    m[11, f - 1] = 0.75                                                          # a single entry
    m[13, :] = (rng.random((1, f)) - 0.5).astype(np.float32)                   # every column, half of them negative
    m = m.tocsr()
    neg = rng.random(m.nnz) < 0.1
    m.data[neg] *= -1.0
    m.eliminate_zeros()
    m.sort_indices()
    return m.astype(np.float32)


def _expected(q, c, k, exclude):
    s = f32_column_oracle(q, c).astype(np.float64)
    return _exact_top_k(_exclude(s, 0) if exclude else s, k)


@pytest.mark.parametrize('k', [1, 7, 32])
def test_exact_ties_binary_linear_kernel(k):
    """Binary rows: every score is a small integer overlap, so ties are real and the answer is known exactly."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    x = _binary(2600, 300, 0.03, 1)
    y = _binary(700, 300, 0.03, 2)
    xi = x.astype(np.int64)
    s = (xi @ xi.T).toarray().astype(np.float64)
    got = top_k_similar(x, k=k, metric='linear kernel')
    want = _exact_top_k(_exclude(s, 0), k)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    got = top_k_similar(y, k=k, corpus=x, metric='linear kernel')
    want = _exact_top_k((y.astype(np.int64) @ xi.T).toarray().astype(np.float64), k)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize('k', [1, 10, 32])
def test_bit_exact_against_the_float32_oracle(k):
    """Corpus of 4 500 rows (two full ranges of 2048 and a partial one), 700 columns; self mode and 1 300 queries against it."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    c = _tfidf_like(4500, 700, 5)
    q = _tfidf_like(1300, 700, 6)
    for got, want in ((top_k_similar(c, k=k, metric='linear kernel'), _expected(c, c, k, True)),
                      (top_k_similar(q, k=k, corpus=c, metric='linear kernel'), _expected(q, c, k, False))):
        assert np.array_equal(got[0], want[0])
        assert np.array_equal(got[1], want[1])
    idx = top_k_similar(c, k=k, metric='linear kernel')[0]
    assert (idx[7] >= 0).all() and (idx != np.arange(4500)[:, None]).all()


def test_empty_query_rows_return_the_lowest_indices_at_zero():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    c = _tfidf_like(3000, 500, 8)
    q = sp.csr_matrix((4, 500), dtype=np.float32)
    idx, val = top_k_similar(q, k=6, corpus=c, metric='linear kernel')
    assert (idx == np.arange(6)[None, :]).all() and (val == 0.0).all()


def test_splits_do_not_change_the_result():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    c = _tfidf_like(9000, 400, 9)
    q = c[:500]
    for corpus, qq in ((None, c), (c, q)):
        ref = top_k_similar(qq, k=10, corpus=corpus, metric='linear kernel', splits=1)
        for splits in (2, 7, 0):
            got = top_k_similar(qq, k=10, corpus=corpus, metric='linear kernel', splits=splits)
            assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), splits
    want = _expected(q, c, 10, False)
    assert np.array_equal(ref[0], want[0]) and np.array_equal(ref[1], want[1])


def test_cosine_against_fp64_and_the_dense_path():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    from sklearn.metrics import pairwise
    c = _tfidf_like(3000, 600, 10)
    q = _tfidf_like(800, 600, 11)
    s_self = _exclude(pairwise.cosine_similarity(c.astype(np.float64)), 0)
    s_q = pairwise.cosine_similarity(q.astype(np.float64), c.astype(np.float64))
    for got, s, dense in ((top_k_similar(c, k=10), s_self, top_k_similar(c.toarray(), k=10)),
                          (top_k_similar(q, k=10, corpus=c), s_q, top_k_similar(q.toarray(), k=10, corpus=c.toarray()))):
        _check_fp64(got[0], got[1], s, 10)
        srt = -np.sort(-s, axis=1)
        clear = srt[:, 9] - srt[:, 10] > 1e-4        # no near-tie at the k-th place: both paths return the same set
        assert clear.mean() > 0.5
        assert (np.sort(got[0], 1) == np.sort(dense[0], 1))[clear].all()


def test_uci_c1_binary_cosine():
    """The real C1 articles (8 000 x 10 000 binary), cosine, k = 10: fp64 sklearn, and k = 1 against pairwise_similarity(sparse)."""
    from helpers import load_uci_c1
    from sklearn.metrics import pairwise
    from dae_rnn_news_recommendation_b200.helpers import pairwise_similarity, top_k_similar
    x = load_uci_c1()['train'].astype(np.float32)
    idx, val = top_k_similar(x, k=10)
    s = pairwise.cosine_similarity(x.astype(np.float64))
    np.fill_diagonal(s, -np.inf)
    _check_fp64(idx, val, s, 10)
    ps = pairwise_similarity(x, metric='cosine')
    np.fill_diagonal(ps, -np.inf)
    first = ps.argmax(1)                              # first maximum
    i1, v1 = top_k_similar(x, k=1)
    assert (i1[:, 0] == first).mean() > 0.999
    assert np.allclose(v1[:, 0], ps.max(1), atol=2e-5)
    assert np.array_equal(i1[:, 0], idx[:, 0]) and np.array_equal(v1[:, 0], val[:, 0])


@pytest.mark.parametrize('f', [10000, 50000])
def test_full_size_sampled_rows_and_memory(f):
    """C2-like (100 000 x 10 000 tf-idf) and C4-like (100 000 x 50 000, 0.2 %) self search, k = 10: 64 sampled rows bit for bit
    against the float32 oracle and within the fp64 bound; device memory above the inputs within the workspace formula."""
    import torch
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    n = 100000
    x = make_sparse(n, f, mean_nnz=100, kind='tfidf', seed=f)
    d = DeviceCSR(x, 'cuda:0')
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    idx, val = helpers._csr_similarity_topk(d, d, 10, exclude=True)
    torch.cuda.synchronize()
    above = torch.cuda.max_memory_allocated() - base
    bound = 8 * x.nnz + 4 * ((n + 2047) // 2048 * f + 1) + n * 10 * 8 + (8 << 20)   # + the allocator's 2 MB rounding
    assert above <= bound, (above, bound)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    rows = np.sort(np.random.default_rng(3).choice(n, 64, replace=False))
    s = f32_column_oracle(x[rows], x).astype(np.float64)
    s[np.arange(64), rows] = -np.inf
    want = _exact_top_k(s, 10)
    assert np.array_equal(idx[rows], want[0]) and np.array_equal(val[rows], want[1])
    s64 = (x[rows].astype(np.float64) @ x.astype(np.float64).T).toarray()
    s64[np.arange(64), rows] = -np.inf
    _check_fp64(idx[rows], val[rows], s64, 10)


def test_fewer_candidates_than_k_are_padded():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    c = _tfidf_like(40, 50, 12)[:5]
    q = _tfidf_like(40, 50, 13)[:9]
    idx, val = top_k_similar(q, k=10, corpus=c, metric='linear kernel')
    assert (idx[:, 5:] == -1).all() and (val[:, 5:] == -np.inf).all()
    want = _expected(q, c, 10, False)
    assert np.array_equal(idx, want[0]) and np.array_equal(val, want[1])
    idx, val = top_k_similar(c, k=10, metric='linear kernel')     # self: 4 candidates per row
    assert (idx[:, 4:] == -1).all() and (val[:, 4:] == -np.inf).all()
    want = _expected(c, c, 10, True)
    assert np.array_equal(idx, want[0]) and np.array_equal(val, want[1])


def test_cli_top_k_input_on_synthetic():
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    argv = ['--model_name', 'syntki', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--top_k', '5', '--top_k_input']
    model = cli.main(argv)
    ev = model.evaluation
    trX, vlX, _, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    for split, n, X in (('', 960, trX), ('_validate', 240, vlX)):
        idx = np.load(model.data_dir + 'article_top_k_input_index%s.npy' % split)
        score = np.load(model.data_dir + 'article_top_k_input_score%s.npy' % split)
        assert idx.shape == (n, 5) and score.shape == (n, 5) and idx.dtype == np.int32
        assert ((idx >= 0) & (idx < 960)).all() and (score <= 1.0 + 1e-5).all()
        want = top_k_similar(X, k=5, corpus=None if split == '' else trX, metric='cosine')
        assert np.array_equal(idx, want[0]) and np.array_equal(score, want[1])
        assert 0.0 <= ev['top_k_input_precision' + split] <= 1.0
        assert 0.0 <= ev['top_k_precision' + split] <= 1.0
        assert np.array_equal(np.load(model.data_dir + 'article_top_k_index%s.npy' % split), ev['top_k' + split][0])
