"""CPU checks of the bag-of-words user profiles (helpers.sparse_profiles / recommend_sparse / impression_metrics_sparse, DESIGN
4.20): the float32 ordered oracle against scipy in fp64 and its order sensitivity, the chunk planner, the argument checks of the
helpers and of the C ABI, and the --user_top_k_input flag rules."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import sparse_profile_oracle as so
from dae_rnn_news_recommendation_b200 import _cabi, helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(U=30, N=40, F=60, seed=0):
    rng = np.random.default_rng(seed)
    X = sp.random(N, F, density=0.15, random_state=seed, format='csr', dtype=np.float32)
    X.data = rng.normal(0, 1, X.nnz).astype(np.float32)
    H = sp.random(U, N, density=0.2, random_state=seed + 1, format='csr', dtype=np.float32)
    H.data = rng.uniform(0.1, 2.0, H.nnz).astype(np.float32)
    return H, X


def _weights(H, X, fn='test'):
    return helpers._history_weights(H, X.shape[0], fn)[0]


def test_oracle_matches_scipy_in_fp64():
    H, X = _case()
    w = _weights(H, X)
    x = helpers._sparse_articles(X, 'test')
    P = so.profiles(w, x)
    ref = (w.astype(np.float64) @ x.astype(np.float64)).toarray()
    np.testing.assert_allclose(P.toarray(), ref, rtol=1e-5, atol=1e-6)
    # the structure is the union of the read rows' columns, whatever the values
    pattern = (sp.csr_matrix((np.ones(w.nnz), w.indices, w.indptr), shape=w.shape) @
               sp.csr_matrix((np.ones(x.nnz), x.indices, x.indptr), shape=x.shape)).tocsr()
    pattern.sort_indices()
    assert np.array_equal(P.indptr, pattern.indptr) and np.array_equal(P.indices, pattern.indices)
    Pn = so.profiles(w, x, normalise=True)
    norm = np.sqrt((ref ** 2).sum(1, keepdims=True))
    np.testing.assert_allclose(Pn.toarray(), np.divide(ref, norm, out=np.zeros_like(ref), where=norm > 0), rtol=1e-5, atol=1e-6)
    for i, a in [(0, 0), (3, 5), (7, 11)]:
        q = Pn
        got = so.pair_score(q, i, x, a)
        assert abs(float(got) - (q[i].toarray() @ x[a].toarray().T)[0, 0]) < 1e-5
        c = so.pair_score(P, i, x, a, cosine=True)
        qa, xa = P[i].toarray().ravel().astype(np.float64), x[a].toarray().ravel().astype(np.float64)
        nq, nx = np.linalg.norm(qa), np.linalg.norm(xa)
        assert abs(float(c) - (qa @ xa / (nq * nx) if nq and nx else 0.0)) < 1e-5


def test_oracle_follows_the_article_order():
    # one user reads three articles sharing column 0 with values 1, 1e8, -1e8: fp32 in article order gives (1 + 1e8) - 1e8 = 0,
    # the reverse order (-1e8 + 1e8) + 1 = 1, which is also the exact value
    vals = np.array([1.0, 1e8, -1e8], np.float32)
    X = sp.csr_matrix((vals, np.zeros(3, np.int32), np.arange(4)), shape=(3, 2))
    Xr = sp.csr_matrix((vals[::-1].copy(), np.zeros(3, np.int32), np.arange(4)), shape=(3, 2))
    w = sp.csr_matrix((np.ones(3, np.float32), np.arange(3, dtype=np.int32), np.array([0, 3])), shape=(1, 3))
    fwd, rev = so.profiles(w, X).data, so.profiles(w, Xr).data
    assert fwd.tobytes() != rev.tobytes()
    assert fwd[0] == 0.0 and rev[0] == 1.0
    assert (w.astype(np.float64) @ X.astype(np.float64)).toarray()[0, 0] == 1.0


def _chunks_restated(p, budget):
    out, u0, n_u = [], 0, len(p) - 1
    while u0 < n_u:
        u1 = u0 + 1
        while u1 < n_u and p[u1 + 1] - p[u0] <= budget:
            u1 += 1
        out.append((u0, u1))
        u0 = u1
    return out


@pytest.mark.parametrize('seed', range(6))
def test_chunk_planner_restatement(seed):
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 50, rng.integers(1, 200))
    counts[rng.random(counts.size) < 0.2] = 0
    p = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    for budget in (1, 10, 49, 50, 120, int(p[-1]), int(p[-1]) + 5):
        got = helpers._profile_chunks(p, budget)
        assert got == _chunks_restated(p, budget)
        assert got[0][0] == 0 and got[-1][1] == counts.size
        for u0, u1 in got:
            assert u1 > u0 and (p[u1] - p[u0] <= budget or u1 == u0 + 1)


def test_helpers_refuse_bad_arguments_before_device_work():
    H, X = _case()
    imp = {'indptr': np.array([0, 2]), 'items': np.array([0, 1], np.int32), 'clicked': np.array([1, 0], np.uint8)}
    P1 = sp.csr_matrix((1, X.shape[1]), dtype=np.float32)
    for k in (0, 33, 1.5, True):
        with pytest.raises(ValueError, match='recommend_sparse: k'):
            helpers.recommend_sparse(H, X, k=k)
    with pytest.raises(ValueError, match='metric'):
        helpers.recommend_sparse(H, X, metric='dot')
    with pytest.raises(ValueError, match='scipy sparse'):
        helpers.recommend_sparse(H, X.toarray())
    with pytest.raises(ValueError, match='scipy sparse'):
        helpers.sparse_profiles(H, X.toarray())
    with pytest.raises(ValueError, match='2\\^24'):
        helpers.sparse_profiles(sp.csr_matrix((1, 2)), sp.csr_matrix((2, (1 << 24) + 1), dtype=np.float32))
    with pytest.raises(ValueError, match='histories'):
        helpers.sparse_profiles(H[:, :5], X)
    with pytest.raises(ValueError, match='no user'):
        helpers.sparse_profiles(sp.csr_matrix((0, X.shape[0])), X)
    with pytest.raises(ValueError, match='candidates'):
        helpers.recommend_sparse(H, X, candidates=[3, 1])
    with pytest.raises(ValueError, match='groups'):
        helpers.recommend_sparse(H, X, groups=np.zeros(3, np.int64))
    bad = H.copy()
    bad.data[0] = np.nan
    with pytest.raises(ValueError, match='not finite'):
        helpers.recommend_sparse(bad, X)
    with pytest.raises(ValueError, match='metric'):
        helpers.impression_metrics_sparse(P1, X, imp, metric='dot')
    with pytest.raises(ValueError, match='shape'):
        helpers.impression_metrics_sparse(sp.csr_matrix((2, X.shape[1])), X, imp)
    with pytest.raises(ValueError, match='scipy sparse matrix or sparse_profiles'):
        helpers.impression_metrics_sparse(np.zeros((1, X.shape[1]), np.float32), X, imp)
    with pytest.raises(ValueError):
        helpers.impression_metrics_sparse(P1, X, {'indptr': np.array([0, 2]), 'items': np.array([0, X.shape[0]]),
                                                  'clicked': np.array([1, 0], np.uint8)})
    Xinf = X.copy()
    Xinf.data[0] = np.inf
    with pytest.raises(ValueError, match='finite'):
        helpers.impression_metrics_sparse(P1, Xinf, imp)
    big = P1.tolil()
    big[0, 0] = 2.0 ** 62
    with pytest.raises(ValueError, match='magnitude'):
        helpers.impression_metrics_sparse(big.tocsr(), X, imp)


def test_exports_refuse_bad_arguments_without_gpu():
    x = 1 << 20   # a non-null, aligned pointer value: every call below fails its checks before reading it
    with pytest.raises(_cabi.DaeError, match='dae_csr_profiles_count: null'):
        _cabi.call('dae_csr_profiles_count', None, x, 4, 5, x, x, 10, x, None)
    with pytest.raises(_cabi.DaeError, match='dae_csr_profiles_count: bad sizes'):
        _cabi.call('dae_csr_profiles_count', x, x, 4, 5, x, x, (1 << 24) + 1, x, None)
    with pytest.raises(_cabi.DaeError, match='dae_csr_profiles_count: bad sizes'):
        _cabi.call('dae_csr_profiles_count', x, x, 0, 5, x, x, 10, x, None)
    with pytest.raises(_cabi.DaeError, match='dae_csr_profiles_count: indptr'):
        _cabi.call('dae_csr_profiles_count', x + 4, x, 4, 5, x, x, 10, x, None)
    args = [x, x, x, 4, 5, x, x, x, 10, x, 0, 4, 0, x, x, None]
    for i, v, msg in ((0, None, 'null'), (8, 0, 'bad sizes'), (10, 1, 'range'), (11, 0, 'range'), (10, -1, 'range'),
                      (12, 2, 'normalise'), (13, x + 2, 'aligned')):
        a = list(args)
        a[i] = v
        with pytest.raises(_cabi.DaeError, match='dae_csr_profiles: .*' + msg):
            _cabi.call('dae_csr_profiles', *a)
    args = [x, x, x, x, x, x, 5, 10, 0, x, x, x, 3, x, x, None]
    for i, v, msg in ((0, None, 'null'), (14, None, 'null'), (8, 2, 'cosine = 2'), (12, 0, 'bad arguments'), (6, 0, 'bad arguments'),
                      (13, x + 2, 'aligned')):
        a = list(args)
        a[i] = v
        with pytest.raises(_cabi.DaeError, match='dae_csr_impression_metrics: .*' + msg):
            _cabi.call('dae_csr_impression_metrics', *a)


def test_user_top_k_input_flags(tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    h = tmp_path / 'h.npz'
    sp.save_npz(h, sp.csr_matrix(np.ones((2, 3), np.float32)))
    s = tmp_path / 's.npz'
    np.savez(s, indptr=np.array([0, 1]), items=np.array([0]))
    p = cli.build_parser()
    assert cli.check_flags(p.parse_args(['--top_k', '5', '--user_histories', str(h), '--user_top_k_input'])).user_top_k_input
    assert cli.check_flags(p.parse_args(['--top_k', '32', '--user_sequences', str(s), '--user_top_k_input'])).user_top_k_input
    assert not cli.check_flags(p.parse_args(['--top_k', '5', '--user_histories', str(h)])).user_top_k_input
    with pytest.raises(AssertionError, match='--user_top_k_input needs --user_histories or --user_sequences'):
        cli.check_flags(p.parse_args(['--top_k', '5', '--user_top_k_input']))
    with pytest.raises(AssertionError, match='--user_top_k_input needs --top_k K in 1..32'):
        cli.check_flags(p.parse_args(['--top_k', '33', '--long_lists', '--user_histories', str(h), '--user_top_k_input']))
    with pytest.raises(AssertionError, match='needs --top_k K'):
        cli.check_flags(p.parse_args(['--user_histories', str(h), '--user_top_k_input']))
