"""Bag-of-words user profiles on the GPU (DESIGN 4.20): dae_csr_profiles_count / dae_csr_profiles bit for bit against the float32
ordered oracle, recommend_sparse bit for bit against the sparse top-k of the oracle's profiles, impression_metrics_sparse against
the oracle, the sparse top-k's pair scores and the dense dae_impression_metrics, and the --user_top_k_input CLI runs."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import sparse_profile_oracle as so  # noqa: E402

from dae_rnn_news_recommendation_b200 import helpers  # noqa: E402
from dae_rnn_news_recommendation_b200._cabi import call  # noqa: E402
from dae_rnn_news_recommendation_b200.engine import DeviceCSR  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import check_impressions  # noqa: E402

D = 'cuda:0'


def _same(a, b):
    """two scipy CSR matrices with the same structure and the same value bits"""
    assert a.shape == b.shape
    assert np.array_equal(np.asarray(a.indptr, np.int64), np.asarray(b.indptr, np.int64))
    assert np.array_equal(a.indices, b.indices)
    assert np.array_equal(np.asarray(a.data, np.float32).view(np.uint32), np.asarray(b.data, np.float32).view(np.uint32))


def _articles(N, F, density, seed, zero_rows=(), explicit_zeros=0):
    """a canonical fp32 CSR [N, F] of normal values, about density F entries per row; zero_rows store nothing, and
    explicit_zeros stored entries are 0"""
    rng = np.random.default_rng(seed)
    cols = [np.unique(rng.integers(0, F, rng.binomial(F, density))) for _ in range(N)]
    for r in zero_rows:
        cols[r] = cols[r][:0]
    indptr = np.concatenate([[0], np.cumsum([c.size for c in cols])]).astype(np.int64)
    data = rng.normal(0, 1, int(indptr[-1])).astype(np.float32)
    if explicit_zeros:
        data[rng.choice(data.size, explicit_zeros, replace=False)] = 0.0
    X = sp.csr_matrix((data, np.concatenate(cols).astype(np.int32), indptr), shape=(N, F))
    return helpers._sparse_articles(X, 'test')


def _histories(U, N, seed, empty=(), zero=(), repeats=0):
    rng = np.random.default_rng(seed)
    rows, cols, vals = [], [], []
    for u in range(U):
        if u in empty:
            continue
        n = int(rng.integers(1, 12))
        c = rng.choice(N, n, replace=False)
        rows += [u] * n
        cols += list(c)
        vals += list(np.zeros(n) if u in zero else rng.uniform(0.1, 3.0, n))
    for _ in range(repeats):   # repeated reads: the same position stored twice, summed by the helpers
        i = int(rng.integers(len(rows)))
        rows.append(rows[i]); cols.append(cols[i]); vals.append(vals[i])
    return sp.coo_matrix((np.asarray(vals, np.float32), (rows, cols)), shape=(U, N))


def _device_profiles(w, x, normalise, cuts=()):
    """count once, fill the user ranges between the cuts, glue the ranges: a scipy CSR"""
    hist, xd = DeviceCSR(w, D), DeviceCSR(x, D)
    p = helpers._profile_structure(hist, xd)
    ph = p.cpu().numpy()
    bounds = [0, *cuts, w.shape[0]]
    ind, val = [], []
    for u0, u1 in zip(bounds[:-1], bounds[1:]):
        if u1 > u0:
            r = helpers._profile_rows(hist, xd, p, ph, u0, u1, normalise)
            assert np.array_equal(r.indptr.cpu().numpy(), ph[u0:u1 + 1] - ph[u0])
            ind.append(r.indices.cpu().numpy())
            val.append(r.values.cpu().numpy())
    return sp.csr_matrix((np.concatenate(val), np.concatenate(ind), ph), shape=(w.shape[0], x.shape[1]))


PROFILE_CASES = {
    # name: (U, N, F, density, empty users, zero-weight users, repeated reads, empty article rows, explicit zeros)
    'mixed': (40, 60, 300, 0.05, (0, 7), (3, 11), 5, (2, 5, 9), 20),
    'F1': (9, 12, 1, 0.6, (4,), (5,), 2, (0,), 1),
    'F10000': (25, 200, 10000, 0.01, (1,), (2,), 3, (3,), 10),
    'F2^24': (6, 30, 1 << 24, 2e-6, (), (1,), 1, (4,), 2),
}


@pytest.mark.parametrize('name', sorted(PROFILE_CASES))
@pytest.mark.parametrize('normalise', [False, True])
def test_profiles_bit_exact(name, normalise):
    U, N, F, dens, empty, zero, reps, zrows, ez = PROFILE_CASES[name]
    x = _articles(N, F, dens, seed=len(name), zero_rows=zrows, explicit_zeros=min(ez, int(N * F * dens) // 2))
    w, _ = helpers._history_weights(_histories(U, N, seed=1, empty=empty, zero=zero, repeats=reps), N, 'test')
    ref = so.profiles(w, x, normalise)
    _same(_device_profiles(w, x, normalise), ref)
    rng = np.random.default_rng(2)
    for _ in range(3):   # user ranges that split the set anywhere
        cuts = sorted(set(rng.integers(1, U, int(rng.integers(1, 4))).tolist()))
        _same(_device_profiles(w, x, normalise, cuts), ref)
    if not normalise:
        _same(helpers.sparse_profiles(_histories(U, N, seed=1, empty=empty, zero=zero, repeats=reps), x), ref)


def test_profiles_of_a_5000_read_user():
    N, F = 6000, 3000
    x = _articles(N, F, 0.01, seed=3, zero_rows=(10, 11))
    rng = np.random.default_rng(4)
    reads = np.sort(rng.choice(N, 5000, replace=False))
    H = sp.csr_matrix((rng.uniform(0.5, 2, 5000 + 3).astype(np.float32), np.concatenate([reads, [1, 2, 3]]),
                       np.array([0, 5000, 5000, 5003])), shape=(3, N))
    w, _ = helpers._history_weights(H, N, 'test')
    for normalise in (False, True):
        ref = so.profiles(w, x, normalise)
        _same(_device_profiles(w, x, normalise), ref)
        _same(_device_profiles(w, x, normalise, (1,)), ref)


def _topk_reference(H, X, k, metric, candidates=None, groups=None):
    """top_k_similar of the oracle's profiles against _csr_operand(X, metric) with the histories as exclusion lists (and the
    read groups with groups), candidates remapped: the contract recommend_sparse restates"""
    x = helpers._sparse_articles(X, 'test')
    w, empty = helpers._history_weights(H, X.shape[0], 'test')
    P = so.profiles(w, x, metric == 'cosine')
    corpus = helpers._csr_operand(x, metric)
    read = sp.csr_matrix((np.ones(w.nnz, np.float32), w.indices, w.indptr), shape=w.shape)
    cand = np.arange(X.shape[0]) if candidates is None else np.asarray(candidates)
    if groups is not None:
        G = sp.csr_matrix((np.ones(X.shape[0]), (np.arange(X.shape[0]), groups)))
        excl = ((read @ G) @ G.T).tocsr()[:, cand]
    else:
        excl = read[:, cand]
    idx, val = helpers.top_k_similar(P, k=k, corpus=corpus[cand], metric='linear kernel', exclude=excl,
                                     groups=None if groups is None else np.asarray(groups)[cand])
    idx = np.where(idx >= 0, cand[np.maximum(idx, 0)], idx)
    idx[empty], val[empty] = -1, -np.inf
    return idx, val


def _same_lists(got, ref):
    assert np.array_equal(got[0], ref[0])
    assert np.array_equal(got[1].view(np.uint32), ref[1].view(np.uint32))


@pytest.mark.parametrize('metric', ['cosine', 'linear kernel'])
@pytest.mark.parametrize('mode', ['plain', 'candidates', 'groups', 'both'])
def test_recommend_sparse_bit_exact(metric, mode):
    N, F, U, k = 300, 500, 50, 7
    rng = np.random.default_rng(5)
    X = sp.csr_matrix(_articles(N, F, 0.03, seed=6, zero_rows=(8,)))
    H = _histories(U, N, seed=7, empty=(0, 9), zero=(4,), repeats=3)
    cand = np.sort(rng.choice(N, 200, replace=False)) if mode in ('candidates', 'both') else None
    groups = rng.integers(0, 120, N) if mode in ('groups', 'both') else None
    got = helpers.recommend_sparse(H, X, k=k, candidates=cand, metric=metric, groups=groups)
    _same_lists(got, _topk_reference(H, X, k, metric, cand, groups))
    assert (got[0][[0, 9, 4]] == -1).all() and np.isneginf(got[1][[0, 9, 4]]).all()   # no reads / zero weights: padding


def test_recommend_sparse_chunks_do_not_change_the_result(monkeypatch):
    N, F, U = 400, 800, 120
    X = sp.csr_matrix(_articles(N, F, 0.02, seed=8))
    H = _histories(U, N, seed=9, empty=(3, 50), repeats=2)
    groups = np.random.default_rng(1).integers(0, 100, N)
    for metric in ('cosine', 'linear kernel'):
        one = helpers.recommend_sparse(H, X, k=10, metric=metric, groups=groups)
        for budget in (1, 37, 500):
            monkeypatch.setattr(helpers, 'SPARSE_PROFILE_CHUNK_NNZ', budget)
            _same_lists(helpers.recommend_sparse(H, X, k=10, metric=metric, groups=groups), one)
        monkeypatch.undo()


def test_recommend_sparse_integer_ties_match_lexsort():
    # binary articles, four reads per user: weights 1/4 and every profile value and score is exact, with many equal scores
    rng = np.random.default_rng(10)
    N, F, U, k = 80, 12, 30, 9
    X = sp.csr_matrix((rng.random((N, F)) < 0.3).astype(np.float32))
    reads = np.stack([np.sort(rng.choice(N, 4, replace=False)) for _ in range(U)])
    H = sp.csr_matrix((np.ones(4 * U, np.float32), reads.ravel(), np.arange(0, 4 * U + 1, 4)), shape=(U, N))
    idx, val = helpers.recommend_sparse(H, X, k=k, metric='linear kernel')
    S = (H.toarray().astype(np.float64) / 4) @ X.toarray().astype(np.float64) @ X.toarray().T.astype(np.float64)
    for u in range(U):
        c = np.setdiff1d(np.arange(N), reads[u])
        order = np.lexsort((c, -S[u, c]))[:k]
        assert np.array_equal(idx[u], c[order]), u
        assert np.array_equal(val[u].astype(np.float64), S[u, c[order]])


def test_recommend_sparse_on_uci_c1():
    from helpers import load_uci_c1
    from dae_rnn_news_recommendation_b200.synth import make_histories
    d = load_uci_c1()
    X = d['train']
    H, _ = make_histories(2000, d['train_label_category_publish_name'], mean_len=10, seed=11)
    for metric in ('cosine', 'linear kernel'):
        _same_lists(helpers.recommend_sparse(H, X, k=10, metric=metric), _topk_reference(H, X, 10, metric))


def _impressions(N, n_imp, seed, long_one=0):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 12, n_imp)
    if long_one:
        lens[1] = long_one
    items = np.concatenate([rng.choice(N, n, replace=False) for n in lens]).astype(np.int32)
    clicked = (rng.random(items.size) < 0.3).astype(np.uint8)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    clicked[indptr[2]:indptr[3]] = 1        # impression 2: no non-click
    clicked[indptr[3]:indptr[4]] = 0        # impression 3: no click
    return check_impressions({'indptr': indptr, 'items': items, 'clicked': clicked}, N, 'test')


def _show(imp, a):
    """put article a on show in the first impression from the fifth on that does not show it yet (items stay distinct)"""
    for i in range(5, imp['indptr'].size - 1):
        b0, b1 = imp['indptr'][i], imp['indptr'][i + 1]
        if a not in imp['items'][b0:b1]:
            imp['items'][b0] = a
            return
    raise AssertionError('no impression to show %d in' % a)


def _csr_scores(Q, X, imp, metric):
    s, m = helpers._csr_impression_scores(DeviceCSR(Q, D), DeviceCSR(X, D), imp, metric)
    return s.cpu().numpy(), m.cpu().numpy()


@pytest.mark.parametrize('metric', ['cosine', 'linear kernel'])
def test_impression_scores_against_the_oracle(metric):
    N, F, n_imp = 400, 700, 30
    X = _articles(N, F, 0.03, seed=12, zero_rows=(3, 4, 5))
    Q = _articles(n_imp, F, 0.2, seed=13, zero_rows=(0, 6))
    imp = _impressions(N, n_imp, seed=14, long_one=300)   # one impression longer than the kernel's 256-score staging chunk
    _show(imp, 3)                                         # an empty article row on show
    s, m = _csr_scores(Q, X, imp, metric)
    ref = so.impression_scores(Q, X, imp['indptr'], imp['items'], metric == 'cosine')
    assert np.array_equal(s.view(np.uint32), ref.view(np.uint32))
    om = so.impression_metrics(ref, imp['indptr'], imp['clicked'])
    assert np.array_equal(np.isnan(m), np.isnan(om)) and np.isnan(m[[2, 3]]).all()
    np.testing.assert_allclose(m[~np.isnan(m)], om[~np.isnan(om)], rtol=1e-12, atol=1e-12)
    r = helpers.impression_metrics_sparse(Q, X, imp, metric=metric)
    assert r['skipped'] == int(np.isnan(m[:, 0]).sum()) and r['impressions'] == n_imp - r['skipped']
    assert r['auc'] == pytest.approx(float(np.nanmean(m[:, 0])), rel=1e-12)


def test_impression_scores_are_the_sparse_topk_scores():
    N, F, n_imp = 32, 200, 20   # every article is in a k = 32 list, so each pair's top-k score is known
    X = _articles(N, F, 0.1, seed=15)
    Q = _articles(n_imp, F, 0.3, seed=16)
    imp = _impressions(N, n_imp, seed=17)
    s, _ = _csr_scores(Q, X, imp, 'linear kernel')
    idx, val = helpers.top_k_similar(Q, k=N, corpus=X, metric='linear kernel')
    for i in range(n_imp):
        pos = {int(j): v for j, v in zip(idx[i], val[i])}
        for t in range(imp['indptr'][i], imp['indptr'][i + 1]):
            assert np.float32(s[t]).view(np.uint32) == np.float32(pos[int(imp['items'][t])]).view(np.uint32)


@pytest.mark.parametrize('metric', ['cosine', 'linear kernel'])
def test_small_integers_match_the_dense_kernel(metric):
    rng = np.random.default_rng(18)
    N, F, n_imp = 300, 40, 40
    Xd = rng.integers(-2, 3, (N, F)).astype(np.float32) * (rng.random((N, F)) < 0.3)
    Qd = rng.integers(-3, 4, (n_imp, F)).astype(np.float32) * (rng.random((n_imp, F)) < 0.5)
    Xd[7] = 0.0   # an empty article
    Qd[1] = 0.0   # a zero query
    Xd[:, 0] = 0.0
    imp = _impressions(N, n_imp, seed=19, long_one=270)
    _show(imp, 7)
    # ties: impression 4 shows the same row twice under two ids
    Xd[imp['items'][imp['indptr'][4] + 1]] = Xd[imp['items'][imp['indptr'][4]]]
    s, m = _csr_scores(helpers._sparse_articles(sp.csr_matrix(Qd), 't'), helpers._sparse_articles(sp.csr_matrix(Xd), 't'), imp, metric)
    ds, dm = helpers._impression_scores(torch.from_numpy(Qd).to(D), torch.from_numpy(Xd).to(D), imp, metric)
    assert np.array_equal(s.view(np.uint32), ds.cpu().numpy().view(np.uint32))
    assert np.array_equal(m.view(np.uint64), dm.cpu().numpy().view(np.uint64))


def test_impression_metrics_sparse_takes_device_profiles():
    N, F, U = 120, 300, 20
    X = sp.csr_matrix(_articles(N, F, 0.05, seed=20))
    H = _histories(U, N, seed=21, empty=(2,))
    imp = _impressions(N, U, seed=22)
    host = helpers.sparse_profiles(H, X)
    dev = helpers.sparse_profiles(H, X, to_host=False)
    a = helpers.impression_metrics_sparse(host, X, imp, metric='cosine')
    b = helpers.impression_metrics_sparse(dev, X, imp, metric='cosine')
    assert a == b


def test_cli_user_top_k_input(capsys, tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.synth import make_histories, make_impressions, make_sequences
    argv = ['--model_name', 'synbow', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '1', '--batch_size', '200',
            '--seed', '3', '--top_k', '5']
    trX, _, trL, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    H, T = make_histories(200, trL, mean_len=8, seed=4)
    sp.save_npz(tmp_path / 'h.npz', H)
    sp.save_npz(tmp_path / 't.npz', T)
    model = cli.main(argv + ['--user_histories', str(tmp_path / 'h.npz'), '--user_targets', str(tmp_path / 't.npz'),
                             '--user_top_k_input'])
    ev = model.evaluation
    assert np.load(model.data_dir + 'user_top_k_input_index.npy').shape == (200, 5)
    assert np.load(model.data_dir + 'user_top_k_input_score.npy').shape == (200, 5)
    for key in ('user_input_hit_rate', 'user_input_recall'):
        assert 0.0 <= ev[key] <= 1.0
    assert 'input vectors' in capsys.readouterr().out
    indptr, items, targets = make_sequences(200, trL, mean_len=8, seed=5)
    _, test_imp = make_impressions(indptr, items, trL, targets, seed=6)
    np.savez(tmp_path / 's.npz', indptr=indptr, items=items, targets=targets)
    np.savez(tmp_path / 'ti.npz', **test_imp)
    model = cli.main(argv + ['--user_sequences', str(tmp_path / 's.npz'), '--user_epochs', '1', '--user_test_impressions',
                             str(tmp_path / 'ti.npz'), '--user_top_k_input'])
    ev = model.evaluation
    for key in ('user_input_seq_hit_rate', 'user_input_seq_recall', 'user_input_imp_auc', 'user_input_imp_mrr',
                'user_input_imp_ndcg5', 'user_input_imp_ndcg10', 'user_mean_imp_auc', 'user_gru_imp_auc'):
        assert 0.0 <= ev[key] <= 1.0, key
    assert 'mean profile' in capsys.readouterr().out


def test_exports_by_name():
    """the three exports called directly: one user, one article, one impression"""
    i64 = lambda a: torch.tensor(a, dtype=torch.int64, device=D)
    i32 = lambda a: torch.tensor(a, dtype=torch.int32, device=D)
    f32 = lambda a: torch.tensor(a, dtype=torch.float32, device=D)
    w_ptr, w_ind, w_val = i64([0, 2]), i32([0, 1]), f32([0.5, 0.5])
    x_ptr, x_ind, x_val = i64([0, 2, 3]), i32([1, 4, 4]), f32([2.0, 4.0, 2.0])
    p = torch.empty(2, dtype=torch.int64, device=D)
    call('dae_csr_profiles_count', w_ptr.data_ptr(), w_ind.data_ptr(), 1, 2, x_ptr.data_ptr(), x_ind.data_ptr(), 5, p.data_ptr(), None)
    assert p.tolist() == [0, 2]
    pi, pv = torch.empty(2, dtype=torch.int32, device=D), torch.empty(2, dtype=torch.float32, device=D)
    call('dae_csr_profiles', w_ptr.data_ptr(), w_ind.data_ptr(), w_val.data_ptr(), 1, 2, x_ptr.data_ptr(), x_ind.data_ptr(),
         x_val.data_ptr(), 5, p.data_ptr(), 0, 1, 0, pi.data_ptr(), pv.data_ptr(), None)
    assert pi.tolist() == [1, 4] and pv.tolist() == [1.0, 3.0]
    imp_ptr, items, clicked = i64([0, 2]), i32([0, 1]), torch.tensor([0, 1], dtype=torch.uint8, device=D)
    scores, metrics = torch.empty(2, dtype=torch.float32, device=D), torch.empty(1, 4, dtype=torch.float64, device=D)
    call('dae_csr_impression_metrics', p.data_ptr(), pi.data_ptr(), pv.data_ptr(), x_ptr.data_ptr(), x_ind.data_ptr(), x_val.data_ptr(),
         2, 5, 0, imp_ptr.data_ptr(), items.data_ptr(), clicked.data_ptr(), 1, scores.data_ptr(), metrics.data_ptr(), None)
    torch.cuda.synchronize()
    assert scores.tolist() == [14.0, 6.0]   # 1*2 + 3*4, 3*2
    assert metrics[0].tolist() == [0.0, 0.5, pytest.approx(1 / np.log2(3)), pytest.approx(1 / np.log2(3))]
