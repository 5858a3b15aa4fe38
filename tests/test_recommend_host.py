"""Host-side parts of recommending unread articles: argument checks of the exclusion-list entry points (before any CUDA call), the
ValueErrors of top_k_similar(exclude=...), user_profiles and recommend before any device work, recommendation_recall, the
candidate remapping, synth.make_histories and the CLI flags."""
import ctypes
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FAKE = 1 << 20   # 16-byte aligned non-null stand-in for a device pointer: every call below fails validation before using it


def _dense(k=10, ws_bytes=1 << 30, ex_indptr=FAKE, ex_indices=FAKE, ex_nnz=5, ldq=64):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_similarity_topk_excl_bf16x3', 300, 500, 64, FAKE, FAKE, ldq, FAKE, FAKE, 64, k, 0, 1, 1, FAKE, ws_bytes, FAKE, FAKE,
               ex_indptr, ex_indices, ex_nnz, None)


def _sparse(k=10, ws_bytes=1 << 40, ex_indptr=FAKE, ex_indices=FAKE, ex_nnz=5):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_csr_similarity_topk_excl', FAKE, FAKE, FAKE, 300, 100, 50, FAKE, FAKE, FAKE, 500, 100, 50, k, 0, 1, 1, FAKE, ws_bytes,
               FAKE, FAKE, ex_indptr, ex_indices, ex_nnz, None)


@pytest.mark.parametrize('call', [_dense, _sparse])
def test_excl_exports_check_their_arguments(call):
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='null pointer'):
        call(ex_indptr=None)
    with pytest.raises(_cabi.DaeError, match='null pointer'):
        call(ex_indices=None, ex_nnz=3)
    with pytest.raises(_cabi.DaeError, match='bad sizes'):
        call(ex_nnz=-1)
    with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
        call(k=33)
    with pytest.raises(_cabi.DaeError, match='aligned'):
        call(ex_indptr=FAKE + 4)
    with pytest.raises(_cabi.DaeError, match='aligned'):
        call(ex_indices=FAKE + 2)
    with pytest.raises(_cabi.DaeError, match='workspace'):
        call(ws_bytes=16)


def test_dense_excl_export_checks_leading_dimensions():
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='leading dimensions'):
        _dense(ldq=60)


def test_workspace_of_the_excl_exports_is_the_plain_one():
    from dae_rnn_news_recommendation_b200 import _cabi
    out = (ctypes.c_int64 * 1)()
    _cabi.call('dae_similarity_topk_workspace', 300, 500, 10, 1, ctypes.addressof(out))
    with pytest.raises(_cabi.DaeError, match='workspace'):
        _dense(ws_bytes=out[0] - 1)


def _no_device(monkeypatch):
    """Any device work fails the test: the checks must come first."""
    import torch

    def boom(*a, **k):
        raise AssertionError('touched the device')
    monkeypatch.setattr(torch.Tensor, 'to', boom)
    monkeypatch.setattr(torch.Tensor, 'cuda', boom)
    from dae_rnn_news_recommendation_b200 import _cabi
    monkeypatch.setattr(_cabi, 'call', boom)


def test_exclude_errors_before_the_device(monkeypatch):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    _no_device(monkeypatch)
    x = np.zeros((4, 3), np.float32)
    c = np.zeros((6, 3), np.float32)
    with pytest.raises(ValueError, match='scipy sparse'):
        top_k_similar(x, k=2, exclude=np.zeros((4, 4)))
    with pytest.raises(ValueError, match='shape'):
        top_k_similar(x, k=2, exclude=sp.csr_matrix((4, 5)))
    with pytest.raises(ValueError, match='shape'):
        top_k_similar(x, k=2, corpus=c, exclude=sp.csr_matrix((4, 4)))
    bad = sp.csr_matrix((np.ones(1), np.array([9]), np.array([0, 1, 1, 1, 1])), shape=(4, 6))   # column 9 of 6
    with pytest.raises(ValueError, match='outside'):
        top_k_similar(x, k=2, corpus=c, exclude=bad)
    with pytest.raises(ValueError, match='outside'):
        top_k_similar(sp.csr_matrix(x), k=2, corpus=sp.csr_matrix(c), exclude=bad)


def test_stored_positions_are_canonical_and_keep_explicit_zeros():
    from dae_rnn_news_recommendation_b200.helpers import _stored_positions
    m = sp.coo_matrix((np.array([0.0, 2.0, 1.0, 5.0]), (np.array([1, 0, 1, 1]), np.array([4, 3, 2, 4]))), shape=(3, 6))
    indptr, indices, data = _stored_positions(m, (3, 6), 'exclude', 'f')
    assert indptr.tolist() == [0, 1, 3, 3] and indices.tolist() == [3, 2, 4] and data.tolist() == [2.0, 1.0, 5.0]
    assert indptr.dtype == np.int64 and indices.dtype == np.int32
    z = sp.csr_matrix((np.zeros(2), np.array([1, 0]), np.array([0, 2])), shape=(1, 3))       # explicit zeros, unsorted
    assert _stored_positions(z, (1, 3), 'x', 'f')[1].tolist() == [0, 1]


def test_user_profiles_and_recommend_errors_before_the_device(monkeypatch):
    from dae_rnn_news_recommendation_b200.helpers import recommend, user_profiles
    _no_device(monkeypatch)
    emb = np.zeros((6, 4), np.float32)
    good = sp.csr_matrix((2, 6), dtype=np.float32)
    for f in (user_profiles, recommend):
        with pytest.raises(ValueError, match='scipy sparse'):
            f(np.zeros((2, 6)), emb)
        with pytest.raises(ValueError, match='shape'):
            f(sp.csr_matrix((2, 7)), emb)
        with pytest.raises(ValueError, match='outside'):
            f(sp.csr_matrix((np.ones(1), np.array([8]), np.array([0, 1, 1])), shape=(2, 6)), emb)
        with pytest.raises(ValueError, match='finite'):
            f(sp.csr_matrix((np.array([np.nan]), np.array([1]), np.array([0, 1, 1])), shape=(2, 6)), emb)
        with pytest.raises(ValueError, match='dense'):
            f(good, sp.csr_matrix(emb))
    with pytest.raises(ValueError, match='metric'):
        recommend(good, emb, metric='euclidean')
    for cand in ([3, 1], [1, 1], [0, 6], [-1, 2], [], [[1, 2]], [0.5, 1.0]):
        with pytest.raises(ValueError, match='candidates'):
            recommend(good, emb, candidates=np.asarray(cand))


def test_history_weights_are_normalised_per_user():
    from dae_rnn_news_recommendation_b200.helpers import _history_weights
    h = sp.csr_matrix(np.array([[1, 0, 3, 0], [0, 0, 0, 0], [2, 2, 0, 0], [0, 0, 0, 0]], np.float32))
    h = sp.vstack([h, sp.csr_matrix((np.array([0.0]), np.array([1]), np.array([0, 1])), shape=(1, 4))]).tocsr()  # explicit zero only
    w, empty = _history_weights(h, 4, 'f')
    assert np.allclose(w.toarray()[:4], [[0.25, 0, 0.75, 0], [0] * 4, [0.5, 0.5, 0, 0], [0] * 4])
    assert empty.tolist() == [False, True, False, True, True]
    assert w.indptr[-1] == 5 and w.indices[-1] == 1     # the zero-weight read stays in the structure (it is still excluded)


def test_candidate_remapping():
    from dae_rnn_news_recommendation_b200.helpers import _remap_lists
    cand = np.array([2, 5, 7, 9])
    indptr = np.array([0, 3, 3, 6, 8])
    indices = np.array([1, 5, 9, 0, 2, 7, 3, 4])   # rows: {1,5,9}, {}, {0,2,7}, {3,4}
    p, i = _remap_lists(indptr, indices, cand)
    assert p.tolist() == [0, 2, 2, 4, 4] and i.tolist() == [1, 3, 0, 2] and i.dtype == np.int32


def test_recommendation_recall_by_hand():
    from dae_rnn_news_recommendation_b200.helpers import recommendation_recall
    index = np.array([[3, 1, -1],     # targets {1, 4}: one of two -> hit, recall 1/2
                      [0, 2, 5],      # no target: skipped
                      [-1, -1, -1],   # targets {0}: padding is no hit -> 0
                      [5, 4, 0]])     # targets {0, 4, 5}: all three -> 1
    t = sp.csr_matrix((np.ones(6), (np.array([0, 0, 2, 3, 3, 3]), np.array([1, 4, 0, 0, 4, 5]))), shape=(4, 6))
    r = recommendation_recall(index, t)
    assert r == {'users': 3, 'hit_rate': pytest.approx(2 / 3), 'recall': pytest.approx((0.5 + 0 + 1) / 3)}
    r = recommendation_recall(index[1:2], t[1:2])
    assert r['users'] == 0 and np.isnan(r['hit_rate']) and np.isnan(r['recall'])
    with pytest.raises(ValueError, match='shape'):
        recommendation_recall(index, t[:3])
    with pytest.raises(ValueError, match='columns'):
        recommendation_recall(index, sp.csr_matrix((4, 5)))


def test_make_histories():
    from dae_rnn_news_recommendation_b200.synth import make_histories
    rng = np.random.default_rng(0)
    labels = rng.integers(0, 5, 3000)
    labels[:10] = -1
    h, t = make_histories(4000, labels, mean_len=20, seed=3, max_len=60)
    h2, t2 = make_histories(4000, labels, mean_len=20, seed=3, max_len=60)
    assert (h != h2).nnz == 0 and (t != t2).nnz == 0
    assert h.shape == t.shape == (4000, 3000) and h.dtype == np.float32
    assert h.has_canonical_format and (h.data == 1).all() and (t.data == 1).all()
    lens = np.diff(h.indptr)
    assert lens.max() <= 60 and 12 < lens.mean() < 22
    assert (np.diff(t.indptr) == 1).all()
    assert h.multiply(t).nnz == 0                       # a held-out read is not in the history
    assert h[:, :10].nnz == 0 and t[:, :10].nnz == 0    # unlabelled articles are never read
    # each user's reads concentrate on at most two classes
    hd = h.tocoo()
    per = sp.csr_matrix((np.ones(hd.nnz), (hd.row, labels[hd.col])), shape=(4000, 5)).toarray()
    top2 = -np.sort(-per, 1)[:, :2].sum(1)
    assert (top2 == per.sum(1)).all()
    # Zipf popularity: the most read article of a class is read far more than the median one
    counts = np.bincount(hd.col, minlength=3000)
    assert counts.max() > 20 * max(np.median(counts[counts > 0]), 1)
    h3, t3 = make_histories(50, labels, seed=1, holdout=False)
    assert t3 is None and (np.diff(h3.indptr) >= 1).all()


def test_user_flags(tmp_path):
    import main_autoencoder as cli
    p = cli.build_parser()
    F = p.parse_args([])
    assert F.user_histories == '' and F.user_targets == ''
    h = tmp_path / 'h.npz'
    sp.save_npz(h, sp.csr_matrix((3, 10), dtype=np.float32))
    F = cli.check_flags(p.parse_args(['--top_k', '5', '--user_histories', str(h), '--user_targets', str(h)]))
    assert F.user_histories == str(h)
    with pytest.raises(AssertionError, match='--top_k'):
        cli.check_flags(p.parse_args(['--user_histories', str(h)]))
    with pytest.raises(AssertionError, match='no such file'):
        cli.check_flags(p.parse_args(['--top_k', '5', '--user_histories', str(tmp_path / 'missing.npz')]))
    with pytest.raises(AssertionError, match='needs --user_histories'):
        cli.check_flags(p.parse_args(['--top_k', '5', '--user_targets', str(h)]))
    with pytest.raises(AssertionError, match='no such file'):
        cli.check_flags(p.parse_args(['--top_k', '5', '--user_histories', str(h), '--user_targets', str(tmp_path / 'x.npz')]))
    hs, ts = cli.load_user_files(F, 10)
    assert hs.shape == ts.shape == (3, 10)
    with pytest.raises(ValueError, match='training articles'):
        cli.load_user_files(F, 11)
    t4 = tmp_path / 't4.npz'
    sp.save_npz(t4, sp.csr_matrix((4, 10), dtype=np.float32))
    F.user_targets = str(t4)
    with pytest.raises(ValueError, match='users'):
        cli.load_user_files(F, 10)
