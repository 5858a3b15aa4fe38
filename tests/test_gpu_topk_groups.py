"""top_k_similar(groups=...) / recommend(groups=...) / dae_*_topk_groups*: at most one row per group in the top-k lists, checked bit
for bit against the host oracle (tests/topk_groups_oracle.py) on exact integer scores and on the kernels' own score bits."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from test_topk_sparse_host import f32_column_oracle
from topk_groups_oracle import grouped_top_k

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _eq(got, want, msg=None):
    assert np.array_equal(got[0], want[0]), msg
    assert np.array_equal(got[1], want[1]), msg


def _self_allowed(n):
    return ~np.eye(n, dtype=bool)


# pairs of exact duplicates in one group: across the 64-column halves, the 128-column tiles, a split boundary and the sparse
# 2048-row ranges, and inside one dense partial list (same half of a tile: the later, equal score must not replace the earlier)
DUPS = ((63, 64), (127, 128), (120, 300), (2047, 2048), (5, 999), (10, 20), (11, 139), (200, 1864), (30, 35))


def _straddling_groups(n, rng, n_groups):
    """Random labels (members spread over the halves, tiles, splits and ranges) plus the DUPS pairs and the two middle rows."""
    g = rng.integers(0, n_groups, n)
    for a, b in DUPS + ((n // 2 - 1, n // 2), (5, n - 1)):
        if b < n:
            g[b] = g[a]
    return g


def _int_dense(n, h, rng, dup_pairs):
    x = rng.integers(-2, 3, (n, h)).astype(np.float32)
    for a, b in dup_pairs:                       # exact ties inside a group (the lower index represents it)
        if b < n:
            x[b] = x[a]
    return x


@pytest.mark.parametrize('k', [1, 5, 10, 17, 32])
def test_exact_ties_dense(k):
    """Small-integer embeddings, linear kernel: every bf16x3 score is the exact integer dot product."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(k)
    c = _int_dense(2300, 24, rng, DUPS)
    q = np.concatenate([c[:40], _int_dense(200, 24, rng, ())])
    g = _straddling_groups(2300, rng, 150)
    s = q.astype(np.float64) @ c.T.astype(np.float64)
    want = grouped_top_k(s, g, k)
    for splits in (1, 3, 0):
        _eq(top_k_similar(q, k=k, corpus=c, metric='linear kernel', groups=g, splits=splits), want, splits)
    cs = c[:700]
    gs = g[:700]
    s = cs.astype(np.float64) @ cs.T.astype(np.float64)
    _eq(top_k_similar(cs, k=k, metric='linear kernel', groups=gs), grouped_top_k(s, gs, k, _self_allowed(700)))


@pytest.mark.parametrize('k', [1, 7, 10, 32])
def test_exact_ties_sparse(k):
    """Binary rows, linear kernel: every score is a small integer overlap; 5 000 corpus rows span three 2048-row ranges."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(10 + k)
    c = sp.random(5000, 300, density=0.03, format='csr', dtype=np.float32, random_state=k).tolil()
    for a, b in DUPS:
        c[b] = c[a]
    c = c.tocsr()
    c.data[:] = 1.0
    q = sp.vstack([c[:30], sp.random(150, 300, density=0.03, format='csr', dtype=np.float32, random_state=k + 1)]).tocsr()
    q.data[:] = 1.0
    g = _straddling_groups(5000, rng, 400)
    s = (q.astype(np.int64) @ c.astype(np.int64).T).toarray().astype(np.float64)
    want = grouped_top_k(s, g, k)
    for splits in (1, 3, 0):
        _eq(top_k_similar(q, k=k, corpus=c, metric='linear kernel', groups=g, splits=splits), want, splits)
    s = (c[:900].astype(np.int64) @ c[:900].astype(np.int64).T).toarray().astype(np.float64)
    _eq(top_k_similar(c[:900], k=k, metric='linear kernel', groups=g[:900]), grouped_top_k(s, g[:900], k, _self_allowed(900)))


@pytest.mark.parametrize('k', [3, 10, 20])
def test_one_group_and_fewer_groups_than_k(k):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(30)
    c = _int_dense(900, 16, rng, DUPS)
    q = _int_dense(50, 16, rng, ())
    cs = sp.csr_matrix(np.maximum(c, 0))
    qs = sp.csr_matrix(np.maximum(q, 0))
    for g in (np.zeros(900, np.int64), rng.integers(0, 3, 900), np.repeat(np.arange(5), 180)):
        for qq, cc in ((q, c), (qs, cs)):
            qd = qq.toarray() if sp.issparse(qq) else qq
            cd = cc.toarray() if sp.issparse(cc) else cc
            want = grouped_top_k(qd.astype(np.float64) @ cd.T.astype(np.float64), g, k)
            n_g = np.unique(g).size
            assert (want[0][:, n_g:] == -1).all() and (want[0][:, :min(n_g, k)] >= 0).all()
            for splits in (1, 0):
                _eq(top_k_similar(qq, k=k, corpus=cc, metric='linear kernel', groups=g, splits=splits), want)


def _clustered(n, h, n_clusters, rng, spread=0.15):
    centres = rng.standard_normal((n_clusters, h))
    lab = rng.integers(0, n_clusters, n)
    return (centres[lab] + spread * rng.standard_normal((n, h))).astype(np.float32), lab


@pytest.mark.parametrize('k', [10, 32])
def test_random_dense_against_the_kernels_score_bits(k):
    """Cosine on random clustered embeddings: the scores are the kernel's own bits, read back through similar_pairs with a
    threshold below every score (the same bf16x3 scores as top_k_similar)."""
    from dae_rnn_news_recommendation_b200.helpers import duplicate_groups, similar_pairs, top_k_similar
    rng = np.random.default_rng(40 + k)
    c, _ = _clustered(3000, 100, 140, rng)
    q, _ = _clustered(300, 100, 140, rng)
    i, j, _ = similar_pairs(c, 0.95)
    g = duplicate_groups(i, j, 3000)
    assert np.unique(g).size < 2000                     # real groups
    i, j, v = similar_pairs(q, -2.0, corpus=c)
    s = np.full((300, 3000), np.nan, np.float32)
    s[i, j] = v
    assert not np.isnan(s).any()
    want = grouped_top_k(s, g, k)
    for splits in (1, 5, 0):
        _eq(top_k_similar(q, k=k, corpus=c, groups=g, splits=splits), want, splits)
    i, j, v = similar_pairs(c[:800], -2.0, corpus=c)
    s = np.full((800, 3000), np.nan, np.float32)
    s[i, j] = v
    allowed = np.ones((800, 3000), bool)
    allowed[np.arange(800), np.arange(800)] = False
    idx, val = top_k_similar(c, k=k, groups=g)
    _eq((idx[:800], val[:800]), grouped_top_k(s, g, k, allowed))


@pytest.mark.parametrize('k', [1, 10, 32])
def test_random_sparse_against_the_float32_oracle(k):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    rng = np.random.default_rng(50 + k)
    c = make_sparse(4500, 700, mean_nnz=25, kind='tfidf', seed=k).astype(np.float32)
    q = make_sparse(600, 700, mean_nnz=25, kind='tfidf', seed=k + 100).astype(np.float32)
    g = _straddling_groups(4500, rng, 600)
    want = grouped_top_k(f32_column_oracle(q, c), g, k)
    _eq(top_k_similar(q, k=k, corpus=c, metric='linear kernel', groups=g), want)
    s = f32_column_oracle(c, c)
    _eq(top_k_similar(c, k=k, metric='linear kernel', groups=g), grouped_top_k(s, g, k, _self_allowed(4500)))


def _exclusions(nq, nc, seed, density=0.02):
    return sp.random(nq, nc, density=density, format='csr', random_state=seed)


@pytest.mark.parametrize('k', [10, 32])
def test_identity_groups_are_the_plain_call_bit_for_bit(k):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    rng = np.random.default_rng(60 + k)
    c, _ = _clustered(2500, 64, 30, rng, spread=0.5)
    q, _ = _clustered(400, 64, 30, rng, spread=0.5)
    cs = make_sparse(4500, 500, mean_nnz=20, kind='tfidf', seed=k).astype(np.float32)
    qs = cs[:400]
    for qq, cc in ((q, c), (qs, cs)):
        ar = np.arange(cc.shape[0])
        _eq(top_k_similar(qq, k=k, corpus=cc, groups=ar), top_k_similar(qq, k=k, corpus=cc))
        _eq(top_k_similar(cc, k=k, groups=ar), top_k_similar(cc, k=k))
        ex = _exclusions(qq.shape[0], cc.shape[0], k)
        _eq(top_k_similar(qq, k=k, corpus=cc, groups=ar, exclude=ex), top_k_similar(qq, k=k, corpus=cc, exclude=ex))
        ex = _exclusions(cc.shape[0], cc.shape[0], k + 1)
        _eq(top_k_similar(cc, k=k, groups=ar, exclude=ex), top_k_similar(cc, k=k, exclude=ex))


def test_splits_do_not_change_the_result():
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    rng = np.random.default_rng(70)
    c, lab = _clustered(6000, 48, 60, rng, spread=0.3)
    g = np.where(rng.random(6000) < 0.5, lab, 1000 + np.arange(6000))
    q = c[:300]
    ref = top_k_similar(q, k=10, corpus=c, groups=g, splits=1)
    for s in list(range(2, 9)) + [11, 16, 23, 31, 32, 0]:
        _eq(top_k_similar(q, k=10, corpus=c, groups=g, splits=s), ref, s)
    cs = make_sparse(9000, 400, mean_nnz=20, kind='tfidf', seed=71).astype(np.float32)
    gs = rng.integers(0, 500, 9000)
    ref = top_k_similar(cs[:300], k=10, corpus=cs, metric='linear kernel', groups=gs, splits=1)
    _eq(ref, grouped_top_k(f32_column_oracle(cs[:300], cs), gs, 10))
    for s in (2, 3, 4, 5, 0):
        _eq(top_k_similar(cs[:300], k=10, corpus=cs, metric='linear kernel', groups=gs, splits=s), ref, s)


def test_groups_and_exclusion_lists():
    """An excluded best member hands its group to the next member; in self mode the query's own group stays a candidate unless
    its members are listed in `exclude`."""
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    rng = np.random.default_rng(80)
    for sparse in (False, True):
        c = np.maximum(_int_dense(1500, 20, rng, DUPS), 0)
        cc = sp.csr_matrix(c) if sparse else c
        g = _straddling_groups(1500, rng, 100)
        s = c.astype(np.float64) @ c.T.astype(np.float64)
        ex = _exclusions(1500, 1500, 81, density=0.05).tolil()
        plain = top_k_similar(cc, k=10, metric='linear kernel', groups=g)
        for r in range(0, 1500, 50):        # exclude each sampled row's best representative
            ex[r, plain[0][r, 0]] = 1.0
        ex = ex.tocsr()
        allowed = (ex.toarray() == 0) & _self_allowed(1500)
        got = top_k_similar(cc, k=10, metric='linear kernel', groups=g, exclude=ex)
        _eq(got, grouped_top_k(s, g, 10, allowed))
        for r in range(0, 1500, 50):
            assert plain[0][r, 0] not in got[0][r]
        # self mode: the own group's other members are candidates ...
        same = g[plain[0]] == g[:, None]
        assert same[plain[0] >= 0].any()
        # ... and leave when listed
        own = sp.csr_matrix(g[:, None] == g[None, :])
        got = top_k_similar(cc, k=10, metric='linear kernel', groups=g, exclude=own)
        assert not (g[np.maximum(got[0], 0)] == g[:, None])[got[0] >= 0].any()
        _eq(got, grouped_top_k(s, g, 10, ~(g[:, None] == g[None, :])))


def _users(n_users, n, rng, mean_len=6):
    lens = rng.geometric(1.0 / mean_len, n_users)
    lens[:3] = 0                                          # users without reads: padding rows
    rows = np.repeat(np.arange(n_users), lens)
    cols = rng.integers(0, n, rows.size)
    h = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=(n_users, n))
    h.sum_duplicates()
    return h


def _profile_scores(h, emb, corpus):
    """The cosine scores recommend ranks, as the kernel computes them: similar_pairs of the same profiles and corpus."""
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs, user_profiles
    prof = user_profiles(h, emb)
    i, j, v = similar_pairs(prof, -2.0, corpus=corpus)
    s = np.full((h.shape[0], corpus.shape[0]), -np.inf, np.float32)
    s[i, j] = v
    return s


def test_recommend_with_groups():
    from dae_rnn_news_recommendation_b200.helpers import recommend
    rng = np.random.default_rng(90)
    n = 3000
    emb, lab = _clustered(n, 64, 40, rng, spread=0.4)
    g = rng.integers(0, 600, n)
    h = _users(500, n, rng).tolil()
    first = np.array([np.flatnonzero(g == grp)[0] for grp in np.unique(g)])
    h[7, first[::2]] = 1.0                                    # user 7 has read half of the groups,
    h[8, first] = 1.0                                         # user 8 every group: a padding row
    h = h.tocsr()
    idx, val = recommend(h, emb, k=10, groups=g)
    hd = h.toarray() != 0
    read_groups = np.zeros((500, g.max() + 1), bool)
    rr, cc = np.nonzero(hd)
    read_groups[rr, g[cc]] = True
    allowed = ~read_groups[:, g]
    s = _profile_scores(h, emb, emb)
    want = grouped_top_k(s, g, 10, allowed)
    want[0][:3], want[1][:3] = -1, -np.inf
    _eq((idx, val), want)
    ok = idx >= 0
    assert not np.take_along_axis(hd, np.maximum(idx, 0), 1)[ok].any()                  # no read article
    assert np.take_along_axis(allowed, np.maximum(idx, 0), 1)[ok].all()                  # no article of a read group
    for r in range(500):
        gr = g[idx[r][idx[r] >= 0]]
        assert np.unique(gr).size == gr.size                                               # one per group
    assert (idx[8] == -1).all() and (val[8] == -np.inf).all()
    assert (idx[:3] == -1).all()
    assert (idx[7] >= 0).all()
    # candidates: only those rows, group labels taken from them, read groups still out
    cand = np.sort(rng.choice(n, 1200, replace=False))
    idx_c, val_c = recommend(h, emb, k=10, groups=g, candidates=cand)
    s = _profile_scores(h, emb, emb[cand])
    want = grouped_top_k(s, g[cand], 10, allowed[:, cand])
    want_i = np.where(want[0] >= 0, cand[np.maximum(want[0], 0)], -1)
    want_i[:3] = -1
    want[1][:3] = -np.inf
    _eq((idx_c, val_c), (want_i, want[1]))
    # exclude_read=False: groups only
    idx_n, val_n = recommend(h, emb, k=10, groups=g, exclude_read=False)
    want = grouped_top_k(_profile_scores(h, emb, emb), g, 10)
    want[0][:3], want[1][:3] = -1, -np.inf
    _eq((idx_n, val_n), want)
    # identity groups: the plain call
    _eq(recommend(h, emb, k=10, groups=np.arange(n)), recommend(h, emb, k=10))


def test_user_gru_passes_groups_through():
    from dae_rnn_news_recommendation_b200.helpers import recommend
    from dae_rnn_news_recommendation_b200.user_model import UserGRU, history_matrix
    rng = np.random.default_rng(95)
    n, h_dim = 1500, 32
    emb, _ = _clustered(n, h_dim, 20, rng, spread=0.5)
    g = rng.integers(0, 300, n)
    lens = rng.integers(1, 12, 200)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, n, int(lens.sum())).astype(np.int32)
    m = UserGRU(h_dim, max_len=10, seed=0, num_epochs=1).fit((indptr, items), emb)
    got = m.recommend((indptr, items), emb, k=10, groups=g)
    prof = m.transform((indptr, items), emb)
    want = recommend(history_matrix(indptr, items, n), emb, k=10, metric='linear kernel', profiles=prof, groups=g)
    _eq(got, want)
    assert not np.array_equal(got[0], m.recommend((indptr, items), emb, k=10)[0])


def test_100k_rows_dense_and_sparse_self_search():
    """100 000 rows: a dense clustered self search (H = 128) and a C2-like sparse one (10 000 tf-idf columns), both with clustered
    groups; the device memory above the inputs stays at the plain call's, and sampled rows match the oracle bit for bit."""
    import torch
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    rng = np.random.default_rng(100)
    n = 100000
    x, lab = _clustered(n, 128, 4000, rng, spread=0.2)
    g = np.where(rng.random(n) < 0.8, lab, 5000 + np.arange(n))
    xd = torch.from_numpy(x).cuda()
    peaks = []
    for groups in (None, g):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        idx, val = helpers.top_k_similar(xd, k=10, groups=groups, to_host=False)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
    assert peaks[1] <= peaks[0] + 4 * n + (2 << 20), peaks
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    rows = np.sort(rng.choice(n, 48, replace=False))
    i, j, v = helpers.similar_pairs(x[rows], -2.0, corpus=x)
    s = np.full((48, n), np.nan, np.float32)
    s[i, j] = v
    allowed = np.ones((48, n), bool)
    allowed[np.arange(48), rows] = False
    _eq((idx[rows], val[rows]), grouped_top_k(s, g, 10, allowed))
    gi = g[idx[rows]]
    assert all(np.unique(r).size == 10 for r in gi)

    xs = make_sparse(n, 10000, mean_nnz=100, kind='tfidf', seed=101)
    gs = rng.integers(0, n // 20, n)
    d = DeviceCSR(xs, 'cuda:0')
    gd = torch.from_numpy(gs.astype(np.int32)).cuda()
    peaks = []
    for groups in (None, gd):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        idx, val = helpers._csr_similarity_topk(d, d, 10, exclude=True, groups=groups)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
    assert peaks[1] <= peaks[0] + (2 << 20), peaks
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    rows = np.sort(rng.choice(n, 32, replace=False))
    s = f32_column_oracle(xs[rows], xs)
    allowed = np.ones((32, n), bool)
    allowed[np.arange(32), rows] = False
    _eq((idx[rows], val[rows]), grouped_top_k(s, gs, 10, allowed))


def test_cli_top_k_dedup_on_synthetic(capsys, tmp_path):
    import re
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.helpers import (duplicate_groups, label_precision_at_k, recommend,
                                                          recommendation_recall, similar_pairs, top_k_similar)
    from dae_rnn_news_recommendation_b200.synth import make_histories
    argv = ['--model_name', 'syndedup', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--top_k', '5']
    trX, _, trL, vlL = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    h, t = make_histories(300, trL, mean_len=8, seed=4)
    sp.save_npz(tmp_path / 'h.npz', h)
    sp.save_npz(tmp_path / 't.npz', t)
    model = cli.main(argv + ['--top_k_dedup', '0.9', '--user_histories', str(tmp_path / 'h.npz'),
                             '--user_targets', str(tmp_path / 't.npz')])
    printed = capsys.readouterr().out
    ev = model.evaluation
    enc = np.load(model.data_dir + 'article_encoded.npy') if os.path.exists(model.data_dir + 'article_encoded.npy') else None
    for split, n in (('', 960), ('_validate', 240)):
        idx = np.load(model.data_dir + 'article_top_k_dedup_index%s.npy' % split)
        score = np.load(model.data_dir + 'article_top_k_dedup_score%s.npy' % split)
        assert idx.shape == score.shape == (n, 5) and idx.dtype == np.int32
        assert np.array_equal(idx, ev['top_k_dedup' + split][0])
        lab = trL if split == '' else vlL
        assert ev['top_k_dedup_precision' + split] == label_precision_at_k(idx, lab, trL)
        m = re.search(r'top 5%s label precision: one per group ([0-9.]+)  plain ([0-9.]+)' % split, printed)
        assert m and m.group(1) == '%.4f' % ev['top_k_dedup_precision' + split]
        assert m.group(2) == '%.4f' % ev['top_k_precision' + split]
    uidx = np.load(model.data_dir + 'user_top_k_dedup_index.npy')
    assert uidx.shape == np.load(model.data_dir + 'user_top_k_dedup_score.npy').shape == (300, 5)
    r = recommendation_recall(uidx, t)
    assert ev['user_dedup_hit_rate'] == r['hit_rate'] and ev['user_dedup_recall'] == r['recall']
    m = re.search(r'users, one per group: hit rate@5 ([0-9.]+) recall@5 ([0-9.]+)', printed)
    assert m and m.group(1) == '%.4f' % r['hit_rate']
    assert not np.take_along_axis(h.toarray() > 0, np.maximum(uidx, 0), 1)[uidx >= 0].any()
    # the saved lists are the helpers' for the run's own embeddings
    plain = np.load(model.data_dir + 'article_top_k_index.npy')
    assert plain.shape == (960, 5)
    if enc is not None:
        i, j, _ = similar_pairs(enc, 0.9)
        g = duplicate_groups(i, j, enc.shape[0])
        _eq(top_k_similar(enc, k=5, groups=g), (np.load(model.data_dir + 'article_top_k_dedup_index.npy'),
                                                 np.load(model.data_dir + 'article_top_k_dedup_score.npy')))
        _eq(recommend(h, enc, k=5, groups=g), (uidx, np.load(model.data_dir + 'user_top_k_dedup_score.npy')))
