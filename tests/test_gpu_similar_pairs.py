"""similar_pairs / dae_similarity_pairs_bf16x3 / dae_csr_similarity_pairs: every pair at or above a threshold, checked exactly on
integer scores, bit for bit against top_k_similar and the float32 column oracle, against fp64, through the overflow protocol and at
100 000 rows."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from test_topk_sparse_host import f32_column_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _expected_pairs(s, tau, self_mode):
    """(i, j, s) of a score matrix with s >= tau (strict lower triangle in self mode), sorted by (i, j)."""
    hit = s >= tau
    if self_mode:
        hit = np.tril(hit, -1)
    i, j = np.nonzero(hit)
    return i.astype(np.int32), j.astype(np.int32), s[i, j]


def _assert_pairs_equal(got, want):
    assert got[0].dtype == np.int32 and got[1].dtype == np.int32 and got[2].dtype == np.float32
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert np.array_equal(got[2].view(np.int32), np.asarray(want[2], np.float32).view(np.int32))


def _clustered(n, h, seed, spread=0.35, per=4):
    """Rows in clusters of about `per` around random centres: intra-cluster cosine ~ 1 / (1 + spread^2)."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((max(1, n // per), h))
    lab = rng.integers(0, centres.shape[0], n)
    return (centres[lab] + spread * rng.standard_normal((n, h))).astype(np.float32), lab


@pytest.mark.parametrize('n', [2, 127, 128, 129, 1000, 3001])
@pytest.mark.parametrize('h', [16, 500])
def test_exact_small_integer_embeddings(n, h):
    """Small integers are exact in bf16 and their dot products in fp32, so the answer is known exactly; tau is a score that occurs,
    so ties at tau are included."""
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs
    rng = np.random.default_rng(n * 7 + h)
    x = rng.integers(-2, 3, (n, h)).astype(np.float32)
    y = rng.integers(-2, 3, (max(1, n // 3) + 5, h)).astype(np.float32)
    s = x.astype(np.int64) @ x.T.astype(np.int64)
    tau = float(np.quantile(s[np.tril_indices(n, -1)], 0.97, method='lower')) if n > 1 else 0.0
    got = similar_pairs(x, tau, metric='linear kernel')
    want = _expected_pairs(s.astype(np.float32), tau, True)
    _assert_pairs_equal(got, want)
    assert len(want[0]) > 0 and (want[2] == tau).any()
    sc = y.astype(np.int64) @ x.T.astype(np.int64)
    tau_c = float(np.quantile(sc, 0.97, method='lower'))
    _assert_pairs_equal(similar_pairs(y, tau_c, corpus=x, metric='linear kernel'), _expected_pairs(sc.astype(np.float32), tau_c, False))


def test_bit_consistency_with_top_k():
    """Every list entry of top_k_similar(k=32) at or above tau is a returned pair with the same score bits; where the 32nd score is
    below tau the list holds all of the row's pairs."""
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs, top_k_similar
    x, _ = _clustered(3000, 96, 1, per=6)
    rng = np.random.default_rng(2)
    x[::37] = rng.standard_normal(96) + 0.35 * rng.standard_normal((len(x[::37]), 96))   # one cluster of 82 rows: lists run full
    y = x[rng.permutation(3000)[:700]] + 0.2 * rng.standard_normal((700, 96)).astype(np.float32)
    tau = 0.8
    for q, corpus in ((x, None), (y, x)):
        idx, val = top_k_similar(q, k=32, corpus=corpus)
        pi, pj, ps = similar_pairs(q, tau, corpus=corpus)
        got = {}
        for a, b, s in zip(pi.tolist(), pj.tolist(), ps.view(np.int32).tolist()):
            got.setdefault(a, {})[b] = s
        full = subset = 0
        for r in range(q.shape[0]):
            keep = (val[r] >= tau) & (idx[r] >= 0)
            if corpus is None:
                keep &= idx[r] < r
            lst = dict(zip(idx[r][keep].tolist(), val[r][keep].view(np.int32).tolist()))
            mine = got.get(r, {})
            if val[r, 31] < tau:
                assert lst == mine, r
                full += 1
            else:
                assert all(mine.get(c) == v for c, v in lst.items()), r
                subset += 1
        assert full > 0 and subset > 0 and len(pi) > 0


@pytest.mark.parametrize('seed', [0, 1])
def test_random_clustered_cosine_against_fp64(seed):
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs
    x, _ = _clustered(4000, 200, seed)
    y = x[:900] + 0.2 * np.random.default_rng(seed + 10).standard_normal((900, 200)).astype(np.float32)
    tau = 0.85
    xn = x.astype(np.float64) / np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True)
    yn = y.astype(np.float64) / np.linalg.norm(y.astype(np.float64), axis=1, keepdims=True)
    for q, qn, corpus, self_mode in ((x, xn, None, True), (y, yn, x, False)):
        s64 = qn @ xn.T
        i, j, s = similar_pairs(q, tau, corpus=corpus)
        assert len(i) > 100
        if self_mode:
            assert (i > j).all()
        order = np.lexsort((j, i))
        assert np.array_equal(order, np.arange(len(i)))
        assert np.abs(s - s64[i, j]).max() <= 2e-5
        assert (s64[i, j] >= tau - 1e-5).all()
        must = s64 >= tau + 1e-5
        if self_mode:
            must = np.tril(must, -1)
        got = np.zeros_like(must)
        got[i, j] = True
        assert not (must & ~got).any()


def _operands(x):
    from dae_rnn_news_recommendation_b200.helpers import _normalised_operands
    return _normalised_operands(torch.from_numpy(x).cuda(), 2)


def test_overflow_counts_exactly_and_writes_nothing_past_capacity():
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs
    x, _ = _clustered(2000, 64, 5)
    tau = 0.8
    want = similar_pairs(x, tau)
    n = len(want[0])
    assert n > 300
    hi, lo, ld = _operands(x)
    for cap in (0, 1, 100, n - 1, n):
        guard = 64
        i = torch.full((cap + guard,), -7, dtype=torch.int32, device='cuda')
        j = torch.full((cap + guard,), -7, dtype=torch.int32, device='cuda')
        s = torch.full((cap + guard,), -7.0, dtype=torch.float32, device='cuda')
        count = torch.zeros(1, dtype=torch.int64, device='cuda')
        _cabi.call('dae_similarity_pairs_bf16x3', x.shape[0], x.shape[0], x.shape[1], hi.data_ptr(), lo.data_ptr(), ld, hi.data_ptr(),
                   lo.data_ptr(), ld, 1, tau, count.data_ptr(), cap, i.data_ptr(), j.data_ptr(), s.data_ptr(), None)
        assert int(count.item()) == n
        gi, gj, gs = i.cpu().numpy(), j.cpu().numpy(), s.cpu().numpy()
        assert (gi[cap:] == -7).all() and (gj[cap:] == -7).all() and (gs[cap:] == -7.0).all()
        wanted = {(a, b): v for a, b, v in zip(want[0].tolist(), want[1].tolist(), want[2].view(np.int32).tolist())}
        written = list(zip(gi[:cap].tolist(), gj[:cap].tolist(), gs[:cap].view(np.int32).tolist()))
        assert len(set((a, b) for a, b, _ in written)) == cap
        assert all(wanted.get((a, b)) == v for a, b, v in written)


def _counting_calls(monkeypatch, helpers, export):
    """Wrap helpers.call so that the calls of `export` are counted."""
    calls = []
    real = helpers.call

    def counting(name, *args):
        if name == export:
            calls.append(args)
        return real(name, *args)
    monkeypatch.setattr(helpers, 'call', counting)
    return calls


@pytest.mark.parametrize('kind', ['dense', 'sparse'])
def test_retry_and_max_pairs(monkeypatch, kind):
    """A first call with too few slots counts the pairs, and exactly one more call with `count` slots returns the full sorted set."""
    from dae_rnn_news_recommendation_b200 import helpers
    x, _ = _clustered(2000, 64, 5)
    export = 'dae_similarity_pairs_bf16x3'
    if kind == 'sparse':
        x = _with_near_copies(_binary(3000, 400, 0.02, 1), 0.2, 2)
        export = 'dae_csr_similarity_pairs'
    tau = 0.8 if kind == 'dense' else 0.5
    want = helpers.similar_pairs(x, tau)
    n = len(want[0])
    assert n > 100
    monkeypatch.setattr(helpers, 'SIMILAR_PAIRS_FIRST_CAPACITY', 50)
    monkeypatch.setattr(helpers, 'SIMILAR_PAIRS_SLOTS_PER_ROW', 0)
    calls = _counting_calls(monkeypatch, helpers, export)
    _assert_pairs_equal(helpers.similar_pairs(x, tau), want)
    cap_arg = -5   # (count, capacity, i, j, s, stream) close both exports' argument lists
    assert [c[cap_arg] for c in calls] == [50, n]
    del calls[:]
    _assert_pairs_equal(helpers.similar_pairs(x, tau, max_pairs=n), want)   # the first call may use all n slots
    assert [c[cap_arg] for c in calls] == [50, n]
    del calls[:]
    with pytest.raises(ValueError, match=r'%d pairs reach the threshold %r.*max_pairs = %d.*%d bytes' % (n, tau, n - 1, 12 * n)):
        helpers.similar_pairs(x, tau, max_pairs=n - 1)
    assert [c[cap_arg] for c in calls] == [50]
    monkeypatch.setattr(helpers, 'SIMILAR_PAIRS_FIRST_CAPACITY', 1 << 20)
    del calls[:]
    _assert_pairs_equal(helpers.similar_pairs(x, tau), want)                 # one call when the first capacity suffices
    assert [c[cap_arg] for c in calls] == [min(1 << 20, 1 << 28)]


def test_deterministic():
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs
    x, _ = _clustered(5000, 128, 9)
    a = similar_pairs(x, 0.7)
    b = similar_pairs(x, 0.7)
    assert len(a[0]) > 1000
    _assert_pairs_equal(a, b)
    xs = sp.csr_matrix(np.where(np.abs(x) > 1.0, x, 0.0).astype(np.float32))
    _assert_pairs_equal(similar_pairs(xs, 0.5), similar_pairs(xs, 0.5))


def _binary(n, f, density, seed):
    m = sp.random(n, f, density=density, format='csr', dtype=np.float32, random_state=seed)
    m.data[:] = 1.0
    return m


def _with_near_copies(m, frac, seed):
    """m plus perturbed copies of a fraction of its rows (so that near-duplicates exist), rows shuffled."""
    from dae_rnn_news_recommendation_b200.synth import perturb_rows
    rng = np.random.default_rng(seed)
    pick = rng.choice(m.shape[0], int(frac * m.shape[0]), replace=False)
    cp = perturb_rows(m[pick], frac=0.2, seed=seed)
    if m.data.size and not np.all(m.data == 1.0):
        from sklearn.preprocessing import normalize
        cp = normalize(cp)   # tf-idf-like: unit rows
    out = sp.vstack([m, cp]).tocsr()
    return out[rng.permutation(out.shape[0])].astype(np.float32)


@pytest.mark.parametrize('kind', ['binary', 'tfidf'])
@pytest.mark.parametrize('metric', ['cosine', 'linear kernel'])
def test_sparse_bit_exact_against_column_oracle(kind, metric):
    from dae_rnn_news_recommendation_b200.helpers import _csr_operand, similar_pairs
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    x = _binary(3000, 400, 0.02, 1) if kind == 'binary' else make_sparse(3000, 400, mean_nnz=12, kind='tfidf', seed=1)
    x = _with_near_copies(x, 0.1, 2)
    y = _with_near_copies(_binary(800, 400, 0.02, 3) if kind == 'binary' else make_sparse(800, 400, mean_nnz=12, kind='tfidf', seed=3),
                          0.1, 4)
    m, my = _csr_operand(x, metric), _csr_operand(y, metric)
    s = f32_column_oracle(m, m)
    tau = 0.5 if metric == 'cosine' or kind == 'tfidf' else 4.0
    want = _expected_pairs(s, np.float32(tau), True)
    assert len(want[0]) > 50
    _assert_pairs_equal(similar_pairs(x, tau, metric=metric), want)
    sc = f32_column_oracle(my, m)
    _assert_pairs_equal(similar_pairs(y, tau, corpus=x, metric=metric), _expected_pairs(sc, np.float32(tau), False))


def test_sparse_uci_c1_binary_cosine():
    from helpers import load_uci_c1
    from dae_rnn_news_recommendation_b200.helpers import _csr_operand, pair_label_agreement, similar_pairs
    d = load_uci_c1()
    x, v = d['train'], d['validate']
    m, mv = _csr_operand(x, 'cosine'), _csr_operand(v, 'cosine')
    s = f32_column_oracle(m, m)
    for tau in (0.5, 0.9):
        got = similar_pairs(x, tau)
        _assert_pairs_equal(got, _expected_pairs(s, np.float32(tau), True))
        agree = pair_label_agreement(got[0], got[1], d['train_label_story'])
        assert 0.0 <= agree['precision'] <= 1.0 and 0.0 <= agree['recall'] <= 1.0
    _assert_pairs_equal(similar_pairs(v, 0.5, corpus=x), _expected_pairs(f32_column_oracle(mv, m), np.float32(0.5), False))


def test_sparse_refuses_non_positive_threshold():
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs
    x = _binary(100, 50, 0.1, 0)
    for tau in (0.0, -0.1):
        with pytest.raises(ValueError, match='> 0'):
            similar_pairs(x, tau)


def _mem_above(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


SORT_SCRATCH = 8 << 20   # the radix sort's fixed workspace, the counter and allocator rounding


def _pairs_bound(p, n_q):
    """Device memory of similar_pairs beyond its operands or postings (DESIGN 4.8): the first call's c = max(2^20, 16 Nq) slots of
    12 B while the sort keys are built (12 c + 12 p), or the sort's two key and two score buffers (24 p), plus a constant."""
    from dae_rnn_news_recommendation_b200 import helpers
    c = max(helpers.SIMILAR_PAIRS_FIRST_CAPACITY, helpers.SIMILAR_PAIRS_SLOTS_PER_ROW * n_q)
    if p > c:   # the second call has exactly p slots
        return 24 * p + SORT_SCRATCH
    return max(12 * c + 12 * p, 24 * p) + SORT_SCRATCH


def test_full_size_dense_100k(monkeypatch):
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs
    n, h, tau = 100_000, 500, 0.75
    x, _ = _clustered(n, h, 3, spread=0.5, per=21)
    xd = torch.from_numpy(x).cuda()
    (i, j, s), extra = _mem_above(lambda: similar_pairs(xd, tau, to_host=False))
    p = i.shape[0]
    ld = (h + 7) // 8 * 8
    operands = 2 * n * ld * 2
    print('dense 100k: %d pairs, %.1f MB above the input (operands %.1f MB, bound %.1f MB)' % (
        p, extra / 1e6, operands / 1e6, (operands + _pairs_bound(p, n)) / 1e6))
    assert p > 2 * n
    assert extra <= operands + _pairs_bound(p, n)
    # with a small first call the peak is the sort's 24 B per pair
    monkeypatch.setattr(helpers, 'SIMILAR_PAIRS_FIRST_CAPACITY', 4096)
    monkeypatch.setattr(helpers, 'SIMILAR_PAIRS_SLOTS_PER_ROW', 0)
    got, extra2 = _mem_above(lambda: similar_pairs(xd, tau, to_host=False))
    print('dense 100k, second call: %.1f MB above the input (%.2f B per pair above the operands)' % (extra2 / 1e6, (extra2 - operands) / p))
    assert extra2 <= operands + 24 * p + SORT_SCRATCH
    assert all(torch.equal(a, b) for a, b in zip(got, (i, j, s)))
    del got
    i, j, s = i.cpu().numpy(), j.cpu().numpy(), s.cpu().numpy()
    xn = x.astype(np.float64) / np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True)
    rows = np.random.default_rng(0).choice(n, 48, replace=False)
    for r in rows:
        s64 = xn[r] @ xn[:r].T
        sel = i == r
        got = np.zeros(r, bool)
        got[j[sel]] = True
        assert not ((s64 >= tau + 1e-5) & ~got).any()
        assert (s64[j[sel]] >= tau - 1e-5).all() and np.abs(s[sel] - s64[j[sel]]).max(initial=0) <= 2e-5


def test_full_size_sparse_c2_like():
    from dae_rnn_news_recommendation_b200.helpers import _csr_operand, similar_pairs
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    x = _with_near_copies(make_sparse(95_000, 10_000, mean_nnz=40, kind='tfidf', seed=5), 5_000 / 95_000, 6)
    n, tau = x.shape[0], 0.6
    m = _csr_operand(x, 'linear kernel')
    (i, j, s), extra = _mem_above(lambda: similar_pairs(x, tau, metric='linear kernel', to_host=False))
    p = i.shape[0]
    postings = 8 * m.nnz + 4 * ((n + 2047) // 2048 * m.shape[1] + 1) + (12 + 4) * m.nnz + 8 * (n + 1)   # + the device CSR
    print('sparse 100k: %d pairs, %.1f MB above the input (postings and CSR %.1f MB)' % (p, extra / 1e6, postings / 1e6))
    assert p > 1000
    assert extra <= postings + _pairs_bound(p, n)
    i, j, s = i.cpu().numpy(), j.cpu().numpy(), s.cpu().numpy()
    rows = np.random.default_rng(1).choice(n, 32, replace=False)
    want = f32_column_oracle(m[rows], m)
    for t, r in enumerate(rows):
        sel = i == r
        w = np.nonzero(want[t, :r] >= np.float32(tau))[0]
        assert np.array_equal(j[sel], w)
        assert np.array_equal(s[sel].view(np.int32), want[t, w].view(np.int32))


def test_cli_dedup_on_synthetic(capsys):
    import re
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs
    argv = ['--model_name', 'syndedup', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--dedup_threshold', '0.95', '--dedup_input']
    model = cli.main(argv)
    printed = capsys.readouterr().out
    ev = model.evaluation
    num = r'(\d+) pairs, (\d+) groups of >= 2 articles, label precision ([0-9.]+|nan) recall ([0-9.]+|nan)'
    for split in ('', '_validate'):
        e, d = ev['duplicates' + split], ev['duplicates_input' + split]
        m = re.search(r'^duplicates%s: %s$' % (split, num), printed, re.M)
        assert m and (int(m.group(1)), int(m.group(2))) == (e['pairs'], e['groups'])
        m = re.search(r'^duplicates_input%s: %s  \(embedding: (\d+) pairs, (\d+) groups, precision ([0-9.]+|nan) recall ([0-9.]+|nan)\)$'
                      % (split, num), printed, re.M)
        assert m, printed
        assert (int(m.group(1)), int(m.group(2)), int(m.group(5)), int(m.group(6))) == (d['pairs'], d['groups'], e['pairs'], e['groups'])
        for g, v in ((3, d['precision']), (4, d['recall']), (7, e['precision']), (8, e['recall'])):
            assert m.group(g) == '%.4f' % v
    trX, vlX, _, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    for split, n in (('', 960), ('_validate', 240)):
        for key in ('duplicates', 'duplicates_input'):
            z = np.load(model.data_dir + 'article_%s%s.npz' % (key, split))
            assert z['group'].shape == (n,) and z['group'].dtype == np.int32
            assert z['i'].shape == z['j'].shape == z['score'].shape and (z['score'] >= np.float32(0.95)).all()
            assert ev[key + split]['pairs'] == len(z['i'])
        z = np.load(model.data_dir + 'article_duplicates_input%s.npz' % split)
        want = similar_pairs(trX if split == '' else vlX, 0.95, corpus=None if split == '' else trX, metric='cosine')
        assert np.array_equal(z['i'], want[0]) and np.array_equal(z['j'], want[1])
