"""The references of tests/sparse_ranking_oracle.py checked on the host: the restated dispatch against the compiled workspace
queries, the postings checker against a direct construction, the score references against each other and the fp64 bound, the
partial-list model against the full answer, and the canonical form the helpers give the kernels."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import ranking_kernel_oracle as ro
import sparse_ranking_oracle as so
from test_auroc_hist_host import host_histograms
from topk_groups_oracle import _stream

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _sms():
    """The SM count the library's sm_count() sees: the device's when there is one, else its fallback of 132."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


@pytest.mark.parametrize('F', [1, 400, 1 << 24])
@pytest.mark.parametrize('n_corpus', [1, 2047, 2048, 2049, 70_000])
def test_layout_matches_the_workspace_queries(n_corpus, F):
    from dae_rnn_news_recommendation_b200 import _cabi
    nnz = 12345
    R = so._cdiv(n_corpus, so.SP_W)
    for n_query in (1, 5, 3000):
        for splits in (0, 1, 2, R, R + 1, 32, 33):
            for k in (1, 7, 32):
                L = so.sp_layout(n_query, n_corpus, nnz, F, k, splits, _sms())
                got = _cabi.query('dae_csr_similarity_topk_workspace', n_query, n_corpus, nnz, F, k, splits)
                assert got == L['total'], (n_query, splits, k, got, L)
                assert L['splits'] == max(1, min(R, 32, splits if splits > 0 else L['splits']))
        L = so.sp_layout(n_query, n_corpus, nnz, F, 0, 0, _sms())
        assert _cabi.query('dae_csr_similarity_pairs_workspace', n_query, n_corpus, nnz, F) == L['total']
        assert L['total'] == L['off_val']   # no lists
    if n_corpus >= 2:
        L = so.sp_layout(n_corpus, n_corpus, nnz, F, 0, 0, _sms())
        assert _cabi.query('dae_csr_similarity_pair_hist_workspace', n_corpus, nnz, F) == L['total']
    # the hashed-vocabulary case of the GPU tests: 8193 rows over 2^24 columns reach two pieces of the second scan level
    L = so.sp_layout(8193, 8193, 3000, 1 << 24, 0, 0)
    assert L['n_tiles'] == 10241 > so.SCAN_TILE and L['n_bucket'] * 4 > 335e6


def test_split_rows_cover_the_corpus():
    for nc in (1, 2047, 2049, 70_000):
        R = so._cdiv(nc, so.SP_W)
        for splits in {1, 2, 7, R, min(R, 32)}:
            s = min(splits, R)
            bounds = [so.split_rows(nc, s, t) for t in range(s)]
            assert bounds[0][0] == 0 and bounds[-1][1] == nc
            assert all(a[1] == b[0] for a, b in zip(bounds, bounds[1:]))
            assert all(c0 % so.SP_W == 0 and c1 > c0 for c0, c1 in bounds)


def test_postings_checker():
    rng = np.random.default_rng(0)
    c = so.edge_rows(rng, 4100, 9)
    starts = so.bucket_starts(c)
    keys = so.bucket_keys(c)
    assert starts[-1] == c.nnz and np.array_equal(np.diff(np.append(starts, c.nnz))[:-1], np.bincount(keys, minlength=starts.size)[:-1])
    # a legitimate posting array: entries placed by bucket, in a random order inside each bucket
    rows = np.repeat(np.arange(c.shape[0]), np.diff(c.indptr))
    post = np.zeros((c.nnz, 2), np.int32)
    order = np.lexsort((rng.random(c.nnz), keys))
    post[:, 0] = rows[order] % so.SP_W
    post[:, 1] = c.data.view(np.int32)[order]
    so.check_postings(c, starts, post)
    # each kind of corruption is caught
    bad = post.copy(); bad[[0, -1]] = bad[[-1, 0]]
    with pytest.raises(AssertionError):
        so.check_postings(c, starts, bad)
    bad = post.copy(); bad[3, 1] ^= 1
    with pytest.raises(AssertionError):
        so.check_postings(c, starts, bad)
    occ = np.unique(keys)[5]
    bad_s = starts.copy(); bad_s[occ + 1] += 1
    with pytest.raises(AssertionError):
        so.check_postings(c, bad_s, post)
    bad_s = starts.copy(); bad_s[occ + 1:occ + 1 + 3] = starts[occ]   # shift an empty run: no longer non-decreasing or off
    if not np.array_equal(bad_s, starts):
        with pytest.raises(AssertionError):
            so.check_postings(c, bad_s, post)
    # the tile area: one total, or the inclusive scan of several
    assert np.array_equal(so.tile_totals(c), [c.nnz])
    wide = so.edge_rows(rng, 4100, 3000)
    t = so.tile_totals(wide)
    full = so.bucket_starts(wide)
    assert t.size == 2 and t[-1] == wide.nnz and t[0] == full[so.SCAN_TILE]


@pytest.mark.parametrize('seed', [0, 1])
def test_dyadic_values_sum_exactly_in_any_order(seed):
    rng = np.random.default_rng(seed)
    x = so.dyadic_csr(rng, 60, 500, 0.5, dup=[(1, 2)], share_col=7)
    d = x.toarray().astype(np.float64)
    for a in range(0, 60, 7):
        for b in range(60):
            p = (d[a] * d[b]).astype(np.float32)       # exact products
            terms = p[p != 0]
            want = float(d[a] @ d[b])
            for order in (terms, terms[::-1], rng.permutation(terms)):
                acc = np.float32(0)
                for t in order:
                    acc = np.float32(acc + t)
                assert float(acc) == want
    S = so.f32_column_oracle(x, x)
    assert np.array_equal(S.astype(np.float64), d @ d.T)
    assert np.array_equal(S[1], S[2]) and (S[:, 0] == S[:, 5]).sum() > 0


def _tfidf(rng, n, F, nnz_row, least=0):
    rows = [np.sort(rng.choice(F, rng.integers(least, nnz_row + 1), replace=False)) for _ in range(n)]
    indptr = np.concatenate([[0], np.cumsum([r.size for r in rows])])
    data = (rng.random(indptr[-1]) * rng.choice([1, 1, 1, -1], indptr[-1]) * 2.0 ** rng.integers(-8, 8, indptr[-1])).astype(np.float32)
    return sp.csr_matrix((data, np.concatenate(rows).astype(np.int32), indptr), shape=(n, F))


def test_shared_column_oracle_is_bit_exact():
    rng = np.random.default_rng(3)
    for q, c in ((_tfidf(rng, 50, 300, 40), _tfidf(rng, 80, 300, 40)), (so.edge_rows(rng, 30, 17), so.edge_rows(rng, 45, 17))):
        a, b = so.f32_shared_oracle(q, c), so.f32_column_oracle(q, c)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    with np.errstate(invalid='ignore', over='ignore'):
        x = so.inf_rows()
        a, b = so.f32_shared_oracle(x, x), so.f32_column_oracle(x, x)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.isnan(a[0, 3]) and a[0, 1] == -np.inf and a[0, 4] == np.inf and a[1, 2] == -np.inf


def test_float32_scores_stay_within_half_the_bound():
    """Rows sharing at least ~50 columns: rounding errors of many terms partly cancel, far from the worst case the bound
    covers (with one shared column a single rounding can reach the whole bound)."""
    rng = np.random.default_rng(4)
    q, c = _tfidf(rng, 60, 200, 150, 120), _tfidf(rng, 90, 200, 150, 120)
    S32 = so.f32_column_oracle(q, c).astype(np.float64)
    S, bound = so.score_bound(q, c)
    nz = bound > 0
    assert np.array_equal(S32[~nz], S[~nz])
    ratio = np.abs(S32[nz] - S[nz]) / bound[nz]
    assert ratio.max() <= 0.5, ratio.max()


def test_sparse_pairs_and_histograms_match_the_dense_references():
    rng = np.random.default_rng(5)
    x = so.edge_rows(rng, 300, 23, dup=((3, 200), (10, 11)))
    S = so.f32_column_oracle(x, x)
    pi, pj, ps = so.sparse_self_pairs(x)
    dense = np.zeros_like(S)
    dense[pi, pj] = ps
    low = np.tril(np.ones(S.shape, bool), -1)
    assert np.array_equal(np.where(low, S, 0).view(np.uint32), dense.view(np.uint32))
    tau = float(np.sort(ps[ps > 0])[len(ps[ps > 0]) // 2])
    want = ro.pairs_set(S, tau, True)
    keep = ps >= tau
    assert np.array_equal(want[0], pi[keep]) and np.array_equal(want[1], pj[keep]) and np.array_equal(want[2], ps[keep])
    for labels in (rng.integers(-1, 4, 300), np.zeros(300, np.int64), np.full(300, -1)):
        for M, bins in ((1.0, 1 << 10), (2.0 ** -4, 1 << 24)):
            h, s, _, _ = host_histograms(S, labels, M, bins)
            h2, s2 = so.hist_from_pairs(300, labels, pi, pj, ps, M, bins)
            assert np.array_equal(h, h2) and np.array_equal(s, s2)


@pytest.mark.parametrize('k', [1, 7, 32])
def test_partial_lists_merge_to_the_answer(k):
    rng = np.random.default_rng(k)
    nq, nc = 9, 7000
    S = rng.integers(-3, 4, (nq, nc)).astype(np.float32)
    S[0, 100:300] = np.nan
    S[1, :] = -np.inf
    S[2, 4000:] = np.inf
    allowed = ro.allowed_mask(nq, nc, True, 2046, [[], [5], list(range(2048, 4096)), list(range(nc))])
    groups = rng.integers(0, 50, nc)
    for splits in (1, 2, 4):
        for g in (None, groups):
            pv, pi = so.partial_lists(S, k, splits, allowed, g)
            idx, val = ro.merge_lists(pv, pi, k, g)
            want = ro.top_k(S, k, allowed) if g is None else ro.top_k_groups(S, k, allowed, g)
            assert np.array_equal(idx, want[0]) and np.array_equal(val.view(np.uint32), want[1].view(np.uint32))
            if g is not None:
                # the grouped list of k lanes is the stream of sp_offer_group (kmax = k): the module docstring's argument
                for r in range(nq):
                    for s in range(splits):
                        c0, c1 = so.split_rows(nc, splits, s)
                        cols = [c for c in range(c0, c1) if allowed[r, c] and S[r, c] > -np.inf]
                        lst = _stream(S[r], cols, g, k, k)
                        assert [i for _, i in lst] == pi[r, s].tolist()
    assert (so.partial_lists(S, k, 3)[1][1] == -1).all()


def test_helpers_canonicalise_duplicate_columns():
    """The kernels need strictly increasing columns in every row (a repeated column would make two lanes add into one slot at
    once); _csr_operand and DeviceCSR hand them that form, duplicates summed and explicit zeros kept."""
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    from dae_rnn_news_recommendation_b200.helpers import _csr_operand
    data = np.array([1.0, 2.0, 0.0, 3.0, 4.0, -4.0], np.float32)
    indices = np.array([5, 2, 7, 5, 1, 1])
    indptr = np.array([0, 4, 6])
    m = sp.csr_matrix((data, indices, indptr), shape=(2, 9))
    assert not m.has_canonical_format
    for metric in ('linear kernel', 'cosine'):
        out = _csr_operand(m, metric)
        assert out.has_canonical_format and out.dtype == np.float32
        assert all((np.diff(out.indices[out.indptr[r]:out.indptr[r + 1]]) > 0).all() for r in range(2))
    out = _csr_operand(m, 'linear kernel')
    assert out.indices.tolist() == [2, 5, 7, 1] and out.data.tolist() == [2.0, 4.0, 0.0, 0.0]
    d = DeviceCSR(m, 'cpu')
    assert d.indptr.tolist() == [0, 3, 4] and d.indices.tolist() == [2, 5, 7, 1] and d.values.tolist() == [2.0, 4.0, 0.0, 0.0]
    assert m.indices.tolist() == indices.tolist()   # the caller's matrix is left as it was
