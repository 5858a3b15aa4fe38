"""References for the sparse ranking kernels of csrc/similarity_sparse.cu (dae_csr_similarity_topk / _excl / _groups,
dae_csr_similarity_pairs, dae_csr_similarity_pair_hist and their *_workspace queries), for the kernel-level tests.  Tests only;
nothing here needs a GPU.

Dispatch.  sp_splits / sp_layout restate the host side: the corpus is cut into ranges of SP_W = 2048 rows, split s of S covers
ranges [s R / S, (s + 1) R / S), and the workspace holds, 16-byte aligned in this order, the bucket starts (R F + 1 int32), the
scan's tile totals, the postings (8 B per corpus entry) and, with S > 1, the partial lists (n_query S k values, then indices).

Postings.  Bucket b = range * F + column.  After the call the bucket array holds the exclusive starts of the buckets in b order,
its last entry the corpus nnz; bucket b's postings are the multiset {(row - 2048 range, value bits)} of its entries, in an
unspecified order (atomic slots), so they are compared sorted.  check_postings() checks both without an R F host array.

Scores.  test_topk_sparse_host.f32_column_oracle is the bit-exact specification; f32_shared_oracle gives the same bits visiting only
the columns present in both operands (a 2^24-column vocabulary).  score_bound() is the fp64 reference with its error bound.

Partial lists.  The kernel's warp for (q, split) keeps exactly k lanes and offers the split's slots in increasing corpus index;
only a strict v > (k-th score) inserts, at the position after every listed entry scoring >= v.  Each listed entry therefore
beats every rejected or evicted candidate in (score desc, index asc) order, and the list after the last offer is the exact top k
of the split's candidates in that order (a NaN or -inf score never passes v > thr, so it is never a candidate).  With groups,
sp_offer_group keeps one entry per group: a candidate whose group is listed replaces that entry only when it scores strictly
more (an equal score has a higher index), and an evicted group's entry scored at most the k-th score, so any later member that
gets in beats it.  The list is then the exact grouped top k of the split's candidates (topk_groups_oracle._stream with
kmax = k streams the same list).  partial_lists() gives those lists; merge_lists() of them is the full answer.
"""
import numpy as np
import scipy.sparse as sp

from ranking_kernel_oracle import allowed_mask, merge_lists, pairs_set, top_k, top_k_groups  # noqa: F401
from test_topk_sparse_host import f32_column_oracle  # noqa: F401

SP_W = 2048
SP_MAX_K = 32
SP_MAX_SPLITS = 32
SP_WARPS_PER_SM = 24
SCAN_TILE = 8192
U32 = 2.0 ** -24   # unit roundoff of fp32


def _cdiv(a, b):
    return -(-a // b)


def _align16(b):
    return _cdiv(b, 16) * 16


# ---------------------------------------------------------------------------------------------------------------------------
# host dispatch (similarity_sparse.cu: sp_splits, sp_layout)
# ---------------------------------------------------------------------------------------------------------------------------
def sp_splits(n_query, ranges, requested, sms=132):
    s = requested
    if s <= 0:
        s = _cdiv(sms * SP_WARPS_PER_SM, n_query)
    return max(min(s, ranges, SP_MAX_SPLITS), 1)


def sp_layout(n_query, n_corpus, corpus_nnz, F, k, splits, sms=132):
    """dict: ranges, splits, n_bucket, n_tiles and the byte offsets off_tiles, off_post, off_val, off_idx, total.  The pairs and
    histogram exports use k = 0 (no lists) and splits = 0."""
    ranges = _cdiv(n_corpus, SP_W)
    s = sp_splits(n_query, ranges, splits, sms)
    n_bucket = ranges * F + 1
    n_tiles = _cdiv(n_bucket, SCAN_TILE)
    off_tiles = _align16(n_bucket * 4)
    off_post = off_tiles + _align16(n_tiles * 4)
    off_val = off_post + _align16(corpus_nnz * 8)
    lists = n_query * s * k if s > 1 else 0
    off_idx = off_val + _align16(lists * 4)
    return dict(ranges=ranges, splits=s, n_bucket=n_bucket, n_tiles=n_tiles, off_tiles=off_tiles, off_post=off_post,
                off_val=off_val, off_idx=off_idx, total=off_idx + _align16(lists * 4))


def split_rows(n_corpus, splits, s):
    """[c0, c1): the corpus rows of split s."""
    ranges = _cdiv(n_corpus, SP_W)
    return s * ranges // splits * SP_W, min((s + 1) * ranges // splits * SP_W, n_corpus)


# ---------------------------------------------------------------------------------------------------------------------------
# postings
# ---------------------------------------------------------------------------------------------------------------------------
def bucket_keys(c):
    """int64 [nnz]: the bucket (row // 2048) F + column of every stored entry of the CSR matrix c, in storage order."""
    rows = np.repeat(np.arange(c.shape[0], dtype=np.int64), np.diff(c.indptr))
    return rows // SP_W * c.shape[1] + c.indices.astype(np.int64)


def bucket_starts(c):
    """int32 [R F + 1]: the exclusive bucket starts, last = nnz (an R F host array: small shapes only)."""
    n_bucket = _cdiv(c.shape[0], SP_W) * c.shape[1] + 1
    counts = np.bincount(bucket_keys(c), minlength=n_bucket)
    return np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32)


def tile_totals(c):
    """int32 [n_tiles]: what the scan leaves in the tile area -- entry t is the number of entries in buckets below
    min((t + 1) 8192, R F + 1): one tile's total, or with several tiles their inclusive scan."""
    n_bucket = _cdiv(c.shape[0], SP_W) * c.shape[1] + 1
    ends = np.minimum(np.arange(1, _cdiv(n_bucket, SCAN_TILE) + 1, dtype=np.int64) * SCAN_TILE, n_bucket)
    return np.searchsorted(np.sort(bucket_keys(c)), ends).astype(np.int32)


def check_postings(c, starts, post):
    """Raise AssertionError unless starts (int32 [R F + 1]) are c's bucket starts and post (int32 [nnz, 2]) holds each bucket's
    (row offset, value bits) multiset in its slice.  Memory O(nnz + R F / 8): the starts are checked as a non-decreasing step
    function with the right steps at the occupied buckets, which pins every entry."""
    keys = bucket_keys(c)
    nnz = keys.size
    n_bucket = _cdiv(c.shape[0], SP_W) * c.shape[1] + 1
    assert starts.shape == (n_bucket,) and starts[0] == 0 and starts[-1] == nnz, 'bucket ends: %r %r' % (starts[0], starts[-1])
    assert not (np.diff(starts) < 0).any(), 'bucket starts decrease'
    occ, first, cnt = np.unique(np.sort(keys), return_index=True, return_counts=True)
    bad = (starts[occ] != first) | (starts[occ + 1] != first + cnt)
    assert not bad.any(), 'bucket %d starts at %d, %d expected' % (occ[bad][0], starts[occ[bad][0]], first[bad][0])
    rows = np.repeat(np.arange(c.shape[0], dtype=np.int64), np.diff(c.indptr))
    want = np.stack([rows % SP_W, np.asarray(c.data, np.float32).view(np.int32).astype(np.int64)], 1)
    order = np.lexsort((want[:, 1], want[:, 0], keys))
    want = want[order]
    got = post.astype(np.int64)
    key_at = np.sort(keys)                 # the bucket of each slot, now that the starts are known to be right
    got = got[np.lexsort((got[:, 1], got[:, 0], key_at))]
    bad = (got != want).any(1)
    assert not bad.any(), 'postings: %d of %d slots differ; first bucket %d: got %s want %s' % (
        int(bad.sum()), nnz, key_at[bad][0], got[bad][0].tolist(), want[bad][0].tolist())


# ---------------------------------------------------------------------------------------------------------------------------
# scores
# ---------------------------------------------------------------------------------------------------------------------------
def f32_shared_oracle(q, c):
    """f32_column_oracle visiting only the columns stored in both q and c: the same bits, for vocabularies of 2^24 columns."""
    q = sp.csc_matrix(q, dtype=np.float32)
    c = sp.csc_matrix(c, dtype=np.float32)
    q.sum_duplicates(); c.sum_duplicates()
    q.sort_indices(); c.sort_indices()
    s = np.zeros((q.shape[0], c.shape[0]), np.float32)
    for f in np.intersect1d(np.nonzero(np.diff(q.indptr))[0], np.nonzero(np.diff(c.indptr))[0]):
        a0, a1, b0, b1 = q.indptr[f], q.indptr[f + 1], c.indptr[f], c.indptr[f + 1]
        s[np.ix_(q.indices[a0:a1], c.indices[b0:b1])] += np.outer(q.data[a0:a1], c.data[b0:b1])
    return s


def score_bound(q, c):
    """(S fp64 [nq, nc], bound fp64 [nq, nc]).  The kernel computes s = fl(...fl(fl(p_1) + fl(p_2)) ... + fl(p_m)) over the m
    columns the two rows share, p_f = q_f c_f.  Each product is rounded once and the m - 1 additions once each (the first,
    0 + fl(p_1), is exact), so with |delta| <= u = 2^-24 per rounding and no underflow or overflow,
    |s - S| <= sum_f |p_f| ((1 + u)^m - 1) <= gamma_m sum_f |p_f|,  gamma_m = m u / (1 - m u)   (Higham, Accuracy and Stability
    of Numerical Algorithms, 3.1)."""
    q64 = sp.csr_matrix(q, dtype=np.float64)
    c64 = sp.csr_matrix(c, dtype=np.float64)
    S = (q64 @ c64.T).toarray()
    mag = (abs(q64) @ abs(c64).T).toarray()
    qp, cp = q64.copy(), c64.copy()
    qp.data[:] = 1.0
    cp.data[:] = 1.0
    m = (qp @ cp.T).toarray()
    return S, m * U32 / (1 - m * U32) * mag


def sparse_self_pairs(x):
    """The pairs i > j of the CSR matrix x that share a column, with the kernel's fp32 score: (i, j, s) sorted by (i, j).  Every
    other pair i > j scores exactly 0.  No n^2 host array: each row against the rows below it."""
    x = sp.csr_matrix(x, dtype=np.float32)
    xc = sp.csc_matrix(x)
    xc.sort_indices()
    out_i, out_j, out_s = [], [], []
    for i in range(x.shape[0]):
        cols = x.indices[x.indptr[i]:x.indptr[i + 1]]
        if cols.size == 0:
            continue
        acc = {}
        for t, f in enumerate(cols):         # increasing column order
            v = np.float32(x.data[x.indptr[i] + t])
            a0, a1 = xc.indptr[f], xc.indptr[f + 1]
            rows, vals = xc.indices[a0:a1], xc.data[a0:a1]
            keep = rows < i
            for j, w in zip(rows[keep].tolist(), vals[keep]):
                acc[j] = np.float32(acc.get(j, np.float32(0)) + np.float32(v * w))
        js = np.array(sorted(acc), np.int32)
        out_i.append(np.full(js.size, i, np.int32))
        out_j.append(js)
        out_s.append(np.array([acc[j] for j in js.tolist()], np.float32))
    cat = lambda a, t: np.concatenate(a).astype(t) if a else np.zeros(0, t)  # noqa: E731
    return cat(out_i, np.int32), cat(out_j, np.int32), cat(out_s, np.float32)


def hist_from_pairs(n, labels, pi, pj, ps, M, bins):
    """test_auroc_hist_host.host_histograms for a matrix given by its (i > j) entries that may be non-zero: every other labelled
    pair i > j scores 0 and is counted in the bin of 0.  Returns (hist int64 [2, bins], sums fp64 [2])."""
    from dae_rnn_news_recommendation_b200.helpers import score_bins
    labels = np.asarray(labels, np.int64)
    lab = labels[labels >= 0]
    sizes = np.bincount(lab) if lab.size else np.zeros(0, np.int64)
    n_rel = int((sizes * (sizes - 1) // 2).sum())
    n_unrel = lab.size * (lab.size - 1) // 2 - n_rel
    li, lj = labels[pi], labels[pj]
    ok = (li >= 0) & (lj >= 0)
    rel = ok & (li == lj)
    unrel = ok & (li != lj)
    hist = np.zeros((2, bins), np.int64)
    sums = np.zeros(2)
    zero_bin = int(score_bins(np.zeros(1, np.float32), M, bins)[0])
    for g, (mask, total) in enumerate(((rel, n_rel), (unrel, n_unrel))):
        s = np.asarray(ps, np.float32)[mask]
        hist[g] = np.bincount(score_bins(s, M, bins), minlength=bins) if s.size else 0
        hist[g, zero_bin] += total - s.size
        sums[g] = s.astype(np.float64).sum()
    return hist, sums


# ---------------------------------------------------------------------------------------------------------------------------
# partial lists
# ---------------------------------------------------------------------------------------------------------------------------
def partial_lists(S, k, splits, allowed=None, groups=None):
    """(val float32 [nq, splits, k], idx int32 [nq, splits, k]): list (q, s) is the exact top k -- or grouped top k -- of split s's
    candidates (see the module docstring)."""
    S = np.asarray(S, np.float32)
    nq, nc = S.shape
    val = np.full((nq, splits, k), -np.inf, np.float32)
    idx = np.full((nq, splits, k), -1, np.int32)
    for s in range(splits):
        c0, c1 = split_rows(nc, splits, s)
        sub_a = None if allowed is None else allowed[:, c0:c1]
        if groups is None:
            i, v = top_k(S[:, c0:c1], k, sub_a)
        else:
            i, v = top_k_groups(S[:, c0:c1], k, sub_a, np.asarray(groups)[c0:c1])
        idx[:, s] = np.where(i >= 0, i + c0, -1)
        val[:, s] = v
    return val, idx


# ---------------------------------------------------------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------------------------------------------------------
def dyadic_csr(rng, n, F, density, j=3, vmax=7, dup=(), share_col=None):
    """CSR [n x F] with values v 2^-j, v a non-zero integer in [-vmax, vmax]: products are multiples of 2^-2j below vmax^2 2^-2j,
    so while m vmax^2 < 2^24 every partial sum of a score is an fp32 integer multiple of 2^-2j -- exact in any order, equal to
    the fp64 score.  dup: (src, dst) row pairs, dst becoming a copy of src (equal scores at different indices).  share_col:
    rows (every 5th) holding one entry at that column only (equal scores of many rows)."""
    m = sp.random(n, F, density=density, format='csr', random_state=np.random.RandomState(int(rng.integers(1 << 31))))
    m.data = (rng.integers(1, vmax + 1, m.nnz) * rng.choice([-1, 1], m.nnz) * 2.0 ** -j)
    m = m.tolil()
    for src, dst in dup:
        m.rows[dst], m.data[dst] = list(m.rows[src]), list(m.data[src])
    if share_col is not None:
        for r in range(0, n, 5):
            m.rows[r], m.data[r] = [share_col], [float(rng.integers(1, 4)) * 2.0 ** -j]
    out = sp.csr_matrix(m, dtype=np.float32)
    out.sort_indices()
    return out


def edge_rows(rng, n, F, j=3, dup=((5, 2047), (2047, 2048), (4095, 4096), (2048, 4097))):
    """Dyadic CSR [n x F] whose rows cycle through the edge kinds: empty, single entry at column 0, single entry at F - 1, every
    column, half the entries negative, explicit stored zeros, and random rows; dup copies rows across the 2048-row range
    edges (pairs outside [0, n) are skipped)."""
    rows, cols, vals = [], [], []
    for r in range(n):
        kind = r % 7
        if kind == 0:
            c = np.zeros(0, np.int64)
        elif kind == 1:
            c = np.array([0])
        elif kind == 2:
            c = np.array([F - 1])
        elif kind == 3:
            c = np.arange(F)
        else:
            c = np.sort(rng.choice(F, int(rng.integers(1, min(F, 12) + 1)), replace=False))
        v = rng.integers(1, 8, c.size).astype(np.float64)
        if kind == 4:
            v[: c.size // 2 + 1] *= -1
        elif kind == 5:
            v[::2] = 0.0                     # explicit stored zeros
        rows.append(np.full(c.size, r)); cols.append(c); vals.append(v * 2.0 ** -j)
    m = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, F)).tolil()
    for src, dst in dup:
        if src < n and dst < n:
            m.rows[dst], m.data[dst] = list(m.rows[src]), list(m.data[src])
    out = sp.csr_matrix(m, dtype=np.float32)   # lil keeps the stored zeros
    out.sort_indices()
    return out


def inf_rows(F=16):
    """A small CSR whose rows hold +inf, -inf, +inf next to an explicit 0, and finite values, with the scores they give:
    inf * 0 = NaN, +inf + (-inf) = NaN, and +-inf times a finite non-zero value."""
    dense = np.array([
        [np.inf, 1, 0, 0],        # +inf at column 0
        [-np.inf, 1, 0, 0],       # -inf at column 0
        [1, 2, 0, 0],             # finite
        [0, 1, 0, 0],             # stored 0 at column 0 (kept below), 1 at column 1
        [np.inf, 0, 1, 0],        # +inf and a stored 0
        [1, 0, 0, 3],             # finite
        [-1, 0, 0, 0],            # negative
        [0, 0, 0, 0],             # empty
    ], np.float64)
    rows, cols = np.nonzero(dense)
    stored = list(zip(rows.tolist(), cols.tolist())) + [(3, 0), (4, 1)]
    r = np.array([t[0] for t in stored]); c = np.array([t[1] for t in stored])
    m = sp.csr_matrix((dense[r, c].astype(np.float32), (r, c)), shape=(dense.shape[0], F))
    m.sort_indices()
    return m
