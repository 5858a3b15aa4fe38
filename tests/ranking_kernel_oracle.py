"""References for the dense ranking kernels of csrc/gemm_tc.cu and csrc/topk.cuh (dae_similarity_topk_bf16x3 / _excl_ / _groups_,
dae_similarity_topk_bound_bf16x3 / _collect_bf16x3 / _select, dae_similarity_pairs_bf16x3, dae_similarity_pair_hist_bf16x3) and
csrc/pairs_sort.cu (dae_pairs_sort), for the kernel-level tests.  Tests only; nothing here needs a GPU.

Exact scores.  The operands come from gemm_kernel_oracle.exact_operands: hi integers, lo on a 2^-4 grid, every partial sum below
2^15.  S = pair_exact(...) is then the fp32 value every tile, split and k order produces, so every list, tau, pair set, histogram
and fp64 sum below is known bit for bit.  Ties come from duplicated rows and from the small value range.

Orders.  top_k(): (score desc, index asc), -0.0 equal to +0.0 (the stored bits are reported), padding -1 / -inf.  A candidate is
an allowed column whose score beats -inf: the kernels insert only v > thr with thr starting at -inf, so neither -inf nor NaN is
ever listed.  Groups: topk_groups_oracle.grouped_top_k, and its streamed model for the partial lists.

Dispatch.  topk_splits / topk_bound_splits / rank_chunk restate the host side of gemm_tc.cu; split_tiles / half_columns the
schedule of TopkSched; partial_lists() the list each (row, split, 64-column half) flushes to the workspace, which holds per row
2 splits lists of k in (split, half) order: all values of all rows first, then all indices.
"""
import numpy as np

from gemm_kernel_oracle import BF16_NAN, bf16_value, exact_h, exact_operands, pair_bound, pair_exact  # noqa: F401
from topk_groups_oracle import _stream, grouped_top_k  # noqa: F401

BLOCK_M = 128
BLOCK_N = 128
HALF_N = 64
TOPK_MAX_K = 32
TOPK_MAX_SPLITS = 32
TOPK_MIN_TILES = 4
LONG_MAX_K = 1024
RANK_THREADS = 256
FLT_MAX = float(np.finfo(np.float32).max)


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------------
# host dispatch (gemm_tc.cu: topk_splits, topk_workspace_bytes, topk_bound_splits, rank_chunk)
# ---------------------------------------------------------------------------------------------------------------------------
def topk_splits(n_query, n_corpus, requested, sms=132):
    tiles_m, tiles_n = _cdiv(n_query, BLOCK_M), _cdiv(n_corpus, BLOCK_N)
    s = requested
    if s <= 0:
        s = min(_cdiv(sms, tiles_m), tiles_n // TOPK_MIN_TILES)
    s = min(s, tiles_n, TOPK_MAX_SPLITS)
    return max(s, 1)


def topk_workspace_bytes(n_query, k, splits):
    return n_query * 2 * splits * k * 8


def topk_bound_splits(n_query, n_corpus, k, requested, sms=132):
    s = topk_splits(n_query, n_corpus, requested, sms)
    return topk_splits(n_query, n_corpus, max(s, _cdiv(k, 32)), sms)


def rank_chunk(k):
    L = RANK_THREADS
    while L < k:
        L <<= 1
    return L


def kmax(k):
    """KMAX of the topk_kernel instantiation a register call with this k runs."""
    return 16 if k <= 16 else 32


def work_items(n_query, splits):
    return _cdiv(n_query, BLOCK_M) * splits


def split_tiles(n_corpus, splits, s):
    """[t0, t1) column tiles of split s (TopkSched::next)."""
    tiles_n = _cdiv(n_corpus, BLOCK_N)
    return s * tiles_n // splits, (s + 1) * tiles_n // splits


def half_columns(n_corpus, splits, s, half):
    """The corpus columns one epilogue thread of split s sees, in increasing order: its 64-column half of every tile, below N."""
    t0, t1 = split_tiles(n_corpus, splits, s)
    c = np.concatenate([np.arange(t * BLOCK_N + half * HALF_N, t * BLOCK_N + (half + 1) * HALF_N) for t in range(t0, t1)])
    return c[c < n_corpus]


# ---------------------------------------------------------------------------------------------------------------------------
# candidates and orders
# ---------------------------------------------------------------------------------------------------------------------------
def allowed_mask(n_query, n_corpus, exclude=False, diag_offset=0, lists=None):
    """bool [n_query, n_corpus]: column i + diag_offset left out when `exclude`; lists: per row an iterable of excluded columns."""
    a = np.ones((n_query, n_corpus), bool)
    if exclude:
        i = np.arange(n_query)
        j = i + diag_offset
        ok = (j >= 0) & (j < n_corpus)
        a[i[ok], j[ok]] = False
    if lists is not None:
        for r, cols in enumerate(lists):
            a[r, np.asarray(cols, np.int64)] = False
    return a


def _rank_cols(s, cols, k):
    """The first k of cols (int [n]) of one score row s by (score desc, index asc) among candidates; (idx, val) padded."""
    v = s[cols]
    cand = v > -np.inf
    cols, v = cols[cand], v[cand]
    order = np.lexsort((cols, -v.astype(np.float64)))[:k]
    idx = np.full(k, -1, np.int32)
    val = np.full(k, -np.inf, np.float32)
    idx[:order.size] = cols[order]
    val[:order.size] = v[order]
    return idx, val


def top_k(s, k, allowed=None):
    """s [nq, nc] float32 scores -> (idx int32 [nq, k], val float32 [nq, k]): the contract of the register and long top-k."""
    s = np.asarray(s, np.float32)
    nq, nc = s.shape
    idx = np.full((nq, k), -1, np.int32)
    val = np.full((nq, k), -np.inf, np.float32)
    cols = np.arange(nc)
    for r in range(nq):
        idx[r], val[r] = _rank_cols(s[r], cols if allowed is None else cols[allowed[r]], k)
    return idx, val


def top_k_groups(s, k, allowed, groups):
    """grouped_top_k over the candidates (allowed and above -inf)."""
    s = np.asarray(s, np.float32)
    cand = s > -np.inf
    return grouped_top_k(s, groups, k, cand if allowed is None else cand & allowed)


def partial_lists(s, k, splits, allowed=None, groups=None, km=None):
    """The workspace the register kernel leaves: (val float32 [nq, 2 splits, k], idx int32 [nq, 2 splits, k]).  List 2 sp + h is
    the running list of (row, split sp, half h) over that half's columns of the split's tiles: the exact top k of those
    candidates, or with groups the streamed list of KMAX slots of topk_offer_group (topk_groups_oracle._stream)."""
    s = np.asarray(s, np.float32)
    nq, nc = s.shape
    km = kmax(k) if km is None else km
    val = np.full((nq, 2 * splits, k), -np.inf, np.float32)
    idx = np.full((nq, 2 * splits, k), -1, np.int32)
    for sp in range(splits):
        for h in range(2):
            cols = half_columns(nc, splits, sp, h)
            if groups is None:
                sub = s[:, cols]
                cand = sub > -np.inf
                if allowed is not None:
                    cand &= allowed[:, cols]
                key = np.where(cand, -sub.astype(np.float64), np.inf)
                order = np.lexsort((np.broadcast_to(cols, sub.shape), key), axis=-1)[:, :k]
                ok = np.take_along_axis(cand, order, 1)
                n = order.shape[1]
                idx[:, 2 * sp + h, :n] = np.where(ok, cols[order], -1)
                val[:, 2 * sp + h, :n] = np.where(ok, np.take_along_axis(sub, order, 1), np.float32(-np.inf))
            else:
                for r in range(nq):
                    c = cols if allowed is None else cols[allowed[r, cols]]
                    lst = _stream(s[r], c, groups, k, km)
                    val[r, 2 * sp + h] = [v for v, _ in lst]
                    idx[r, 2 * sp + h] = [i for _, i in lst]
    return val, idx


def merge_lists(val, idx, k, groups=None):
    """topk_merge_kernel / topk_merge_groups_kernel on host: the lists' entries by (score desc, index asc), first of each group."""
    nq = val.shape[0]
    out_i = np.full((nq, k), -1, np.int32)
    out_v = np.full((nq, k), -np.inf, np.float32)
    for r in range(nq):
        ok = idx[r].ravel() >= 0
        v, c = val[r].ravel()[ok], idx[r].ravel()[ok]
        order = np.lexsort((c, -v.astype(np.float64)))
        if groups is not None:
            _, first = np.unique(np.asarray(groups)[c[order]], return_index=True)
            order = order[np.sort(first)]
        order = order[:k]
        out_i[r, :order.size], out_v[r, :order.size] = c[order], v[order]
    return out_i, out_v


# ---------------------------------------------------------------------------------------------------------------------------
# long lists: bound, collect, select
# ---------------------------------------------------------------------------------------------------------------------------
def bound_tau(val, idx, k, groups=None):
    """topk_bound_kernel: the stored score of the k-th entry of the row's lists by (score desc, list position asc) -- the k-th
    distinct group with groups -- or -FLT_MAX when there are fewer."""
    nq = val.shape[0]
    tau = np.full(nq, -FLT_MAX, np.float32)
    for r in range(nq):
        v, c = val[r].ravel(), idx[r].ravel()
        pos = np.nonzero(c >= 0)[0]
        order = pos[np.lexsort((pos, -v[pos].astype(np.float64)))]
        if groups is not None:
            _, first = np.unique(np.asarray(groups)[c[order]], return_index=True)
            order = order[np.sort(first)]
        if order.size >= k:
            tau[r] = v[order[k - 1]]
    return tau


def collect_set(s, tau, allowed=None):
    """(i, j, score) sorted by (i, j): allowed columns with s >= max(tau_i, -FLT_MAX) (NaN tau acts as -FLT_MAX, as fmaxf)."""
    s = np.asarray(s, np.float32)
    t = np.fmax(np.asarray(tau, np.float32), np.float32(-FLT_MAX))
    with np.errstate(invalid='ignore'):
        keep = s >= t[:, None]
    if allowed is not None:
        keep &= allowed
    i, j = np.nonzero(keep)
    return i.astype(np.int32), j.astype(np.int32), s[i, j]


def pairs_set(s, tau, self_mode):
    """dae_similarity_pairs_bf16x3: (i, j, score) with s >= tau (self mode: j < i only), sorted by (i, j)."""
    s = np.asarray(s, np.float32)
    with np.errstate(invalid='ignore'):
        keep = s >= np.float32(tau)
    if self_mode:
        keep &= np.tril(np.ones(s.shape, bool), -1)
    i, j = np.nonzero(keep)
    return i.astype(np.int32), j.astype(np.int32), s[i, j]


def select(pi, pj, ps, n_query, k, groups=None):
    """topk_select_kernel: per row the k best of its candidates (pi sorted, pj ascending within a row) by (score desc, j asc)."""
    idx = np.full((n_query, k), -1, np.int32)
    val = np.full((n_query, k), -np.inf, np.float32)
    pi, pj, ps = np.asarray(pi), np.asarray(pj), np.asarray(ps, np.float32)
    bounds = np.searchsorted(pi, np.arange(n_query + 1))
    for r in range(n_query):
        j, v = pj[bounds[r]:bounds[r + 1]], ps[bounds[r]:bounds[r + 1]]
        order = np.lexsort((j, -v.astype(np.float64)))
        if groups is not None:
            _, first = np.unique(np.asarray(groups)[j[order]], return_index=True)
            order = order[np.sort(first)]
        order = order[:k]
        idx[r, :order.size], val[r, :order.size] = j[order], v[order]
    return idx, val


def select_brute(pi, pj, ps, n_query, k):
    """select() another way, for the host test: Python sort with the -0.0 fold written out."""
    idx = np.full((n_query, k), -1, np.int32)
    val = np.full((n_query, k), -np.inf, np.float32)
    rows = {}
    for i, j, v in zip(np.asarray(pi).tolist(), np.asarray(pj).tolist(), np.asarray(ps, np.float32)):
        rows.setdefault(i, []).append((0.0 if v == 0 else float(v), j, v))
    for i, lst in rows.items():
        lst.sort(key=lambda t: (-t[0], t[1]))
        for t, (_, j, v) in enumerate(lst[:k]):
            idx[i, t], val[i, t] = j, v
    return idx, val


def membership(ref, bound, idx, k, allowed=None):
    """Top-k membership of data that is not exact: ref / bound fp64 [nq, nc] (pair_bound).  Every listed entry lies within its
    bound of the k-th fp64 score; every entry beating the k-th by more than twice the bounds is listed.  Returns a list of
    violations (empty when the lists pass)."""
    bad = []
    nq, nc = ref.shape
    for r in range(nq):
        cand = np.arange(nc) if allowed is None else np.nonzero(allowed[r])[0]
        if cand.size == 0:
            continue
        order = cand[np.argsort(-ref[r, cand], kind='stable')]
        kk = min(k, cand.size)
        kth = ref[r, order[kk - 1]]
        b_kth = bound[r, order[kk - 1]]
        got = idx[r][idx[r] >= 0]
        if got.size != kk:
            bad.append((r, 'listed %d of %d' % (got.size, kk)))
        for c in got:
            if ref[r, c] < kth - bound[r, c] - b_kth:
                bad.append((r, 'listed %d below the k-th' % c))
        must = cand[ref[r, cand] > kth + 2 * (bound[r, cand] + b_kth)]
        missing = np.setdiff1d(must, got)
        if missing.size:
            bad.append((r, 'missing %s' % missing[:5].tolist()))
    return bad
