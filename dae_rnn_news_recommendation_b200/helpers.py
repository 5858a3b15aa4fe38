"""GPU versions of the evaluation helpers that consume transform()'s output (reference helpers.py:11-50 and the
nearest-article lookup of main_autoencoder.py:307-318,352-359) -- SURVEY section 8f, rank 1.

    pairwise_similarity(in_df, norm='', metric='cosine', set_diagonal_zero=True) -> ndarray [N, N]     (reference signature)
    nearest_neighbors(embeddings, metric='cosine', chunk=8192) -> (index[N], score[N])                (no N x N matrix on the host)
    top_k_similar(embeddings, k=10, corpus=None, metric='cosine', exclude=None, groups=None) -> (index[Nq, k], score[Nq, k])
                                                                                                      (no similarity matrix at all;
                                                                                                        dense or scipy sparse inputs;
                                                                                                        per-query exclusion lists;
                                                                                                        at most one row per group)
    label_precision_at_k(index, query_labels, corpus_labels) -> float                                 (share of same-label neighbours)
    user_profiles(histories, embeddings) -> [U, H]                                                    (weighted mean of the read articles)
    sparse_profiles(histories, X) -> scipy CSR [U, F]                                                 (the same of the bag of words)
    recommend_sparse(histories, X, k=10, candidates=None, exclude_read=True, groups=None) -> (index[U, k], score[U, k])
                                                                                                      (recommend from sparse_profiles)
    recommend(histories, embeddings, k=10, candidates=None, exclude_read=True, profiles=None, groups=None)
                                                                                   -> (index[U, k], score[U, k])
                                                                                                      (k best unread articles per user;
                                                                                                        mean or given profiles;
                                                                                                        one article per story)
    sequences_from_csr(m) -> (indptr[U + 1], items)                                                   (reads ordered by stored time)
    recommendation_recall(index, targets) -> dict                                                     (hit rate / recall of held-out reads)
    impression_metrics(vectors, embeddings, impressions, metric='linear kernel') -> dict              (AUC / MRR / nDCG@5, @10 per
                                                                                                        impression, averaged)
    impression_metrics_sparse(profiles, X, impressions, metric='linear kernel') -> dict               (the same for sparse query rows)
    similar_pairs(data, threshold, corpus=None, metric='cosine') -> (i[P], j[P], score[P])            (every pair with score >= threshold,
                                                                                                        near-duplicates; no matrix)
    duplicate_groups(i, j, n) -> group[n]                                                             (connected components of the pairs)
    pair_label_agreement(i, j, labels, corpus_labels=None) -> dict                                    (precision / recall against labels)
    visualize_pairwise_similarity(labels, pairwise_similarity_metrics, ...) -> dict                   (rank 2: AUROC + box statistics)
    similarity_auroc(data, labels, metric='cosine', bins=1 << 21) -> dict                              (the same numbers on a score
                                                                                                        grid, without the matrix)
    auroc_from_histograms(hist, sums, M, bins) -> dict                                                 (its host half, pure NumPy)

Dense inputs (embeddings) go through the wgmma bf16x3 kernels on row-normalised operands.  Sparse inputs (count / tf-idf
matrices) go through the CSR x CSR kernels (dae_csr_*), except in pairwise_similarity, which runs the CSR encode kernel against
the dense transpose.  top_k_similar, similar_pairs and similarity_auroc build their operands of either kind in one place
(_Operands); recommend and recommend_sparse share their request (_recommend_request) and their output (_recommend_result), and
differ only in how they rank.  No CPU path.
"""
import ctypes
import math

import numpy as np
import scipy.sparse as sp
import torch

from . import _cabi
from ._cabi import call
from .engine import DeviceCSR, canonical_csr
from .io_formats import save_file, read_file  # noqa: F401  (reference helpers.py:138-264; SURVEY 8f rank 3)

_NORM = {'': 0, 'l1': 1, 'l2': 2, 'max': 3}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check_metric(metric, fn):
    if metric not in ('cosine', 'linear kernel'):
        raise ValueError("%s: metric = %r: 'cosine' or 'linear kernel'" % (fn, metric))


def _result(out, to_host):
    """An entry point's return value: the device tensor out (or tuple of them) as ndarrays with to_host, as it is without."""
    if not to_host:
        return out
    return tuple(t.cpu().numpy() for t in out) if isinstance(out, tuple) else out.cpu().numpy()


def _normalised_operands(x_dev, norm_kind):
    n, h = x_dev.shape
    ld = (h + 7) // 8 * 8
    hi = torch.empty(n, ld, dtype=torch.bfloat16, device=x_dev.device)
    lo = torch.empty(n, ld, dtype=torch.bfloat16, device=x_dev.device)
    call('dae_rownorm_split_bf16', x_dev.data_ptr(), n, h, x_dev.stride(0), norm_kind, hi.data_ptr(), lo.data_ptr(), ld, None, 0, _stream())
    return hi, lo, ld


def _gemm_nt(a, b, n_a, n_b, k, out):
    call('dae_gemm_bf16x3', n_a, n_b, k, 1.0, a[0].data_ptr(), a[1].data_ptr(), a[0].stride(0), 0, b[0].data_ptr(), b[1].data_ptr(),
         b[0].stride(0), 0, out.data_ptr(), out.stride(0), 0, -1, None, 1, 0, _stream())


def _to_device_dense(in_df, device):
    if isinstance(in_df, list):
        in_df = np.asarray(in_df)
    if hasattr(in_df, 'values') and not isinstance(in_df, np.ndarray):
        in_df = in_df.values
    return torch.from_numpy(np.ascontiguousarray(in_df, dtype=np.float32)).to(device)


def pairwise_similarity(in_df, norm='', metric='cosine', set_diagonal_zero=True, device='cuda:0', to_host=True):
    """Reference helpers.pairwise_similarity: optional `norm` ('l1','l2','max'), then cosine similarity or the linear kernel
    of every pair of rows, diagonal zeroed.  Returns a float32 ndarray [N, N] (`to_host=False`: the device tensor, which
    visualize_pairwise_similarity accepts as is)."""
    assert metric in ['cosine', 'linear kernel']
    assert norm in _NORM
    if sp.issparse(in_df):
        return _result(_pairwise_sparse(in_df, norm, metric, set_diagonal_zero, device), to_host)
    x = _to_device_dense(in_df, device)
    n, h = x.shape
    if norm != '':   # sklearn.preprocessing.normalize first (helpers.py:42-43) ...
        xn = torch.empty_like(x)
        call('dae_rownorm_split_bf16', x.data_ptr(), n, h, x.stride(0), _NORM[norm], None, None, 0, xn.data_ptr(), xn.stride(0), _stream())
        x = xn
    hi, lo, _ = _normalised_operands(x, 2 if metric == 'cosine' else 0)   # ... then the metric's own L2 normalisation (cosine)
    out = torch.empty(n, n, dtype=torch.float32, device=device)
    _gemm_nt((hi, lo), (hi, lo), n, n, h, out)
    if set_diagonal_zero:
        out.diagonal().zero_()
    return _result(out, to_host)


def _pairwise_sparse(m, norm, metric, set_diagonal_zero, device):
    """X_hat . X_hat^T for a sparse X through the CSR encode kernel: the dense operand is X_hat^T [F x N]."""
    from sklearn.preprocessing import normalize   # host-side row scaling of the CSR values only (data prep, not the contraction)
    m = sp.csr_matrix(m, dtype=np.float32)
    if norm != '':
        m = normalize(m, norm=norm)
    if metric == 'cosine':
        m = normalize(m, norm='l2')
    n, f = m.shape
    csr = DeviceCSR(m, device)
    out = torch.empty(n, n, dtype=torch.float32, device=device)
    rows = torch.repeat_interleave(torch.arange(n, device=device), (csr.indptr[1:] - csr.indptr[:-1]))
    indptr_host = m.indptr
    blk = 2048   # the encode kernel keeps one output row of <= 4096 floats in registers: X_hat^T goes through it in column blocks
    for c0 in range(0, n, blk):
        c1 = min(n, c0 + blk)
        wp = (c1 - c0 + 3) // 4 * 4
        p0, p1 = int(indptr_host[c0]), int(indptr_host[c1])
        dense_t = torch.zeros(f, wp, dtype=torch.float32, device=device)
        dense_t[csr.indices[p0:p1].long(), rows[p0:p1] - c0] = csr.values[p0:p1]
        out_blk = torch.empty(n, wp, dtype=torch.float32, device=device)
        zero_b = torch.zeros(wp, dtype=torch.float32, device=device)
        call('dae_encode_csr_fwd', csr.indptr.data_ptr(), csr.indices.data_ptr(), csr.values.data_ptr(), None, n, f, wp, 1.0,
             dense_t.data_ptr(), zero_b.data_ptr(), _cabi.ACT['none'], out_blk.data_ptr(), wp, None, None, None, 0, _stream())
        out[:, c0:c1] = out_blk[:, :c1 - c0]
    if set_diagonal_zero:
        out.diagonal().zero_()
    return out


def nearest_neighbors(embeddings, metric='cosine', chunk=8192, device='cuda:0'):
    """For every row the most similar OTHER row and its score (the lookup of main_autoencoder.py:352-353) without materialising
    N x N: row chunks of the similarity are produced by the GEMM and reduced by dae_row_argmax on the device.  The first maximum
    wins and NaN scores are skipped, as np.nanargmax does, but the row itself is never a candidate: where every other score is
    negative the best of them is returned (the reference's nanargmax over the zero-diagonal matrix returns the row itself, with
    score 0), and top_k_similar(k=1) follows the same rule.  A single row gets index -1 and score -inf."""
    x = _to_device_dense(embeddings, device)
    n, h = x.shape
    hi, lo, _ = _normalised_operands(x, 2 if metric == 'cosine' else 0)
    idx = torch.empty(n, dtype=torch.int32, device=device)
    val = torch.empty(n, dtype=torch.float32, device=device)
    buf = torch.empty(min(chunk, n), n, dtype=torch.float32, device=device)
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        _gemm_nt((hi[r0:r1], lo[r0:r1]), (hi, lo), r1 - r0, n, h, buf)
        call('dae_row_argmax', buf.data_ptr(), r1 - r0, n, buf.stride(0), r0, 0, idx[r0:r1].data_ptr(), val[r0:r1].data_ptr(), _stream())
    torch.cuda.synchronize()
    return idx.cpu().numpy(), val.cpu().numpy()


def _similarity_topk(q, c, n_q, n_c, h, k, diag_offset=0, exclude=False, splits=0, lists=None, groups=None):
    """k best corpus rows per query row of the bf16 hi / lo operand pairs q and c (dae_similarity_topk_bf16x3): device tensors
    (index int32 [n_q, k], score float32 [n_q, k]); with `exclude`, column i + diag_offset is not a candidate of row i.  lists:
    per-row exclusion lists (_DeviceLists) through dae_similarity_topk_excl_bf16x3.  groups: device int32 [n_c] labels, at most
    one row per group (dae_similarity_topk_groups_bf16x3, with or without lists)."""
    dev = q[0].device
    need = (ctypes.c_int64 * 1)()
    call('dae_similarity_topk_workspace', n_q, n_c, k, splits, ctypes.addressof(need))
    ws = torch.empty(max(int(need[0]), 16), dtype=torch.uint8, device=dev)
    idx = torch.empty(n_q, k, dtype=torch.int32, device=dev)
    val = torch.empty(n_q, k, dtype=torch.float32, device=dev)
    args = (n_q, n_c, h, q[0].data_ptr(), q[1].data_ptr(), q[0].stride(0), c[0].data_ptr(), c[1].data_ptr(), c[0].stride(0), k, diag_offset,
            1 if exclude else 0, splits, ws.data_ptr(), ws.numel(), idx.data_ptr(), val.data_ptr())
    if groups is not None:
        call('dae_similarity_topk_groups_bf16x3', *args, *_list_args(lists), groups.data_ptr(), _stream())
    elif lists is None:
        call('dae_similarity_topk_bf16x3', *args, _stream())
    else:
        call('dae_similarity_topk_excl_bf16x3', *args, lists.indptr.data_ptr(), lists.indices.data_ptr(), lists.nnz, _stream())
    return idx, val


TOPK_MAX_K = 32                    # the register kernels (dae_similarity_topk_*)
TOPK_LONG_MAX_K = 1024             # long_lists=True, dense inputs (dae_similarity_topk_bound / _collect / _select)
TOPK_LONG_MAX_CANDIDATES = 1 << 24  # default candidate budget of the long lists: 12 B per candidate, 24 B more in the sort


def _check_k(k, long_lists, sparse, fn):
    """k validation of top_k_similar / recommend, before any device work."""
    if long_lists:
        if not 1 <= k <= TOPK_LONG_MAX_K:
            raise _cabi.DaeError('%s: k = %d is outside the supported range 1 <= k <= %d' % (fn, k, TOPK_LONG_MAX_K))
        if sparse and k > TOPK_MAX_K:
            raise ValueError('%s: k = %d: sparse inputs rank at most %d results per query (long_lists needs dense inputs)'
                             % (fn, k, TOPK_MAX_K))
    elif not 1 <= k <= TOPK_MAX_K:
        raise _cabi.DaeError('%s: k = %d is outside the supported range 1 <= k <= %d (long_lists=True ranks up to %d for dense '
                             'inputs)' % (fn, k, TOPK_MAX_K, TOPK_LONG_MAX_K))


def _check_budget(max_candidates, fn):
    if isinstance(max_candidates, bool) or not isinstance(max_candidates, (int, np.integer)) or max_candidates < 1:
        raise ValueError('%s: max_candidates = %r must be a positive integer' % (fn, max_candidates))
    return int(max_candidates)


def _similarity_topk_long(q, c, n_q, n_c, h, k, exclude=False, splits=0, lists=None, groups=None,
                          max_candidates=TOPK_LONG_MAX_CANDIDATES):
    """_similarity_topk for any 1 <= k <= 1024 in three stages per chunk of query rows (DESIGN 4.14): a lower bound tau_i on each
    row's k-th score from the register kernels' partial lists (dae_similarity_topk_bound_bf16x3), every candidate with s >= tau_i
    (dae_similarity_topk_collect_bf16x3), sorted by (i, j) (dae_pairs_sort), and each row's k best of them
    (dae_similarity_topk_select).  The output equals the register kernels' for k <= 32, bit for bit.
    Memory: at most max(max_candidates, n_c) candidates are held at once (12 B each, 24 B more during the sort), so a single row
    always fits; the chunks hold max_candidates // (2k) rows.  When a chunk's candidates exceed that, its per-row counts cut it into
    row ranges that fit, and each range is collected once more."""
    dev = q[0].device
    budget = max(int(max_candidates), n_c)
    rows = max(1, min(n_q, budget // (2 * k)))
    cap = min(budget, rows * n_c)
    idx = torch.empty(n_q, k, dtype=torch.int32, device=dev)
    val = torch.empty(n_q, k, dtype=torch.float32, device=dev)
    need = (ctypes.c_int64 * 1)()
    call('dae_similarity_topk_bound_workspace', rows, n_c, k, splits, ctypes.addressof(need))
    ws = torch.empty(max(int(need[0]), 16), dtype=torch.uint8, device=dev)
    tau = torch.empty(rows, dtype=torch.float32, device=dev)
    row_count = torch.zeros(rows, dtype=torch.int32, device=dev)   # uint32 in the kernel
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    i_buf = torch.empty(cap, dtype=torch.int32, device=dev)
    j_buf = torch.empty(cap, dtype=torch.int32, device=dev)
    s_buf = torch.empty(cap, dtype=torch.float32, device=dev)
    ex_ptr, ex_ind, ex_nnz = _list_args(lists)
    g_ptr = None if groups is None else groups.data_ptr()
    row_bytes = lists.indptr.element_size() if lists is not None else 0

    def operands(r0):   # (n_corpus, dim, q_hi, q_lo, ldq, c_hi, c_lo, ldc) of the query rows from r0 on
        return (n_c, h, q[0][r0:].data_ptr(), q[1][r0:].data_ptr(), q[0].stride(0), c[0].data_ptr(), c[1].data_ptr(), c[0].stride(0))

    def lists_from(r0):   # the exclusion lists of the query rows from r0 on (their indices stay absolute)
        return (None if ex_ptr is None else ex_ptr + r0 * row_bytes), ex_ind, ex_nnz

    def collect(r0, m, t0):   # rows [r0, r0 + m), tau[t0:]; the self match of query row r is column r
        count.zero_()
        row_count[:m].zero_()
        call('dae_similarity_topk_collect_bf16x3', m, *operands(r0), r0, 1 if exclude else 0, tau[t0:].data_ptr(), *lists_from(r0),
             count.data_ptr(), row_count.data_ptr(), cap, i_buf.data_ptr(), j_buf.data_ptr(), s_buf.data_ptr(), _stream())
        return int(count.item())

    def select(r0, m, n):
        i, j, s = _sort_pairs([i_buf, j_buf, s_buf], n, m, n_c, dev)
        call('dae_similarity_topk_select', m, n, i.data_ptr() if n else None, j.data_ptr() if n else None, s.data_ptr() if n else None,
             k, g_ptr, idx[r0].data_ptr(), val[r0].data_ptr(), _stream())

    for r0 in range(0, n_q, rows):
        m = min(rows, n_q - r0)
        call('dae_similarity_topk_bound_bf16x3', m, *operands(r0), k, r0, 1 if exclude else 0, splits, ws.data_ptr(), ws.numel(),
             *lists_from(r0), g_ptr, tau.data_ptr(), _stream())
        n = collect(r0, m, 0)
        if n <= cap:
            select(r0, m, n)
            continue
        per_row = row_count[:m].cpu().numpy().astype(np.int64)   # exact: the capacity only limits what is written
        a = 0
        while a < m:   # row ranges [a, b) of at most cap candidates; one row alone always fits (per_row <= n_c <= cap)
            b = a + max(1, int(np.searchsorted(np.cumsum(per_row[a:]), cap, side='right')))
            want = int(per_row[a:b].sum())
            got = collect(r0 + a, b - a, a)
            if got != want:
                raise RuntimeError('top_k_similar: the second collect call counted %d candidates, the first %d' % (got, want))
            select(r0 + a, b - a, got)
            a = b
    return idx, val


def _list_args(lists):
    """(ex_indptr, ex_indices, ex_nnz) of the *_groups exports: NULL pointers for no lists."""
    if lists is None:
        return None, None, 0
    return lists.indptr.data_ptr(), (lists.indices.data_ptr() if lists.nnz else None), lists.nnz


class _DeviceLists:
    """Per-query exclusion lists on the device: the CSR structure indptr int64 [n + 1], indices int32 [nnz], rows sorted and
    without duplicates (the layout dae_*_topk_excl* read)."""

    def __init__(self, indptr, indices, nnz):
        self.indptr, self.indices, self.nnz = indptr, indices, int(nnz)

    @staticmethod
    def from_host(indptr, indices, device):
        return _DeviceLists(torch.from_numpy(np.ascontiguousarray(indptr, dtype=np.int64)).to(device),
                            torch.from_numpy(np.ascontiguousarray(indices, dtype=np.int32)).to(device), len(indices))


def _stored_positions(m, shape, what, fn):
    """The stored positions of the scipy sparse matrix m (values ignored, explicit zeros included) as a canonical CSR structure:
    (indptr int64 [rows + 1], indices int32, data float64 summed over repeated positions).  ValueError when m is not scipy sparse,
    has another shape (a None entry of `shape` accepts any size) or holds an index outside it."""
    if not sp.issparse(m):
        raise ValueError('%s: %s must be a scipy sparse matrix, not %s' % (fn, what, type(m).__name__))
    if len(m.shape) != 2 or any(want is not None and got != want for got, want in zip(m.shape, shape)):
        raise ValueError('%s: %s has shape %s, (%s) expected' % (fn, what, tuple(m.shape),
                                                                 ', '.join('any' if s is None else str(s) for s in shape)))
    n_r, n_c = m.shape
    try:
        coo = m.tocoo()
    except (ValueError, IndexError) as e:
        raise ValueError('%s: %s is malformed or holds an index outside its shape %s (%s)' % (fn, what, (n_r, n_c), e))
    r, c = np.asarray(coo.row, dtype=np.int64), np.asarray(coo.col, dtype=np.int64)
    if r.size and (r.min() < 0 or r.max() >= n_r or c.min() < 0 or c.max() >= n_c):
        raise ValueError('%s: %s holds an index outside its shape %s' % (fn, what, (n_r, n_c)))
    data = np.asarray(coo.data, dtype=np.float64) if coo.data.dtype != object else np.ones(r.size)
    out = sp.csr_matrix((data, (r, c)), shape=(n_r, n_c))   # sums repeated positions, keeps explicit zeros
    out.sum_duplicates()
    out.sort_indices()
    return out.indptr.astype(np.int64), out.indices.astype(np.int32), out.data


def _as_device_dense(x, device):
    if isinstance(x, torch.Tensor):
        return x.to(device=device, dtype=torch.float32).contiguous()
    return _to_device_dense(x, device)


def _csr_operand(x, metric):
    """The CSR matrix the sparse top-k ranks: canonical (sorted, no duplicates), fp32, rows L2-normalised for 'cosine' with
    all-zero rows left zero (sklearn.preprocessing.normalize, as _pairwise_sparse)."""
    m = canonical_csr(x).astype(np.float32)
    if metric == 'cosine':
        from sklearn.preprocessing import normalize   # host-side row scaling of the CSR values only (data prep)
        m = canonical_csr(normalize(m, norm='l2')).astype(np.float32)
    return m


def _csr_similarity_topk(q, c, k, diag_offset=0, exclude=False, splits=0, lists=None, groups=None):
    """k best corpus rows per query row of the DeviceCSR matrices q and c by S = Q.C^T (dae_csr_similarity_topk): device tensors
    (index int32 [n_q, k], score float32 [n_q, k]); with `exclude`, column i + diag_offset is not a candidate of row i.  lists:
    per-row exclusion lists (_DeviceLists) through dae_csr_similarity_topk_excl.  groups: device int32 [n_c] labels, at most one
    row per group (dae_csr_similarity_topk_groups)."""
    dev = q.indptr.device
    n_q, n_c = q.shape[0], c.shape[0]
    need = (ctypes.c_int64 * 1)()
    call('dae_csr_similarity_topk_workspace', n_q, n_c, c.nnz, c.shape[1], k, splits, ctypes.addressof(need))
    ws = torch.empty(max(int(need[0]), 16), dtype=torch.uint8, device=dev)
    idx = torch.empty(n_q, k, dtype=torch.int32, device=dev)
    val = torch.empty(n_q, k, dtype=torch.float32, device=dev)
    args = (q.indptr.data_ptr(), q.indices.data_ptr(), q.values.data_ptr(), n_q, q.nnz, q.shape[1], c.indptr.data_ptr(),
            c.indices.data_ptr(), c.values.data_ptr(), n_c, c.nnz, c.shape[1], k, diag_offset, 1 if exclude else 0, splits, ws.data_ptr(),
            ws.numel(), idx.data_ptr(), val.data_ptr())
    if groups is not None:
        call('dae_csr_similarity_topk_groups', *args, *_list_args(lists), groups.data_ptr(), _stream())
    elif lists is None:
        call('dae_csr_similarity_topk', *args, _stream())
    else:
        call('dae_csr_similarity_topk_excl', *args, lists.indptr.data_ptr(), lists.indices.data_ptr(), lists.nnz, _stream())
    return idx, val


class _Operands:
    """Queries and corpus of top_k_similar, similar_pairs and similarity_auroc as their kernels read them.  The constructor only
    checks on the host that both are dense or both sparse (ValueError), so that it runs among the entry point's other argument
    checks; build(device) then makes the device operands.  corpus=None (self mode) ranks the queries against themselves, and the
    corpus operand is the query one."""

    def __init__(self, queries, corpus, metric, fn):
        self.sparse, self.self_mode = sp.issparse(queries), corpus is None
        if corpus is not None and sp.issparse(corpus) != self.sparse:
            raise ValueError('%s: queries and corpus must be both sparse or both dense' % fn)
        self._inputs = (queries,) if corpus is None else (queries, corpus)
        self._metric, self._fn = metric, fn

    def build(self, device):
        """Sets q and c: the bf16 hi / lo pairs of _normalised_operands (rows L2-normalised for 'cosine') of dense rows (arrays or
        tensors), the DeviceCSR of _csr_operand of sparse ones (scipy sparse matrices); n_q, n_c and dim; and rows, the query rows
        before the kernels' normalisation (the device fp32 tensor, or _csr_operand's host CSR).  ValueError when the corpus
        rows are not as wide as the queries.  Returns self."""
        if self.sparse:
            rows = [_csr_operand(x, self._metric) for x in self._inputs]
        else:
            rows = [_as_device_dense(x, device) for x in self._inputs]
        self.rows = rows[0]
        self.n_q, self.dim = rows[0].shape
        self.n_c = rows[-1].shape[0]
        if rows[-1].shape[1] != self.dim:
            raise ValueError('%s: corpus rows have %d columns, queries %d' % (self._fn, rows[-1].shape[1], self.dim))
        if self.sparse:
            ops = [DeviceCSR(m, device) for m in rows]
        else:
            ops = [_normalised_operands(x, 2 if self._metric == 'cosine' else 0)[:2] for x in rows]
        self.q, self.c = ops[0], ops[-1]
        return self


def _group_labels(groups, n, fn):
    """groups as int32 [n] on the host: ValueError unless it is a 1-D integer array of n labels in [0, 2^31)."""
    g = np.asarray(groups.cpu() if isinstance(groups, torch.Tensor) else groups)
    if g.ndim != 1 or g.shape[0] != n:
        raise ValueError('%s: groups has shape %s, [%d] (one label per corpus row) expected' % (fn, g.shape, n))
    if not np.issubdtype(g.dtype, np.integer):
        raise ValueError('%s: groups must hold integers, not %s' % (fn, g.dtype))
    if g.size and (g.min() < 0 or g.max() > np.iinfo(np.int32).max):
        raise ValueError('%s: groups hold a label outside [0, 2^31)' % fn)
    return g.astype(np.int32)


def _read_group_lists(indptr, indices, groups, corpus_groups):
    """recommend's exclusion lists with groups: user u's list holds every corpus position whose group holds an article u read.
    indptr int64 [U + 1] / indices int32: the canonical history CSR over article rows; groups: int32 labels of the article rows;
    corpus_groups: int32 labels of the corpus positions (groups[candidates], or groups).  Torch tensors on one device; vectorised,
    no per-user loop.  Returns (indptr int64 [U + 1], indices int32), rows sorted and without duplicates."""
    dev = indices.device
    n_u, n_c = indptr.numel() - 1, corpus_groups.numel()
    users = torch.repeat_interleave(torch.arange(n_u, device=dev), indptr[1:] - indptr[:-1])
    n_g = max(int(groups.max()), int(corpus_groups.max())) + 1
    pairs = torch.unique(users * n_g + groups[indices.long()].long())              # the (user, group) pairs read, sorted
    p_user, p_group = pairs // n_g, pairs % n_g
    cg = corpus_groups.long()
    order = torch.argsort(cg, stable=True)                                         # corpus positions by group
    cg_sorted = cg[order]
    start = torch.searchsorted(cg_sorted, p_group)
    count = torch.searchsorted(cg_sorted, p_group, right=True) - start
    pair = torch.repeat_interleave(torch.arange(pairs.numel(), device=dev), count)
    offset = torch.arange(pair.numel(), device=dev) - (torch.cumsum(count, 0) - count)[pair]
    keys = torch.sort(p_user[pair] * n_c + order[start[pair] + offset]).values     # groups are disjoint: no duplicates
    out_ptr = torch.zeros(n_u + 1, dtype=torch.int64, device=dev)
    out_ptr[1:] = torch.cumsum(torch.bincount(keys // n_c, minlength=n_u), 0)
    return out_ptr, (keys % n_c).to(torch.int32)


def top_k_similar(embeddings, k=10, corpus=None, metric='cosine', device='cuda:0', to_host=True, splits=0, exclude=None, groups=None,
                  long_lists=False, max_candidates=TOPK_LONG_MAX_CANDIDATES):
    """For every row of `embeddings` the k most similar rows of `corpus` and their scores, best first (among equal scores the
    lower index first), without forming the similarity matrix.  corpus=None ranks the set against itself and leaves each row's
    self match out.  Rows with fewer than k candidates are padded with index -1 and score -inf.  metric: 'cosine' or
    'linear kernel', as in pairwise_similarity.
    Dense inputs (arrays or torch tensors) run on the tensor cores (bf16x3).  Sparse inputs (scipy sparse matrices: the binary /
    tf-idf bag of words) run through dae_csr_similarity_topk, which only spends work on the columns two rows share; every score
    is the fp32 sum of the rounded products in increasing column order.  Queries and corpus must be both dense or both sparse.
    exclude: a scipy sparse matrix [Nq, Nc] whose stored positions (i, j) are never returned for query i (values ignored,
    explicit zeros count), e.g. the articles a user has read; the kernels skip them in their epilogues (dae_*_topk_excl*), and
    the self match stays out with corpus=None.  A wrong shape or an index outside it raises ValueError before any device work.
    groups: an integer array [Nc] of labels >= 0 of the corpus rows (the rows themselves with corpus=None), e.g. duplicate_groups'
    output: rows with equal labels are one story, and at most one row per group is returned -- the group's best candidate by
    (score desc, index asc), with scores bit-identical to the call without groups.  The selection happens in the kernels
    (dae_*_topk_groups*), so a story with many rewrites cannot leave the list short.  It composes with `exclude`: an excluded row
    hands its group to the group's next best candidate.  With corpus=None only the self match is left out; the other members of
    the query's own group remain candidates (pass them in `exclude` to leave them out too).  A wrong length, a non-integer dtype
    or a label outside [0, 2^31) raises ValueError before any device work.
    Returns (index int32 [Nq, k], score float32 [Nq, k]) as ndarrays, or device tensors with to_host=False.  `splits`
    (> 0) fixes the number of corpus parts the work is cut into; it does not change the result.
    1 <= k <= 32, or with long_lists=True 1 <= k <= 1024 for dense inputs (sparse inputs stay at 32: ValueError).  k <= 32 runs
    the register kernels either way; a larger k runs the long-list stages (DESIGN 4.14) with the same contract -- order, ties,
    padding, exclusion and groups -- and the same score bits.  They hold at most max(max_candidates, Nc) candidate pairs at once
    (36 B each at the peak), cutting the queries into chunks of max_candidates // (2k) rows."""
    assert metric in ['cosine', 'linear kernel']
    _check_k(k, long_lists, sp.issparse(embeddings), 'top_k_similar')
    max_candidates = _check_budget(max_candidates, 'top_k_similar')
    ops = _Operands(embeddings, corpus, metric, 'top_k_similar')
    n_c = embeddings.shape[0] if corpus is None else corpus.shape[0]
    if exclude is not None:
        indptr, indices, _ = _stored_positions(exclude, (embeddings.shape[0], n_c), 'exclude', 'top_k_similar')
    g = None if groups is None else _group_labels(groups, n_c, 'top_k_similar')
    ops.build(device)
    lists = None if exclude is None else _DeviceLists.from_host(indptr, indices, device)
    g_dev = None if g is None else torch.from_numpy(g).to(device)
    if ops.sparse:
        idx, val = _csr_similarity_topk(ops.q, ops.c, k, exclude=ops.self_mode, splits=splits, lists=lists, groups=g_dev)
    elif k > TOPK_MAX_K:
        idx, val = _similarity_topk_long(ops.q, ops.c, ops.n_q, ops.n_c, ops.dim, k, exclude=ops.self_mode, splits=splits, lists=lists,
                                         groups=g_dev, max_candidates=max_candidates)
    else:
        idx, val = _similarity_topk(ops.q, ops.c, ops.n_q, ops.n_c, ops.dim, k, exclude=ops.self_mode, splits=splits, lists=lists,
                                    groups=g_dev)
    return _result((idx, val), to_host)


def _history_weights(histories, n_articles, fn):
    """Host side of user_profiles / recommend: the canonical history CSR (U x N, float32) with every row's weights divided by their
    sum (the weighted mean), rows whose weights sum to 0 left at 0, and the boolean mask of those rows (no reads or zero weight)."""
    indptr, indices, w = _stored_positions(histories, (None, n_articles), 'histories', fn)
    if not np.isfinite(w).all():
        raise ValueError('%s: histories hold a weight that is not finite' % fn)
    n_u = len(indptr) - 1
    rows = np.repeat(np.arange(n_u), np.diff(indptr))
    tot = np.bincount(rows, weights=w, minlength=n_u)
    empty = tot == 0
    w = np.where(empty[rows], 0.0, w / np.where(empty, 1.0, tot)[rows]).astype(np.float32)
    m = sp.csr_matrix((w, indices, indptr), shape=(n_u, n_articles))
    m.has_sorted_indices = True
    return m, empty


def _dense_embeddings(embeddings, device, fn):
    from .user_model import ArticleEncoder
    if isinstance(embeddings, ArticleEncoder):   # a fine-tuned article encoder stands for its vectors (DESIGN 4.19)
        return embeddings.vectors(to_host=False)
    if sp.issparse(embeddings):
        raise ValueError('%s: embeddings must be dense (an array or a tensor [N, H]); sparse bag-of-words profiles are not supported' % fn)
    x = _as_device_dense(embeddings, device)
    if x.dim() != 2 or x.shape[0] == 0 or x.shape[1] == 0:
        raise ValueError('%s: embeddings have shape %s, [N, H] with N, H > 0 expected' % (fn, tuple(x.shape)))
    return x


def _profiles(hist, emb):
    """Profiles [U, H] fp32 on the device: hist (DeviceCSR of the normalised weights, U x N) times emb [N, H] through the CSR encode
    kernel with activation none and a zero bias, i.e. exactly X.W."""
    n_u, h = hist.shape[0], emb.shape[1]
    out = torch.empty(n_u, h, dtype=torch.float32, device=emb.device)
    zero_b = torch.zeros(h, dtype=torch.float32, device=emb.device)
    call('dae_encode_csr_fwd', hist.indptr.data_ptr(), hist.indices.data_ptr(), hist.values.data_ptr(), None, n_u, emb.shape[0], h, 1.0,
         emb.data_ptr(), zero_b.data_ptr(), _cabi.ACT['none'], out.data_ptr(), h, None, None, None, 0, _stream())
    return out


def user_profiles(histories, embeddings, device='cuda:0', to_host=True):
    """User profiles from reading histories: row u is the weighted mean of the embeddings of the articles user u read.
    histories: scipy sparse [U, N]; the stored values are the weights (1 for a plain mean, or e.g. decaying with the age of the
    read), repeated positions add up.  embeddings: [N, H] array or tensor (transform()'s output).  The weights are normalised per
    user on the host; a user whose weights sum to 0 (no reads, or zero weights) gets a zero row.  The product runs through the CSR
    encode kernel (dae_encode_csr_fwd, activation none, zero bias).  Returns fp32 [U, H] (ndarray, or a device tensor with
    to_host=False)."""
    if sp.issparse(embeddings):
        _dense_embeddings(embeddings, device, 'user_profiles')
    w, _ = _history_weights(histories, embeddings.shape[0], 'user_profiles')
    emb = _dense_embeddings(embeddings, device, 'user_profiles')
    return _result(_profiles(DeviceCSR(w, device), emb), to_host)


def _candidate_rows(candidates, n, fn):
    c = np.asarray(candidates.cpu() if isinstance(candidates, torch.Tensor) else candidates)
    if c.ndim != 1 or c.size == 0 or not np.issubdtype(c.dtype, np.integer):
        raise ValueError('%s: candidates must be a non-empty 1-D integer array' % fn)
    c = c.astype(np.int64)
    if c.min() < 0 or c.max() >= n:
        raise ValueError('%s: candidates hold a row outside [0, %d)' % (fn, n))
    if c.size > 1 and not (np.diff(c) > 0).all():
        raise ValueError('%s: candidates must be sorted and without duplicates' % fn)
    return c


def _remap_lists(indptr, indices, cand):
    """Exclusion lists over article rows -> lists over candidate positions: entries that are not candidates drop out, the others
    become their position in the sorted `cand` (so each row stays sorted)."""
    pos = np.searchsorted(cand, indices)
    keep = pos < cand.size
    keep[keep] = cand[pos[keep]] == indices[keep]
    rows = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    new_ptr = np.zeros(len(indptr), dtype=np.int64)
    np.cumsum(np.bincount(rows[keep], minlength=len(indptr) - 1), out=new_ptr[1:])
    return new_ptr, pos[keep].astype(np.int32)


def _recommend_request(w, n_art, candidates, groups, exclude_read, device, fn):
    """The request recommend and recommend_sparse share, for the normalised histories w (scipy CSR [U, N]): candidates and groups
    checked on the host (ValueError before any device work), then on the device the history CSR, the candidate rows, the group
    labels of the corpus positions and, with exclude_read, the exclusion lists: every position of a group the user read
    (_read_group_lists), the reads remapped to candidate positions, or the history CSR itself.
    Returns (hist DeviceCSR, cand host int64 or None, cand_dev, corpus group labels or None, lists _DeviceLists or None)."""
    cand = None if candidates is None else _candidate_rows(candidates, n_art, fn)
    g = None if groups is None else _group_labels(groups, n_art, fn)
    hist = DeviceCSR(w, device)
    cand_dev = None if cand is None else torch.from_numpy(cand).to(device)
    g_dev = cg_dev = None
    if g is not None:
        g_dev = torch.from_numpy(g).to(device)
        cg_dev = g_dev if cand_dev is None else g_dev.index_select(0, cand_dev)
    lists = None
    if exclude_read and g is not None:
        ptr, ind = _read_group_lists(hist.indptr, hist.indices, g_dev, cg_dev)
        lists = _DeviceLists(ptr, ind, ind.numel())
    elif exclude_read and cand is not None:
        lists = _DeviceLists.from_host(*_remap_lists(w.indptr, w.indices, cand), device)
    elif exclude_read:
        lists = _DeviceLists(hist.indptr, hist.indices, hist.nnz)
    return hist, cand, cand_dev, cg_dev, lists


def _recommend_result(idx, val, empty, cand_dev, device, to_host):
    """recommend's output from the top-k over the corpus positions: padding rows (-1 / -inf) for the users in `empty`, the
    candidate positions mapped back to article rows."""
    if empty.any():
        e = torch.from_numpy(empty).to(device)
        idx[e] = -1
        val[e] = float('-inf')
    if cand_dev is not None:
        idx = torch.where(idx >= 0, cand_dev[idx.clamp(min=0).long()].int(), idx)
    return _result((idx, val), to_host)


def sequences_from_csr(m):
    """Reading sequences from a scipy sparse [U, N] matrix whose stored values are read times or positions: user u's articles are
    the stored columns of row u ordered by value (ties by column).  Explicit zeros count as reads (time 0).  Returns
    (indptr int64 [U + 1], items int32 [nnz]), the input of user_model.UserGRU."""
    if not sp.issparse(m):
        raise ValueError('sequences_from_csr: a scipy sparse matrix is expected, not %s' % type(m).__name__)
    coo = m.tocoo()
    r, c, v = np.asarray(coo.row, np.int64), np.asarray(coo.col, np.int64), np.asarray(coo.data, np.float64)
    order = np.lexsort((c, v, r))
    indptr = np.zeros(m.shape[0] + 1, dtype=np.int64)
    np.cumsum(np.bincount(r, minlength=m.shape[0]), out=indptr[1:])
    return indptr, c[order].astype(np.int32)


def recommend(histories, embeddings, k=10, candidates=None, metric='cosine', exclude_read=True, device='cuda:0', to_host=True,
              splits=0, profiles=None, groups=None, long_lists=False, max_candidates=TOPK_LONG_MAX_CANDIDATES):
    """For every user the k best articles by `metric` between the user's profile (user_profiles: the weighted mean of the read
    articles' embeddings) and the articles: 'cosine', or 'linear kernel' (the plain inner product).  Order, ties and padding as in
    top_k_similar.  exclude_read: no article of the user's history is returned -- the history goes to the top-k kernel as the
    user's exclusion list, so a long history costs nothing extra on the host.  candidates: an optional sorted int array of rows of
    `embeddings` that may be recommended (e.g. today's articles); the indices returned are rows of `embeddings` either way.
    A user without reads, or whose weights sum to 0, gets a padding row (-1 / -inf).  Embeddings only: dense [N, H].
    profiles: an optional [U, H] array or tensor ranked in place of the mean profiles (e.g. UserGRU.transform's user vectors); the
    histories still give the exclusion lists and the padding rows.
    groups: an integer array [N] of labels >= 0 of the article rows (e.g. duplicate_groups' output): at most one article per group
    is recommended, as in top_k_similar(groups=...).  With exclude_read, every article of a group the user has read is excluded
    too, so a user is not shown a rewrite of a story they read; those lists are built on the device from the histories and the
    labels (over the candidates' positions when candidates are given).
    long_lists / max_candidates: as in top_k_similar -- up to k = 1024 with long_lists=True.
    Returns (index int32 [U, k], score float32 [U, k]) as ndarrays (device tensors with to_host=False)."""
    _check_metric(metric, 'recommend')
    _check_k(k, long_lists, False, 'recommend')
    max_candidates = _check_budget(max_candidates, 'recommend')
    n_art = embeddings.shape[0]
    if sp.issparse(embeddings):
        _dense_embeddings(embeddings, device, 'recommend')
    w, empty = _history_weights(histories, n_art, 'recommend')
    if profiles is not None:
        if sp.issparse(profiles) or tuple(profiles.shape) != (w.shape[0], embeddings.shape[1]):
            raise ValueError('recommend: profiles have shape %s, [%d, %d] (users x embedding width) expected'
                             % (tuple(profiles.shape), w.shape[0], embeddings.shape[1]))
    hist, _, cand_dev, cg_dev, lists = _recommend_request(w, n_art, candidates, groups, exclude_read, device, 'recommend')
    emb = _dense_embeddings(embeddings, device, 'recommend')
    prof = _profiles(hist, emb) if profiles is None else _as_device_dense(profiles, emb.device)
    corpus = emb if cand_dev is None else emb.index_select(0, cand_dev)
    idx, val = _recommend_topk(prof, corpus, k, metric, lists, splits, cg_dev, max_candidates)
    return _recommend_result(idx, val, empty, cand_dev, device, to_host)


def _recommend_topk(prof, corpus, k, metric, lists, splits=0, groups=None, max_candidates=TOPK_LONG_MAX_CANDIDATES):
    """The ranking half of recommend: profiles [U, H] against corpus [Nc, H] on the tensor cores, with the exclusion lists and
    the corpus rows' group labels; k > 32 through the long-list stages."""
    norm_kind = 2 if metric == 'cosine' else 0
    q = _normalised_operands(prof, norm_kind)[:2]
    c = _normalised_operands(corpus, norm_kind)[:2]
    if k > TOPK_MAX_K:
        return _similarity_topk_long(q, c, prof.shape[0], corpus.shape[0], prof.shape[1], k, splits=splits, lists=lists, groups=groups,
                                     max_candidates=max_candidates)
    return _similarity_topk(q, c, prof.shape[0], corpus.shape[0], prof.shape[1], k, splits=splits, lists=lists, groups=groups)


SPARSE_PROFILE_CHUNK_NNZ = 1 << 27   # recommend_sparse: profile entries filled and ranked at once (8 B each: 1 GB)
PROFILE_MAX_FEATURES = 1 << 24       # the profile kernels' column limit


def _data_ptr(t):
    """device pointer of a tensor, NULL when it holds nothing (the CSR exports accept NULL indices / values then)"""
    return t.data_ptr() if t.numel() else None


def _sparse_articles(X, fn):
    """X as the canonical fp32 CSR the profile kernels read: ValueError unless X is a scipy sparse matrix [N, F] with N >= 1 and
    1 <= F <= 2^24."""
    if not sp.issparse(X):
        raise ValueError('%s: X must be a scipy sparse matrix [N, F] (the articles\' bag of words), not %s' % (fn, type(X).__name__))
    if len(X.shape) != 2 or X.shape[0] < 1 or not 1 <= X.shape[1] <= PROFILE_MAX_FEATURES:
        raise ValueError('%s: X has shape %s, [N, F] with N >= 1 and 1 <= F <= 2^24 expected' % (fn, tuple(X.shape)))
    return canonical_csr(X).astype(np.float32)


def _profile_weights(histories, m, fn):
    """_history_weights for the profile kernels, with at least one user."""
    w, empty = _history_weights(histories, m.shape[0], fn)
    if w.shape[0] < 1:
        raise ValueError('%s: histories hold no user' % fn)
    return w, empty


def _profile_structure(hist, x):
    """dae_csr_profiles_count: the row pointers int64 [U + 1] of the profiles hist.X, on the device (DeviceCSR operands)."""
    n_u, n = hist.shape
    p_indptr = torch.empty(n_u + 1, dtype=torch.int64, device=hist.indptr.device)
    call('dae_csr_profiles_count', hist.indptr.data_ptr(), _data_ptr(hist.indices), n_u, n, x.indptr.data_ptr(), _data_ptr(x.indices),
         x.shape[1], p_indptr.data_ptr(), _stream())
    return p_indptr


def _profile_rows(hist, x, p_indptr, p_host, u0, u1, normalise):
    """dae_csr_profiles: the profile rows [u0, u1) (L2-normalised with `normalise`) as a DeviceCSR.  p_indptr: the row pointers on
    the device, p_host: their host copy."""
    dev = hist.indptr.device
    base, nnz = int(p_host[u0]), int(p_host[u1] - p_host[u0])
    indices = torch.empty(nnz, dtype=torch.int32, device=dev)
    values = torch.empty(nnz, dtype=torch.float32, device=dev)
    call('dae_csr_profiles', hist.indptr.data_ptr(), _data_ptr(hist.indices), _data_ptr(hist.values), hist.shape[0], hist.shape[1],
         x.indptr.data_ptr(), _data_ptr(x.indices), _data_ptr(x.values), x.shape[1], p_indptr.data_ptr(), u0, u1 - u0,
         1 if normalise else 0, _data_ptr(indices), _data_ptr(values), _stream())
    return DeviceCSR.from_tensors(p_indptr[u0:u1 + 1] - base, indices, values, (u1 - u0, x.shape[1]))


def _profile_chunks(p_indptr, budget):
    """recommend_sparse's user chunks: consecutive ranges [u0, u1) covering every user, each as long as its profiles hold at most
    `budget` entries together; a user over the budget gets a range of its own.  p_indptr: the host row pointers."""
    n_u, out, u0 = len(p_indptr) - 1, [], 0
    while u0 < n_u:
        u1 = int(np.searchsorted(p_indptr, p_indptr[u0] + budget, side='right')) - 1
        u1 = min(max(u1, u0 + 1), n_u)
        out.append((u0, u1))
        u0 = u1
    return out


def sparse_profiles(histories, X, device='cuda:0', to_host=True):
    """Bag-of-words user profiles: row u is the weighted mean of the rows of X (the articles' binary / tf-idf vectors, scipy
    sparse [N, F], F <= 2^24) that user u read, with the weights of user_profiles (histories: scipy sparse [U, N], normalised per
    user; a user whose weights sum to 0 gets an empty row).  The sparse x sparse product runs on the GPU (dae_csr_profiles_count,
    then dae_csr_profiles) without a dense [U, F] buffer: row u stores the union of the columns of the rows read, explicit zeros
    included, in increasing order, and each value is the fp32 sum of the rounded products w.x in increasing article order.
    Returns a canonical scipy CSR [U, F] fp32, or an engine.DeviceCSR with to_host=False (impression_metrics_sparse takes both)."""
    m = _sparse_articles(X, 'sparse_profiles')
    w, _ = _profile_weights(histories, m, 'sparse_profiles')
    hist, x = DeviceCSR(w, device), DeviceCSR(m, device)
    p_indptr = _profile_structure(hist, x)
    p_host = p_indptr.cpu().numpy()
    out = _profile_rows(hist, x, p_indptr, p_host, 0, w.shape[0], False)
    if not to_host:
        return out
    return sp.csr_matrix((out.values.cpu().numpy(), out.indices.cpu().numpy(), p_host), shape=out.shape)


def recommend_sparse(histories, X, k=10, candidates=None, metric='cosine', exclude_read=True, groups=None, device='cuda:0',
                     to_host=True):
    """recommend for bag-of-words profiles: for every user the k best articles by `metric` between the user's sparse_profiles row
    and the rows of X (scipy sparse [N, F]), ranked by the sparse top-k kernel (dae_csr_similarity_topk*): the content-based
    baseline of the learned user vectors.  'cosine' ranks the L2-normalised profiles (dae_csr_profiles' normalise) against
    the L2-normalised rows of X (as top_k_similar does), 'linear kernel' the plain ones.  Order, ties, padding (-1 / -inf for a
    user whose weights sum to 0), exclude_read, candidates and groups as in recommend.  1 <= k <= 32 (ValueError otherwise).
    The profiles are counted once for all users, then filled and ranked in chunks of users holding at most SPARSE_PROFILE_CHUNK_NNZ
    profile entries (a single larger user is a chunk of its own), so they are never all resident.  The result does not depend on
    the chunks.  Returns (index int32 [U, k], score float32 [U, k]) as ndarrays (device tensors with to_host=False)."""
    _check_metric(metric, 'recommend_sparse')
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= TOPK_MAX_K:
        raise ValueError('recommend_sparse: k = %r is outside the supported range 1 <= k <= %d (sparse profiles rank at most %d)'
                         % (k, TOPK_MAX_K, TOPK_MAX_K))
    k = int(k)
    m = _sparse_articles(X, 'recommend_sparse')
    w, empty = _profile_weights(histories, m, 'recommend_sparse')
    hist, cand, cand_dev, cg_dev, lists = _recommend_request(w, m.shape[0], candidates, groups, exclude_read, device, 'recommend_sparse')
    corpus_host = _csr_operand(m, metric)
    x, corpus = DeviceCSR(m, device), DeviceCSR(corpus_host if cand is None else corpus_host[cand], device)
    n_u = w.shape[0]
    idx = torch.empty(n_u, k, dtype=torch.int32, device=device)
    val = torch.empty(n_u, k, dtype=torch.float32, device=device)
    p_indptr = _profile_structure(hist, x)
    p_host = p_indptr.cpu().numpy()
    l_host = None if lists is None else lists.indptr.cpu().numpy()
    for u0, u1 in _profile_chunks(p_host, SPARSE_PROFILE_CHUNK_NNZ):
        q = _profile_rows(hist, x, p_indptr, p_host, u0, u1, metric == 'cosine')
        chunk_lists = None
        if lists is not None:
            a, b = int(l_host[u0]), int(l_host[u1])
            chunk_lists = _DeviceLists(lists.indptr[u0:u1 + 1] - a, lists.indices[a:b], b - a)
        i, v = _csr_similarity_topk(q, corpus, k, lists=chunk_lists, groups=cg_dev)
        idx[u0:u1] = i
        val[u0:u1] = v
        del q
    return _recommend_result(idx, val, empty, cand_dev, device, to_host)


def recommendation_recall(index, targets):
    """How many held-out reads (e.g. each user's last click) the recommendations find, on the host.  index [U, k] (recommend's
    output, -1 = padding, never a hit); targets: scipy sparse [U, N] whose stored positions are the held-out articles.  Users
    without a target are skipped.  Returns {'users': users counted, 'hit_rate': share of them with at least one target among
    their k, 'recall': mean over them of (targets found) / (their targets)}; NaN when no user counts."""
    index = np.asarray(index.cpu() if isinstance(index, torch.Tensor) else index)
    if index.ndim != 2:
        raise ValueError('recommendation_recall: index has shape %s, [U, k] expected' % (index.shape,))
    indptr, indices, _ = _stored_positions(targets, (index.shape[0], None), 'targets', 'recommendation_recall')
    n_u, n = index.shape[0], targets.shape[1]
    if index.size and index.max() >= n:
        raise ValueError('recommendation_recall: index holds article %d, targets have %d columns' % (index.max(), n))
    n_t = np.diff(indptr)
    use = n_t > 0
    users = int(use.sum())
    if users == 0:
        return {'users': 0, 'hit_rate': float('nan'), 'recall': float('nan')}
    t_keys = np.repeat(np.arange(n_u, dtype=np.int64), n_t) * n + indices   # sorted: canonical CSR
    keys = np.arange(n_u, dtype=np.int64)[:, None] * n + index.astype(np.int64)
    pos = np.minimum(np.searchsorted(t_keys, keys), t_keys.size - 1)
    hits = ((index >= 0) & (t_keys[pos] == keys)).sum(1)
    return {'users': users, 'hit_rate': float((hits[use] > 0).mean()), 'recall': float((hits[use] / n_t[use]).mean())}


def _impression_call(export, operands, n_imp, imp, device):
    """What the impression-metric exports share: the score and metric buffers on `device`, the impression arrays uploaded, and
    export(*operands, indptr, items, clicked, n_imp, scores, metrics, stream) -- unless there is nothing to score.  Returns
    (scores fp32 [nnz], metrics fp64 [I, 4] = AUC, MRR, nDCG@5, nDCG@10, NaN where not scored) as device tensors."""
    scores = torch.empty(imp['items'].size, dtype=torch.float32, device=device)
    metrics = torch.full((n_imp, 4), float('nan'), dtype=torch.float64, device=device)
    if n_imp == 0 or imp['items'].size == 0:
        return scores, metrics
    indptr, items, clicked = (torch.from_numpy(imp[key]).to(device) for key in ('indptr', 'items', 'clicked'))
    call(export, *operands, indptr.data_ptr(), items.data_ptr(), clicked.data_ptr(), n_imp, scores.data_ptr(), metrics.data_ptr(),
         _stream())
    return scores, metrics


def _impression_scores(q, emb, imp, metric):
    """dae_impression_metrics on device tensors: (scores fp32 [nnz], metrics fp64 [I, 4] = AUC, MRR, nDCG@5, nDCG@10) as device
    tensors.  imp: check_impressions' host arrays."""
    operands = (q.data_ptr(), q.stride(0), emb.data_ptr(), emb.stride(0), emb.shape[1], int(metric == 'cosine'))
    return _impression_call('dae_impression_metrics', operands, q.shape[0], imp, emb.device)


def impression_metrics(vectors, embeddings, impressions, metric='linear kernel', device='cuda:0'):
    """Ranking quality on impression logs: for impression i the shown articles are scored against vectors[i] ('linear kernel':
    the inner product, 'cosine': with a zero vector scoring 0) and ranked by score, descending, ties to the earlier position in
    the impression's list.  Per impression: AUC of the clicks against the non-clicks (ties count one half; sklearn's
    roc_auc_score), MRR (the mean of 1 / (rank + 1) over the clicks, as MIND's mrr_score) and nDCG@5 / nDCG@10 with binary gains
    (MIND's ndcg_score).  MIND's scripts leave the order of tied scores to argsort; the tie rule above is the only place where
    the ranks may differ from theirs.  The scores and the metrics come from dae_impression_metrics, one warp per impression.
    vectors: [I, H] query vectors (UserGRU.impression_states, or user_profiles of user_model.prefix_histories); embeddings:
    [N, H]; impressions: a mapping with 'indptr', 'items', 'clicked' (user_model.check_impressions).  Both must be finite with
    every |x| <= 2^63 / sqrt(H), so that no fp32 sum of the kernel overflows (ValueError otherwise).  Under 'cosine' a non-zero
    vector whose fp32 squared norm underflows to 0 (every |x| <= 2^-75, about 2.6e-23) scores 0, as a zero vector does, and one
    whose squared norm is subnormal (below 2^-126) scores without fp32's relative accuracy.
    Returns {'impressions': impressions scored, 'skipped': impressions without a click or without a non-click (left out of the
    means), 'auc', 'mrr', 'ndcg@5', 'ndcg@10': means over the scored ones (NaN when none)}."""
    from .user_model import check_impressions
    _check_metric(metric, 'impression_metrics')
    emb = _dense_embeddings(embeddings, device, 'impression_metrics')
    imp = check_impressions(impressions, emb.shape[0], 'impression_metrics')
    n_imp = imp['indptr'].size - 1
    if sp.issparse(vectors) or tuple(vectors.shape) != (n_imp, emb.shape[1]):
        raise ValueError('impression_metrics: vectors have shape %s, [%d, %d] (impressions x embedding width) expected'
                         % (tuple(vectors.shape), n_imp, emb.shape[1]))
    q = _as_device_dense(vectors, emb.device)
    if not bool(torch.isfinite(emb).all()) or not bool(torch.isfinite(q).all()):
        raise ValueError('impression_metrics: embeddings and vectors must be finite')
    # |x| <= 2^63 / sqrt(H) keeps every fp32 dot product and squared norm of the kernel below 2^126: no inf, so no NaN score
    lim = 2.0 ** 63 / math.sqrt(emb.shape[1])
    if float(emb.abs().max()) > lim or (q.numel() and float(q.abs().max()) > lim):
        raise ValueError('impression_metrics: embeddings and vectors must lie within 2^63 / sqrt(H) = %.3g in magnitude' % lim)
    _, m = _impression_scores(q, emb, imp, metric)
    return _impression_means(m.cpu().numpy(), n_imp)


def _impression_means(m, n_imp):
    """impression_metrics' dict from the per-impression metrics m [I, 4] (NaN rows: impressions left out)."""
    ok = ~np.isnan(m[:, 0])
    mean = m[ok].mean(0) if ok.any() else np.full(4, np.nan)
    return {'impressions': int(ok.sum()), 'skipped': int(n_imp - ok.sum()), 'auc': float(mean[0]), 'mrr': float(mean[1]),
            'ndcg@5': float(mean[2]), 'ndcg@10': float(mean[3])}


def _csr_impression_scores(q, x, imp, metric):
    """dae_csr_impression_metrics on DeviceCSR operands: (scores fp32 [nnz], metrics fp64 [I, 4]) as device tensors."""
    operands = (q.indptr.data_ptr(), _data_ptr(q.indices), _data_ptr(q.values), x.indptr.data_ptr(), _data_ptr(x.indices),
                _data_ptr(x.values), x.shape[0], x.shape[1], int(metric == 'cosine'))
    return _impression_call('dae_csr_impression_metrics', operands, q.shape[0], imp, x.indptr.device)


def impression_metrics_sparse(profiles, X, impressions, metric='linear kernel', device='cuda:0'):
    """impression_metrics for bag-of-words query rows: impression i's shown articles (rows of X, scipy sparse [N, F]) are scored
    against row i of `profiles` -- a scipy sparse [I, F] or sparse_profiles(..., to_host=False), e.g.
    sparse_profiles(user_model.prefix_histories(sequences, impressions, N), X) -- and ranked as impression_metrics ranks them.
    'linear kernel': the fp32 sum of the rounded products over the shared columns in increasing column order (the sparse top-k's
    score of the pair, bit for bit); 'cosine': that over sqrt(qq) sqrt(ee), the squared norms summed the same way, 0 when either
    is 0.  The metrics come from the same device code as impression_metrics' (dae_csr_impression_metrics).  Both matrices must be
    finite with every |x| <= 2^63 / sqrt(F) (ValueError otherwise, before any device work).  Returns impression_metrics' dict."""
    from .user_model import check_impressions
    fn = 'impression_metrics_sparse'
    _check_metric(metric, fn)
    m = _sparse_articles(X, fn)
    imp = check_impressions(impressions, m.shape[0], fn)
    n_imp, n_f = imp['indptr'].size - 1, m.shape[1]
    if not (isinstance(profiles, DeviceCSR) or sp.issparse(profiles)):
        raise ValueError('%s: profiles must be a scipy sparse matrix or sparse_profiles(..., to_host=False), not %s'
                         % (fn, type(profiles).__name__))
    if tuple(profiles.shape) != (n_imp, n_f):
        raise ValueError('%s: profiles have shape %s, [%d, %d] (impressions x features) expected' % (fn, tuple(profiles.shape), n_imp, n_f))
    q_host = None if isinstance(profiles, DeviceCSR) else canonical_csr(profiles).astype(np.float32)
    # |x| <= 2^63 / sqrt(F) keeps every fp32 dot product and squared norm of the kernel below 2^126: no inf, so no NaN score
    lim = 2.0 ** 63 / math.sqrt(n_f)
    if q_host is not None:
        q_ok = bool(np.isfinite(q_host.data).all()) and (q_host.nnz == 0 or float(np.abs(q_host.data).max()) <= lim)
    else:
        v = profiles.values
        q_ok = bool(torch.isfinite(v).all()) and (v.numel() == 0 or float(v.abs().max()) <= lim)
    x_ok = bool(np.isfinite(m.data).all()) and (m.nnz == 0 or float(np.abs(m.data).max()) <= lim)
    if not (q_ok and x_ok):
        raise ValueError('%s: X and profiles must be finite and lie within 2^63 / sqrt(F) = %.3g in magnitude' % (fn, lim))
    x = DeviceCSR(m, device)
    q = profiles if q_host is None else DeviceCSR(q_host, device)
    _, mt = _csr_impression_scores(q, x, imp, metric)
    return _impression_means(mt.cpu().numpy(), n_imp)


def label_precision_at_k(index, query_labels, corpus_labels):
    """Mean over the queries of the fraction of returned neighbours (index [Nq, k] from top_k_similar) whose corpus label equals
    the query's label.  Padding (index -1) is not a neighbour; queries labelled -1, or without any neighbour, are skipped.
    NaN when no query counts."""
    index = np.asarray(index.cpu() if isinstance(index, torch.Tensor) else index)
    ql = np.asarray(query_labels.values if hasattr(query_labels, 'values') else query_labels).reshape(-1)
    cl = np.asarray(corpus_labels.values if hasattr(corpus_labels, 'values') else corpus_labels).reshape(-1)
    assert index.ndim == 2 and index.shape[0] == ql.shape[0]
    valid = index >= 0
    hit = valid & (cl[np.where(valid, index, 0)] == ql[:, None])
    n = valid.sum(1)
    use = (ql != -1) & (n > 0)
    if not use.any():
        return float('nan')
    return float((hit.sum(1)[use] / n[use]).mean())


SIMILAR_PAIRS_FIRST_CAPACITY = 1 << 20   # least slots of similar_pairs' first kernel call (12 MB)
SIMILAR_PAIRS_SLOTS_PER_ROW = 16         # and per query row (192 B): a larger result takes a second call


def _pairs_call(run, n_q, n_c, max_pairs, threshold, device):
    """Two-call protocol of the thresholded-pair kernels: run(count, capacity, i, j, s) accumulates the exact count into the zeroed
    device counter and fills the first `capacity` slots.  The first call gets max(SIMILAR_PAIRS_FIRST_CAPACITY,
    SIMILAR_PAIRS_SLOTS_PER_ROW * n_q) slots (at most max_pairs); only a larger count reallocates exactly `count` slots and runs once
    more.  Returns device tensors (i, j, s) sorted by (i, j)."""
    count = torch.zeros(1, dtype=torch.int64, device=device)   # uint64 in the kernels
    cap = min(max(SIMILAR_PAIRS_FIRST_CAPACITY, SIMILAR_PAIRS_SLOTS_PER_ROW * n_q), max_pairs)

    def alloc(n):
        return (torch.empty(max(n, 1), dtype=torch.int32, device=device), torch.empty(max(n, 1), dtype=torch.int32, device=device),
                torch.empty(max(n, 1), dtype=torch.float32, device=device))
    i, j, s = alloc(cap)
    run(count, cap, i, j, s)
    n = int(count.item())
    if n > max_pairs:
        raise ValueError('similar_pairs: %d pairs reach the threshold %r, more than max_pairs = %d; the output alone would take %d bytes '
                         '(12 B per pair). Raise the threshold or max_pairs.' % (n, threshold, max_pairs, 12 * n))
    if n > cap:
        del i, j, s
        i, j, s = alloc(n)
        count.zero_()
        run(count, n, i, j, s)
        got = int(count.item())
        if got != n:
            raise RuntimeError('similar_pairs: the second call counted %d pairs, the first %d' % (got, n))
    bufs = [i, j, s]
    del i, j, s
    return _sort_pairs(bufs, n, n_q, n_c, device)


def _sort_pairs(bufs, n, n_q, n_c, device):
    """The first n pairs of bufs = [i, j, s] (device int32, int32, float32; i < n_q, j < n_c) sorted by (i, j).  Takes the buffers:
    the list is emptied, so that the caller keeps no reference to them."""
    i, j, s = bufs
    bufs.clear()
    # canonical order: the unique int64 keys i * Nc + j radix-sorted with the scores as payload (dae_pairs_sort), which writes the
    # decoded (i, j) into the key buffer it leaves free.  The first call's unused slots are released first, so from here on the
    # peak is 24 B per pair (two key and two score buffers) plus the sort's fixed scratch (DESIGN 4.8).
    if n == 0:
        return i[:0], j[:0], s[:0]
    keys = i[:n].to(torch.int64)
    keys.mul_(n_c).add_(j[:n])
    s = s[:n].clone() if n < s.shape[0] else s
    del i, j
    bits = max(1, (n_q * n_c - 1).bit_length())
    need = (ctypes.c_int64 * 1)()
    call('dae_pairs_sort_workspace', n, bits, ctypes.addressof(need))
    ws = torch.empty(max(int(need[0]), 16), dtype=torch.uint8, device=device)
    keys_alt = torch.empty_like(keys)
    s_alt = torch.empty_like(s)
    which = (ctypes.c_int32 * 1)()
    call('dae_pairs_sort', n, n_c, bits, keys.data_ptr(), keys_alt.data_ptr(), s.data_ptr(), s_alt.data_ptr(), ws.data_ptr(), ws.numel(),
         ctypes.addressof(which), _stream())
    del ws
    ij = (keys if which[0] else keys_alt).view(torch.int32)   # i in the first n int32s, j in the next n
    s = s_alt if which[0] else s
    del keys, keys_alt, s_alt
    return ij[:n], ij[n:2 * n], s


def _csr_similarity_pairs(q, c, self_mode, tau, max_pairs, threshold):
    """similar_pairs of the DeviceCSR matrices q and c (c is q in self mode) through dae_csr_similarity_pairs: device tensors
    (i, j, s) sorted by (i, j).  tau: the float32 threshold as a Python float (> 0)."""
    dev = q.indptr.device
    n_q, n_c = q.shape[0], c.shape[0]
    need = (ctypes.c_int64 * 1)()
    call('dae_csr_similarity_pairs_workspace', n_q, n_c, c.nnz, c.shape[1], ctypes.addressof(need))
    ws = torch.empty(max(int(need[0]), 16), dtype=torch.uint8, device=dev)

    def run(count, cap, i, j, s):
        call('dae_csr_similarity_pairs', q.indptr.data_ptr(), q.indices.data_ptr(), q.values.data_ptr(), n_q, q.nnz, q.shape[1],
             c.indptr.data_ptr(), c.indices.data_ptr(), c.values.data_ptr(), n_c, c.nnz, c.shape[1], 1 if self_mode else 0, tau,
             ws.data_ptr(), ws.numel(), count.data_ptr(), cap, i.data_ptr(), j.data_ptr(), s.data_ptr(), _stream())
    return _pairs_call(run, n_q, n_c, max_pairs, threshold, dev)


def _similarity_pairs(q, c, n_q, n_c, h, self_mode, tau, max_pairs, threshold):
    """similar_pairs of the bf16 hi / lo operand pairs q and c (c is q in self mode) through dae_similarity_pairs_bf16x3: device
    tensors (i, j, s) sorted by (i, j).  tau: the float32 threshold as a Python float."""
    def run(count, cap, i, j, s):
        call('dae_similarity_pairs_bf16x3', n_q, n_c, h, q[0].data_ptr(), q[1].data_ptr(), q[0].stride(0), c[0].data_ptr(),
             c[1].data_ptr(), c[0].stride(0), 1 if self_mode else 0, tau, count.data_ptr(), cap, i.data_ptr(), j.data_ptr(),
             s.data_ptr(), _stream())
    return _pairs_call(run, n_q, n_c, max_pairs, threshold, q[0].device)


def similar_pairs(data, threshold, corpus=None, metric='cosine', device='cuda:0', to_host=True, max_pairs=1 << 28):
    """Every pair of rows whose similarity reaches `threshold` (near-duplicate articles), without forming the similarity matrix.
    corpus=None: the pairs (i, j) with i > j of `data` against itself, scored S[i, j] with row i as the query.  With a corpus: every
    (i, j) of a query row i and a corpus row j.  A pair qualifies when its fp32 score s >= float32(threshold); NaN never does.
    metric: 'cosine' or 'linear kernel', as in top_k_similar, and the scores are those of top_k_similar bit for bit: dense arrays or
    tensors run on the tensor cores (dae_similarity_pairs_bf16x3, bf16x3), scipy sparse matrices through dae_csr_similarity_pairs
    (fp32 sums over the shared columns), where the threshold must be > 0.  Queries and corpus must be both dense or both sparse.
    Memory beyond the inputs: the operands (dense) or the corpus postings (sparse), the output and the sort of its keys.  The first
    kernel call counts the pairs into max(2^20, 16 Nq) slots (12 B each); more than `max_pairs` qualifying pairs then raise
    ValueError before the full output is allocated, and more than the first capacity take exactly one more call.
    Returns (i int32, j int32, score float32), sorted by (i, j), as ndarrays (device tensors with to_host=False)."""
    _check_metric(metric, 'similar_pairs')
    ops = _Operands(data, corpus, metric, 'similar_pairs')
    try:
        with np.errstate(over='ignore'):   # out of float32 range: inf, refused below
            tau = np.float32(threshold)
    except (TypeError, ValueError):
        raise ValueError('similar_pairs: threshold %r is not a number' % (threshold,))
    if not np.isfinite(tau):
        raise ValueError('similar_pairs: threshold %r is not finite (as float32)' % (threshold,))
    if ops.sparse and not tau > 0:
        raise ValueError('similar_pairs: threshold %r must be > 0 on sparse input: a pair that shares no column scores exactly 0, so '
                         'almost every pair would qualify' % (threshold,))
    if not isinstance(max_pairs, (int, np.integer)) or max_pairs < 0:
        raise ValueError('similar_pairs: max_pairs = %r must be a non-negative integer' % (max_pairs,))
    max_pairs = int(max_pairs)
    tau = float(tau)
    ops.build(device)
    if ops.sparse:
        i, j, s = _csr_similarity_pairs(ops.q, ops.c, ops.self_mode, tau, max_pairs, threshold)
    else:
        i, j, s = _similarity_pairs(ops.q, ops.c, ops.n_q, ops.n_c, ops.dim, ops.self_mode, tau, max_pairs, threshold)
    return _result((i, j, s), to_host)


def _host_ints(a):
    return np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a).reshape(-1)


def duplicate_groups(i, j, n):
    """Connected components of the graph on n rows whose edges are the pairs (i[t], j[t]) (similar_pairs' output): int32 [n], each
    row labelled by the smallest row index of its component, so a row without any pair is its own group.  Runs on the host
    (scipy.sparse.csgraph)."""
    from scipy.sparse.csgraph import connected_components
    i, j = _host_ints(i).astype(np.int64), _host_ints(j).astype(np.int64)
    n = int(n)
    if n < 0 or i.shape != j.shape:
        raise ValueError('duplicate_groups: %d row and %d column indices for n = %d' % (i.size, j.size, n))
    if i.size and (min(i.min(), j.min()) < 0 or max(i.max(), j.max()) >= n):
        raise ValueError('duplicate_groups: pair indices outside [0, %d)' % n)
    if n == 0:
        return np.zeros(0, dtype=np.int32)
    g = sp.coo_matrix((np.ones(i.size, dtype=np.int8), (i, j)), shape=(n, n)).tocsr()
    _, comp = connected_components(g, directed=False)
    first = np.unique(comp, return_index=True)[1]   # the first (smallest) row of each component, components in label order
    return first[comp].astype(np.int32)


def pair_label_agreement(i, j, labels, corpus_labels=None):
    """How well thresholded pairs (similar_pairs' i, j) agree with known groups such as the UCI `story` labels.
    Pairs with a row labelled -1 on either side are skipped.  Returns {'pairs': the pairs counted, 'precision': the share of them
    whose two labels are equal, 'recall': those same-label pairs over all same-label pairs -- sum_l n_l (n_l - 1) / 2 against itself
    (corpus_labels None: i and j index `labels`), sum_l n_q(l) n_c(l) against a corpus}.  NaN where a denominator is 0."""
    i, j = _host_ints(i).astype(np.int64), _host_ints(j).astype(np.int64)
    ql = _host_ints(labels.values if hasattr(labels, 'values') else labels)
    cl = ql if corpus_labels is None else _host_ints(corpus_labels.values if hasattr(corpus_labels, 'values') else corpus_labels)
    if i.shape != j.shape:
        raise ValueError('pair_label_agreement: %d row and %d column indices' % (i.size, j.size))
    li, lj = ql[i], cl[j]
    use = (li != -1) & (lj != -1)
    n_pairs = int(use.sum())
    same = int((use & (li == lj)).sum())
    qv = ql[ql != -1]
    if corpus_labels is None:
        counts = np.unique(qv, return_counts=True)[1].astype(np.int64)
        total = int((counts * (counts - 1) // 2).sum())
    else:
        cv = cl[cl != -1]
        uq, nq = np.unique(qv, return_counts=True)
        uc, nc = np.unique(cv, return_counts=True)
        _, a, b = np.intersect1d(uq, uc, return_indices=True)
        total = int((nq[a].astype(np.int64) * nc[b].astype(np.int64)).sum())
    return {'pairs': n_pairs, 'precision': same / n_pairs if n_pairs else float('nan'), 'recall': same / total if total else float('nan')}


def _group_sizes(labels):
    """R = #related pairs, U = #unrelated pairs of the strict lower triangle among rows with label >= 0."""
    lab = labels[labels >= 0]
    m = int(lab.shape[0])
    counts = np.unique(lab, return_counts=True)[1].astype(np.int64)
    r = int((counts * (counts - 1) // 2).sum())
    return r, m * (m - 1) // 2 - r


def related_unrelated_scores(labels, pairwise_similarity_metrics, device='cuda:0'):
    """The two groups the reference compares (helpers.py:88-97) as ASCENDING device tensors: scores of same-label pairs and
    of different-label pairs of the strict lower triangle, rows labelled -1 dropped."""
    labels = np.asarray(labels.values if hasattr(labels, 'values') else labels).reshape(-1)
    assert labels.shape[0] == pairwise_similarity_metrics.shape[0]
    assert pairwise_similarity_metrics.shape[0] == pairwise_similarity_metrics.shape[1]
    lab_i = np.where(labels >= 0, np.unique(labels, return_inverse=True)[1].reshape(-1), -1).astype(np.int32)  # any numeric dtype
    if isinstance(pairwise_similarity_metrics, torch.Tensor):
        sim = pairwise_similarity_metrics.to(device=device, dtype=torch.float32)
    else:
        sim = torch.from_numpy(np.ascontiguousarray(pairwise_similarity_metrics, dtype=np.float32)).to(device)
    if sim.stride(1) != 1:
        sim = sim.contiguous()
    n = sim.shape[0]
    n_rel, n_unrel = _group_sizes(lab_i)
    rel = torch.empty(max(n_rel, 1), dtype=torch.float32, device=sim.device)
    unrel = torch.empty(max(n_unrel, 1), dtype=torch.float32, device=sim.device)
    cursors = torch.zeros(2, dtype=torch.int64, device=sim.device)
    lab_dev = torch.from_numpy(lab_i).to(sim.device)
    call('dae_pair_partition', sim.data_ptr(), sim.stride(0), n, lab_dev.data_ptr(), rel.data_ptr(), unrel.data_ptr(), cursors.data_ptr(),
         _stream())
    got = cursors.cpu().numpy()
    if int(got[0]) != n_rel or int(got[1]) != n_unrel:
        raise RuntimeError('dae_pair_partition wrote %s pairs, expected (%d, %d)' % (got.tolist(), n_rel, n_unrel))
    return torch.sort(rel[:n_rel])[0], torch.sort(unrel[:n_unrel])[0]   # device radix sort (library call), keys only


def auroc_from_groups(related_sorted, unrelated_sorted):
    """AUROC with 'Related' as the positive class (helpers.py:99-100) = (#(r > u) + #(r == u) / 2) / (R U), counted exactly
    on the device: the smaller group queries the larger (sorted) one."""
    n_rel, n_unrel = int(related_sorted.shape[0]), int(unrelated_sorted.shape[0])
    if n_rel == 0 or n_unrel == 0:
        return float('nan'), 0
    acc = torch.zeros(1, dtype=torch.int64, device=related_sorted.device)
    if n_rel <= n_unrel:
        call('dae_auroc_count', related_sorted.data_ptr(), n_rel, unrelated_sorted.data_ptr(), n_unrel, 1, acc.data_ptr(), _stream())
    else:
        call('dae_auroc_count', unrelated_sorted.data_ptr(), n_unrel, related_sorted.data_ptr(), n_rel, 0, acc.data_ptr(), _stream())
    twice = int(acc.item())
    return twice / (2.0 * n_rel * n_unrel), twice


def _box_stats(d):
    """Quartiles (linear interpolation, as np.percentile / plt.boxplot) and Tukey whiskers of one ASCENDING device tensor."""
    n = int(d.shape[0])
    if n == 0:
        return {'n': 0}

    def pct(q):
        pos = q * (n - 1)
        i0 = int(np.floor(pos))
        i1 = min(i0 + 1, n - 1)
        a, b = float(d[i0].item()), float(d[i1].item())
        return a + (b - a) * (pos - i0)
    q1, med, q3 = pct(0.25), pct(0.5), pct(0.75)
    iqr = q3 - q1
    dd = d.double()   # thresholds are compared in float64, like numpy does on the host
    lim = torch.tensor([q1 - 1.5 * iqr, q3 + 1.5 * iqr], dtype=torch.float64, device=d.device)
    lo_i = int(torch.searchsorted(dd, lim[:1], right=False).item())    # first datum >= q1 - 1.5 IQR
    hi_i = int(torch.searchsorted(dd, lim[1:], right=True).item())     # one past the last datum <= q3 + 1.5 IQR
    return {'q1': q1, 'median': med, 'q3': q3, 'whisker_lo': float(d[lo_i].item()) if lo_i < n else q1,
            'whisker_hi': float(d[hi_i - 1].item()) if hi_i > 0 else q3, 'mean': float(dd.mean().item()), 'n': n}


def visualize_pairwise_similarity(labels, pairwise_similarity_metrics, plot='boxplot', title=None, figsize=(16, 9), save_path=None,
                                  device='cuda:0', **plot_kwargs):
    """Reference helpers.visualize_pairwise_similarity (helpers.py:79-135), numeric part on the GPU: the related / unrelated
    split of the lower triangle, the AUROC shown in its ROC legend and the statistics its boxplot draws (computed on ALL pairs;
    the reference subsamples each group to 1e7 before plotting).  Drawing itself is out of scope (no matplotlib in this image):
    the numbers are returned, and written as JSON next to `save_path` when one is given."""
    assert plot in ['scatter', 'boxplot']
    rel, unrel = related_unrelated_scores(labels, pairwise_similarity_metrics, device=device)
    auroc, twice = auroc_from_groups(rel, unrel)
    out = {'title': title, 'auroc': auroc, 'twice_u': twice, 'related': _box_stats(rel), 'unrelated': _box_stats(unrel)}
    if save_path is not None:
        import json
        import os
        with open(os.path.splitext(save_path)[0] + '.json', 'w') as f:
            json.dump(out, f, indent=1)
    return out


HIST_MIN_BINS, HIST_MAX_BINS = 1 << 10, 1 << 24


def _check_bins(bins):
    if not isinstance(bins, (int, np.integer)) or not HIST_MIN_BINS <= bins <= HIST_MAX_BINS or bins & (bins - 1):
        raise ValueError('bins = %r is not a power of two in [2^10, 2^24]' % (bins,))


def grid_range(max_sq_norm, metric):
    """M of the score grid [-M, M]: 1 for cosine; for the linear kernel the smallest power of two >= (1 - 1e-6) max_i ||x_i||^2,
    which bounds |x_i . x_j| (l2-normalised tf-idf rows get M = 1; 1 as well when every row is zero)."""
    if metric == 'cosine':
        return 1.0
    v = (1.0 - 1e-6) * float(max_sq_norm)
    if not v > 0.0:
        return 1.0
    m, e = math.frexp(v)
    return math.ldexp(1.0, e - 1 if m == 0.5 else e)


def score_bins(scores, M, bins):
    """The bin of every float32 score, as the pair-histogram kernels compute it: clamp(floor(fl32(s + M) * bins / (2M)), 0, bins - 1).
    bins / (2M) is a power of two, so the product is exact and the float32 add is the only rounding; NaN goes to bin 0."""
    with np.errstate(over='ignore', invalid='ignore'):   # +-inf scores clamp into the end bins
        u = (np.asarray(scores, dtype=np.float32) + np.float32(M)) * np.float32(bins / (2.0 * M))
    return np.clip(np.floor(np.where(np.isnan(u), np.float32(0), u)), 0, bins - 1).astype(np.int64)


def _hist_box_stats(counts, total, centres):
    """_box_stats of a group known only by its bin counts: every datum is taken as the centre of its bin."""
    n = int(counts.sum())
    if n == 0:
        return {'n': 0}
    cum = np.cumsum(counts)

    def at(k):
        return float(centres[int(np.searchsorted(cum, k, side='right'))])

    def pct(q):
        pos = q * (n - 1)
        i0 = int(np.floor(pos))
        i1 = min(i0 + 1, n - 1)
        a, b = at(i0), at(i1)
        return a + (b - a) * (pos - i0)
    q1, med, q3 = pct(0.25), pct(0.5), pct(0.75)
    iqr = q3 - q1
    occupied = centres[counts > 0]
    lo = occupied[occupied >= q1 - 1.5 * iqr]
    hi = occupied[occupied <= q3 + 1.5 * iqr]
    return {'q1': q1, 'median': med, 'q3': q3, 'whisker_lo': float(lo.min()) if len(lo) else q1,
            'whisker_hi': float(hi.max()) if len(hi) else q3, 'mean': float(total) / n, 'n': n}


def auroc_from_histograms(hist, sums, M, bins):
    """Host half of similarity_auroc: the related-vs-unrelated AUROC and box statistics from the pair histograms hist [2, bins]
    (row 0 related, row 1 unrelated) and the fp64 score sums [2] of the grid [-M, M].
      twice_u = sum_b n_r[b] (2 sum_{b' < b} n_u[b'] + n_u[b])  -- exact, in Python integers; auroc = twice_u / (2 R U)
      auroc_error_bound = sum_b n_r[b] n_u[b] / (2 R U): the exact AUROC of the same scores lies within it (the bin map is monotone,
      so only pairs that share a bin can be ordered differently, and the grid counts each of those as one half).
    Order statistics are the centres of their bins (quartiles interpolated as np.percentile does, Tukey whiskers on those values),
    the mean comes from the sums.  No related or no unrelated pair: auroc and the bound are NaN, as in the sort path."""
    _check_bins(bins)
    if not M > 0:
        raise ValueError('M = %r must be positive' % (M,))
    hist = np.asarray(hist).astype(np.int64)
    if hist.shape != (2, bins):
        raise ValueError('hist has shape %s, (2, %d) expected' % (hist.shape, bins))
    sums = np.asarray(sums, dtype=np.float64).reshape(2)
    w = 2.0 * M / bins
    centres = -M + (np.arange(bins, dtype=np.float64) + 0.5) * w
    nr, nu = hist[0], hist[1]
    r, u = int(nr.sum()), int(nu.sum())
    if r == 0 or u == 0:
        auroc, twice, bound = float('nan'), 0, float('nan')
    else:
        occ = np.nonzero(nr)[0]
        below = (np.cumsum(nu) - nu)[occ]
        a = nr[occ].astype(object)
        twice = int((a * (2 * below + nu[occ]).astype(object)).sum())   # products reach ~1e23 at 10^6 rows: Python integers
        ties = int((a * nu[occ].astype(object)).sum())
        auroc, bound = twice / (2.0 * r * u), ties / (2.0 * r * u)
    return {'auroc': auroc, 'twice_u': twice, 'auroc_error_bound': bound, 'bin_width': w,
            'related': _hist_box_stats(nr, sums[0], centres), 'unrelated': _hist_box_stats(nu, sums[1], centres)}


def _max_sq_norm_dense(x, chunk=1 << 16):
    return max(float(x[i:i + chunk].double().pow(2).sum(1).max()) for i in range(0, x.shape[0], chunk))


def similarity_auroc(data, labels, metric='cosine', bins=1 << 21, title=None, save_path=None, device='cuda:0'):
    """The numbers of visualize_pairwise_similarity (related-vs-unrelated AUROC and box statistics of the strict lower triangle,
    rows labelled -1 dropped) at any number of rows, without the similarity matrix: the scores are counted into `bins` bins over
    [-M, M] (grid_range) on the GPU and evaluated by auroc_from_histograms.  Dense arrays or tensors run on the tensor cores
    (dae_similarity_pair_hist_bf16x3, bf16x3 scores as top_k_similar); scipy sparse matrices through dae_csr_similarity_pair_hist
    (the fp32 scores of the sparse top_k_similar).  metric: 'cosine' or 'linear kernel'.  Memory beyond the inputs is O(bins) plus
    the operands (dense) or the postings (sparse), never N x N.
    Returns {title, auroc, twice_u, auroc_error_bound, bin_width, related, unrelated}; the exact AUROC of the same scores (the
    sort path) lies within auroc_error_bound of auroc.  Written as JSON next to `save_path` when one is given."""
    hist, sums, M = _pair_histograms(data, labels, metric, bins, device)
    out = {'title': title, **auroc_from_histograms(hist.cpu().numpy(), sums.cpu().numpy(), M, bins)}
    if save_path is not None:
        import json
        import os
        with open(os.path.splitext(save_path)[0] + '.json', 'w') as f:
            json.dump(out, f, indent=1)
    return out


def _pair_histograms(data, labels, metric, bins, device='cuda:0'):
    """Device half of similarity_auroc: (hist int64 [2, bins], sums float64 [2]) device tensors and the grid's M."""
    _check_metric(metric, 'similarity_auroc')
    _check_bins(bins)
    labels = np.asarray(labels.values if hasattr(labels, 'values') else labels).reshape(-1)
    n = data.shape[0]
    if labels.shape[0] != n:
        raise ValueError('similarity_auroc: %d labels for %d rows' % (labels.shape[0], n))
    lab_i = np.where(labels >= 0, np.unique(labels, return_inverse=True)[1].reshape(-1), -1).astype(np.int32)
    lab_dev = torch.from_numpy(lab_i).to(device)
    hist = torch.zeros(2, bins, dtype=torch.int64, device=device)      # uint64 counts in the kernels
    sums = torch.zeros(2, dtype=torch.float64, device=device)
    ops = _Operands(data, None, metric, 'similarity_auroc').build(device)
    q, x = ops.q, ops.rows
    if ops.sparse:
        M = grid_range(float(np.asarray(x.multiply(x).sum(1), dtype=np.float64).max()) if metric != 'cosine' else 1.0, metric)
        need = (ctypes.c_int64 * 1)()
        call('dae_csr_similarity_pair_hist_workspace', n, q.nnz, ops.dim, ctypes.addressof(need))
        ws = torch.empty(max(int(need[0]), 16), dtype=torch.uint8, device=device)
        call('dae_csr_similarity_pair_hist', q.indptr.data_ptr(), q.indices.data_ptr(), q.values.data_ptr(), n, q.nnz, ops.dim,
             lab_dev.data_ptr(), M, bins, ws.data_ptr(), ws.numel(), hist.data_ptr(), sums.data_ptr(), _stream())
    else:
        M = grid_range(_max_sq_norm_dense(x) if metric != 'cosine' else 1.0, metric)
        call('dae_similarity_pair_hist_bf16x3', n, ops.dim, q[0].data_ptr(), q[1].data_ptr(), q[0].stride(0), lab_dev.data_ptr(), M,
             bins, hist.data_ptr(), sums.data_ptr(), _stream())
    return hist, sums, M
