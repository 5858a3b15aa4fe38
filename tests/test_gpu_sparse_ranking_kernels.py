"""The sparse ranking kernels through the C ABI (dae_csr_similarity_topk / _excl / _groups, dae_csr_similarity_pairs,
dae_csr_similarity_pair_hist) against the references of tests/sparse_ranking_oracle.py.

Harness.  Every output has a guard region of sentinels that must survive.  The workspace starts as a byte pattern, its partial-list
area as (+inf, n_corpus - 1) in every slot: after the call the bucket starts, the scan's tile area and the per-bucket postings are
compared with the postings model, and with splits > 1 the partial list of every (query, split) with its exact top k, so a slot
the kernel fails to write shows up.  Counters, histograms and sums start at known non-zero values, since the contract
accumulates.  On dyadic data (sparse_ranking_oracle.dyadic_csr / edge_rows) every partial sum is exact, so lists, pair sets,
histograms and fp64 sums are compared bit for bit; random tf-idf data is bit-exact against the column oracle and within the fp64
bound, and the exports must report the same bits for the same (i, j)."""
import functools
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import ranking_kernel_oracle as ro
import sparse_ranking_oracle as so
from test_auroc_hist_host import host_histograms

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SENT_I = -7
SENT_V = np.float32(-7.25)
GUARD = 40
INF_BITS = 0x7F800000
WS_FILL = 0x5A5A5A5A
MODES = ['kSpTopk', 'kSpHist', 'kSpPairs', 'kSpTopkExcl', 'kSpTopkGroups']   # SpMode, in declaration order
TINY = 2.0 ** -100   # a pairs threshold below every non-zero score here

_PROFILED = None   # _profile_exports: a list receiving (export, kernel names) for every export call


def _call(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    if _PROFILED is None:
        _cabi.call(name, *args)
        return
    # one profiler session around this export alone, so that each launch is attributed to the call that made it
    from torch.profiler import ProfilerActivity, profile
    # A session can come back without any kernel record after many sessions in one process; it is repeated once then (the
    # outputs of a profiled call are not checked, so accumulating them twice does no harm).  A call that launches nothing
    # still shows an empty list.
    for _ in range(2):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _cabi.call(name, *args)
            torch.cuda.synchronize()
        names = [re.sub(r'\s+', '', e.name) for e in prof.events() if e.device_type.name == 'CUDA']
        if names:
            break
    _PROFILED.append((name, names))


def _query(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    return _cabi.query(name, *args)


def _st():
    return torch.cuda.current_stream().cuda_stream


@functools.lru_cache(None)
def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


class Guarded:
    """A device array of n entries followed by GUARD sentinels (optionally starting from `init` instead of the sentinel)."""

    def __init__(self, n, dtype, sent, init=None):
        host = np.full(n + GUARD, sent, dtype)
        if init is not None:
            host[:n] = init
        self.n, self.sent = n, sent
        self.t = _dev(host)

    @property
    def ptr(self):
        return self.t.data_ptr()

    def get(self):
        h = self.t.cpu().numpy()
        g = h[self.n:]
        assert (g.view(np.uint8) == np.full(GUARD, self.sent, h.dtype).view(np.uint8)).all(), 'guard overwritten'
        return h[:self.n]


class Csr:
    """A scipy CSR matrix on the device as given (stored zeros kept); NULL indices / values when it stores nothing."""

    def __init__(self, m):
        m = sp.csr_matrix(m, dtype=np.float32)
        assert all((np.diff(m.indices[m.indptr[r]:m.indptr[r + 1]]) > 0).all() for r in range(m.shape[0]))
        self.m, (self.n, self.F), self.nnz = m, m.shape, int(m.nnz)
        self.indptr = _dev(m.indptr.astype(np.int64))
        self.indices = _dev(m.indices.astype(np.int32)) if self.nnz else None
        self.values = _dev(m.data.astype(np.float32)) if self.nnz else None
        self.args = (self.indptr.data_ptr(), self.indices.data_ptr() if self.nnz else None,
                     self.values.data_ptr() if self.nnz else None, self.n, self.nnz, self.F)


def _same(name, got, want):
    """Bit equality of float32 arrays, +0.0 and -0.0 taken as equal."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    bad = (got.view(np.uint32) != want.view(np.uint32)) & ~((got == 0) & (want == 0))
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError('%s: %d of %d differ; first %s: got %r want %r' % (name, int(bad.sum()), bad.size, i, got[i], want[i]))


def _eq(name, got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    bad = got != want
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError('%s: %d of %d differ; first %s: got %r want %r' % (name, int(bad.sum()), bad.size, i, got[i], want[i]))


def _scores(Q, C, exact=True):
    """The kernel's fp32 scores (column oracle); on dyadic data also asserted equal to fp64."""
    with np.errstate(invalid='ignore', over='ignore'):
        S = so.f32_shared_oracle(Q.m, C.m)
    if exact:
        assert np.array_equal(S.astype(np.float64), (Q.m.astype(np.float64) @ C.m.astype(np.float64).T).toarray())
    return S


# ---------------------------------------------------------------------------------------------------------------------------
# workspace
# ---------------------------------------------------------------------------------------------------------------------------
def _workspace(L, nq, nc, k):
    """The workspace of layout L as a Guarded int32 array: the byte pattern, (+inf, nc - 1) in the partial-list area."""
    words = L['total'] // 4
    init = np.full(words, WS_FILL, np.int32)
    n = nq * L['splits'] * k if L['splits'] > 1 else 0
    init[L['off_val'] // 4:L['off_val'] // 4 + n] = INF_BITS
    init[L['off_idx'] // 4:L['off_idx'] // 4 + n] = nc - 1
    return Guarded(words, np.int32, SENT_I, init), n


def _check_postings(name, C, L, w):
    """The bucket starts, the tile area and the postings the call left in the workspace (int32 words w)."""
    try:
        so.check_postings(C.m, w[:L['n_bucket']], w[L['off_post'] // 4:L['off_post'] // 4 + 2 * C.nnz].reshape(-1, 2))
    except AssertionError as e:
        raise AssertionError('%s: %s' % (name, e))
    _eq(name + ' tile area', w[L['off_tiles'] // 4:L['off_tiles'] // 4 + L['n_tiles']], so.tile_totals(C.m))


# ---------------------------------------------------------------------------------------------------------------------------
# top-k: dae_csr_similarity_topk / _excl / _groups
# ---------------------------------------------------------------------------------------------------------------------------
class Lists:
    """Exclusion lists as the device CSR structure (rows sorted, unique, inside [0, n_corpus))."""

    def __init__(self, rows, n_query):
        rows = [np.unique(np.asarray(r, np.int64)) for r in rows] + [np.zeros(0, np.int64)] * (n_query - len(rows))
        self.rows = rows
        self.indptr = np.concatenate([[0], np.cumsum([r.size for r in rows])]).astype(np.int64)
        self.nnz = int(self.indptr[-1])
        self.d_indptr = _dev(self.indptr)
        self.d_indices = _dev(np.concatenate(rows + [np.zeros(1, np.int64)]).astype(np.int32))
        self.args = (self.d_indptr.data_ptr(), self.d_indices.data_ptr() if self.nnz else None, self.nnz)


def _edge_lists(nq, nc, splits, rng):
    """Per row: empty; the range edges 2047, 2048, 4095, 4096 with every split's first and last row; 40 rows inside one range
    and 40 across a range edge; a whole range; every row; a random subset."""
    bounds = [so.split_rows(nc, splits, s) for s in range(splits)]
    edges = [0, 2047, 2048, 4095, 4096, nc - 1] + [c for b in bounds for c in (b[0], b[1] - 1)]
    rows = []
    for r in range(nq):
        kind = r % 7
        if kind == 0:
            cols = []
        elif kind == 1:
            cols = edges
        elif kind == 2:
            cols = list(range(100, 140)) + list(range(2030, 2070))
        elif kind == 3:
            cols = range(2048, 4096) if nc > 2048 else range(0, nc)
        elif kind == 4:
            cols = range(nc)
        elif kind == 5:
            cols = range(max(0, nc - 2100), nc)
        else:
            cols = rng.choice(nc, rng.integers(0, nc // 2 + 1), replace=False)
        rows.append([c for c in cols if 0 <= c < nc])
    return rows


def _topk(mode, Q, C, k, splits, exclude=False, diag=0, lists=None, groups=None, check_ws=True):
    """One call; returns (idx, val, ws_val [nq, s, k], ws_idx, s) after checking every guard and the postings."""
    nq, nc = Q.n, C.n
    L = so.sp_layout(nq, nc, C.nnz, C.F, k, splits, _sms())
    ws_bytes = _query('dae_csr_similarity_topk_workspace', nq, nc, C.nnz, C.F, k, splits)
    assert ws_bytes == L['total']
    ws, n = _workspace(L, nq, nc, k)
    idx = Guarded(nq * k, np.int32, SENT_I)
    val = Guarded(nq * k, np.float32, SENT_V)
    args = [*Q.args, *C.args, k, diag, 1 if exclude else 0, splits, ws.ptr, ws_bytes, idx.ptr, val.ptr]
    if mode == 'plain':
        assert lists is None and groups is None
        _call('dae_csr_similarity_topk', *args, _st())
    elif mode == 'excl':
        _call('dae_csr_similarity_topk_excl', *args, *(lists if lists is not None else Lists([], nq)).args, _st())
    else:
        g = _dev(np.asarray(groups, np.int32))
        _call('dae_csr_similarity_topk_groups', *args, *(lists.args if lists is not None else (None, None, 0)), g.data_ptr(), _st())
    torch.cuda.synchronize()
    w = ws.get()
    s = L['splits']
    if check_ws:
        _check_postings('%s topk' % mode, C, L, w)
    wv = w[L['off_val'] // 4:L['off_val'] // 4 + n].view(np.float32).reshape(nq, -1, k)
    wi = w[L['off_idx'] // 4:L['off_idx'] // 4 + n].reshape(nq, -1, k)
    return idx.get().reshape(nq, k), val.get().reshape(nq, k), wv, wi, s


def _check_topk(name, mode, S, k, got, allowed, groups):
    idx, val, wv, wi, s = got
    if mode == 'groups':
        want = ro.top_k_groups(S, k, allowed, groups)
    else:
        want = ro.top_k(S, k, allowed)
    _eq(name + ' idx', idx, want[0])
    _same(name + ' val', val, want[1])
    if s > 1:
        pv, pi = so.partial_lists(S, k, s, allowed, groups if mode == 'groups' else None)
        _eq(name + ' partial idx', wi, pi)
        _same(name + ' partial val', wv, pv)
    return want


# (nq, n_corpus, F, r0): queries are corpus rows r0 .. r0 + nq - 1 (a row window); corpus sizes on the range edges
TOPK_SHAPES = [(1, 1, 1, 0), (3, 20, 8, 5), (40, 2047, 50, 2000), (33, 2048, 400, 2015), (65, 2049, 64, 1984),
               (20, 4096, 33, 4070), (70, 4097, 100, 4027)]
TOPK_SPLITS = [1, 2, 7, 0, -1]   # -1: the range count R


@pytest.mark.parametrize('k', [1, 7, 31, 32])
@pytest.mark.parametrize('mode', ['plain', 'excl', 'groups'])
def test_topk_exact(mode, k):
    for t, (nq, nc, F, r0) in enumerate(TOPK_SHAPES):
        rng = np.random.default_rng(1000 * k + t)
        c = so.edge_rows(rng, nc, F)
        C = Csr(c)
        Q = Csr(c[r0:r0 + nq])
        assert Q.n == nq
        S = _scores(Q, C)
        R = so._cdiv(nc, so.SP_W)
        for u, splits in enumerate((TOPK_SPLITS[t % 5], TOPK_SPLITS[(t + 2) % 5])):
            splits = R if splits < 0 else splits
            s = so.sp_splits(nq, R, splits, _sms())
            diag = [0, r0, -5, nc, nc + 7][(t + u + k) % 5]
            exclude = (t + k + u) % 3 != 0
            rows = _edge_lists(nq, nc, s, rng) if mode != 'plain' and (t + u) % 2 == 0 else None
            groups = rng.integers(0, max(1, nc // 3), nc) if mode == 'groups' else None
            got = _topk(mode, Q, C, k, splits, exclude, diag, None if rows is None else Lists(rows, nq), groups)
            allowed = ro.allowed_mask(nq, nc, exclude, diag, rows)
            _check_topk('%s k=%d %s splits=%d diag=%d' % (mode, k, (nq, nc, F), splits, diag), mode, S, k, got, allowed, groups)


def _tfidf(rng, n, F, per_row, signed=True):
    """Random tf-idf-like rows: 0 .. per_row distinct columns, values spread over 2^+-8 (some negative when signed)."""
    rows = [np.sort(rng.choice(F, rng.integers(0, per_row + 1), replace=False)) for _ in range(n)]
    indptr = np.concatenate([[0], np.cumsum([r.size for r in rows])])
    nnz = int(indptr[-1])
    data = rng.random(nnz) * 2.0 ** rng.integers(-8, 8, nnz)
    if signed:
        data *= rng.choice([1, 1, 1, -1], nnz)
    return sp.csr_matrix((data.astype(np.float32), np.concatenate(rows + [np.zeros(0, int)]).astype(np.int32), indptr), shape=(n, F))


def _ratio(name, S, got_idx, got_val, ref, bound):
    """The worst |err| / bound of the listed entries, recorded for the report."""
    m = got_idx >= 0
    r = np.nonzero(m)[0]
    b = bound[r, got_idx[m]]
    err = np.abs(got_val[m].astype(np.float64) - ref[r, got_idx[m]])
    assert (err <= b).all(), '%s: an entry outside its fp64 bound' % name
    return float(np.max(np.where(b > 0, err / np.where(b > 0, b, 1), 0))) if b.size else 0.0


@pytest.mark.parametrize('k', [1, 7, 31, 32])
@pytest.mark.parametrize('mode', ['plain', 'excl', 'groups'])
def test_topk_random_every_split_count_gives_the_same_bits(mode, k):
    nq, nc, F = 24, 9000, 700
    rng = np.random.default_rng(k + 7)
    C = Csr(_tfidf(rng, nc, F, 40))
    Q = Csr(_tfidf(rng, nq, F, 60))
    S = _scores(Q, C, exact=False)
    ref, bound = so.score_bound(Q.m, C.m)
    R = so._cdiv(nc, so.SP_W)
    rows = _edge_lists(nq, nc, 2, rng) if mode != 'plain' else None
    groups = rng.integers(0, 2000, nc) if mode == 'groups' else None
    allowed = ro.allowed_mask(nq, nc, True, 3, rows)
    first = None
    for splits in (1, 2, 7, R, 0):
        got = _topk(mode, Q, C, k, splits, True, 3, None if rows is None else Lists(rows, nq), groups, check_ws=splits == 2)
        _check_topk('%s k=%d splits=%d' % (mode, k, splits), mode, S, k, got, allowed, groups)
        if first is None:
            first = got
        _eq('idx vs splits=1', got[0], first[0])
        _eq('val bits vs splits=1', got[1].view(np.uint32), first[1].view(np.uint32))
    print('\nworst |err| / bound, %s k=%d: %.3g' % (mode, k, _ratio('topk %s' % mode, S, first[0], first[1], ref, bound)))


@pytest.mark.parametrize('mode', ['plain', 'excl', 'groups'])
def test_topk_70000_rows_few_queries(mode):
    """35 ranges: automatic splits clamp at 32 (uneven split widths), the count / scatter kernels run five grid passes and the
    bucket array spans two scan tiles."""
    nq, nc, F, k = 5, 70_000, 400, 32
    assert so._cdiv(nc, 8 * _sms() * 16) >= 4
    rng = np.random.default_rng(70)
    c = so.dyadic_csr(rng, nc, F, 0.02, dup=[(3, 2048), (2047, 4096), (69_999, 69_998), (5, 67_583), (5, 67_584)], share_col=9)
    C = Csr(c)
    Q = Csr(so.dyadic_csr(rng, nq, F, 0.1))
    S = _scores(Q, C)
    L = so.sp_layout(nq, nc, C.nnz, F, k, 0, _sms())
    assert L['splits'] == 32 and L['n_tiles'] == 2
    rows = groups = None
    if mode != 'plain':
        rows = [[], list(range(2040, 2100)) + [69_999], list(range(6144, 8192)), list(range(nc)), rng.choice(nc, 30_000, replace=False)]
    if mode == 'groups':
        groups = rng.integers(0, 20_000, nc)
    for splits in (0, 7):
        got = _topk(mode, Q, C, k, splits, True, 67_583, None if rows is None else Lists(rows, nq), groups)
        _check_topk('%s splits=%d' % (mode, splits), mode, S, k, got, ro.allowed_mask(nq, nc, True, 67_583, rows), groups)


def test_topk_empty_operands():
    """nnz = 0 with NULL indices / values: every score is 0, so the lowest allowed indices are listed."""
    rng = np.random.default_rng(2)
    nq, nc, F, k = 9, 4100, 50, 32
    empty_q = Csr(sp.csr_matrix((nq, F), dtype=np.float32))
    empty_c = Csr(sp.csr_matrix((nc, F), dtype=np.float32))
    full_q = Csr(so.dyadic_csr(rng, nq, F, 0.3))
    full_c = Csr(so.dyadic_csr(rng, nc, F, 0.1))
    rows = _edge_lists(nq, nc, 2, rng)
    for Q, C in ((empty_q, full_c), (full_q, empty_c), (empty_q, empty_c)):
        assert not (Q.nnz and C.nnz)
        S = np.zeros((nq, nc), np.float32)
        for mode in ('plain', 'excl', 'groups'):
            lists = Lists(rows, nq) if mode != 'plain' else None
            groups = np.arange(nc) // 3 if mode == 'groups' else None
            got = _topk(mode, Q, C, k, 0, True, 2, lists, groups)
            allowed = ro.allowed_mask(nq, nc, True, 2, None if lists is None else rows)
            _check_topk('empty %s' % mode, mode, S, k, got, allowed, groups)
            if mode == 'plain':
                assert (got[0][0] == np.arange(1, k + 1) - (np.arange(1, k + 1) <= 2)).all()   # row 0 skips column 2
                assert (got[1] == 0).all()


def test_topk_fewer_candidates_than_k():
    rng = np.random.default_rng(3)
    for nc in (1, 5, 31):
        c = so.dyadic_csr(rng, nc, 12, 0.5)
        C = Csr(c)
        Q = Csr(so.dyadic_csr(rng, 4, 12, 0.5))
        S = _scores(Q, C)
        rows = [[0], [], list(range(nc)), [nc - 1]]
        for mode in ('plain', 'excl', 'groups'):
            got = _topk(mode, Q, C, 32, 1, True, 1, Lists(rows, 4) if mode != 'plain' else None,
                        np.zeros(nc) if mode == 'groups' else None)
            allowed = ro.allowed_mask(4, nc, True, 1, rows if mode != 'plain' else None)
            want = _check_topk('nc=%d %s' % (nc, mode), mode, S, 32, got, allowed, np.zeros(nc) if mode == 'groups' else None)
            assert (want[0][:, max(nc, 1):] == -1).all() and np.isneginf(got[1][got[0] < 0]).all()


@pytest.mark.parametrize('k', [7, 32])
def test_excl_empty_lists_and_identity_groups_give_the_plain_bits(k):
    nq, nc, F = 40, 4200, 60
    rng = np.random.default_rng(k)
    c = so.edge_rows(rng, nc, F, dup=((5, 2047), (2047, 2048), (4095, 4096), (2048, 4097), (100, 2100)))
    C = Csr(c)
    Q = Csr(c[2020:2020 + nq])
    S = _scores(Q, C)
    for splits in (1, 3, 0):
        plain = _topk('plain', Q, C, k, splits, True, 2020)
        empty = _topk('excl', Q, C, k, splits, True, 2020, Lists([], nq))
        ident = _topk('groups', Q, C, k, splits, True, 2020, None, np.arange(nc))
        for name, got in (('empty lists', empty), ('identity groups', ident)):
            for a, b in zip(plain[:4], got[:4]):
                assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), name
        _check_topk('plain splits=%d' % splits, 'plain', S, k, plain, ro.allowed_mask(nq, nc, True, 2020), None)
        rows = _edge_lists(nq, nc, plain[4], rng)
        L = Lists(rows, nq)
        ex = _topk('excl', Q, C, k, splits, True, 2020, L)
        gi = _topk('groups', Q, C, k, splits, True, 2020, L, np.arange(nc))
        for a, b in zip(ex[:4], gi[:4]):
            assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))
        _check_topk('excl splits=%d' % splits, 'excl', S, k, ex, ro.allowed_mask(nq, nc, True, 2020, rows), None)


@pytest.mark.parametrize('k', [7, 32])
def test_groups_edges(k):
    """Duplicates across range and split edges sharing a group, a single group, fewer groups than k, groups with lists."""
    nq, nc, F = 30, 6200, 40
    rng = np.random.default_rng(k + 1)
    c = so.edge_rows(rng, nc, F, dup=((5, 2047), (2047, 2048), (4095, 4096), (2048, 4097), (2048, 6199), (4097, 6144)))
    C = Csr(c)
    Q = Csr(c[4080:4080 + nq])
    S = _scores(Q, C)
    straddle = np.arange(nc) % 2048            # rows c, c + 2048, c + 4096 share a label: one per range
    dup_groups = np.arange(nc)
    for src, dst in ((5, 2047), (2047, 2048), (4095, 4096), (2048, 4097), (2048, 6199), (4097, 6144)):
        dup_groups[dst] = dup_groups[src]
    for splits in (1, 2, 3):
        s = so.sp_splits(nq, 4, splits, _sms())
        rows = _edge_lists(nq, nc, s, rng)
        for name, g, lists in (('straddle', straddle, None), ('duplicates', dup_groups, rows), ('one group', np.zeros(nc), rows),
                               ('few groups', np.arange(nc) % 3, None), ('few groups, lists', np.arange(nc) % 5, rows)):
            got = _topk('groups', Q, C, k, splits, True, 4080, None if lists is None else Lists(lists, nq), g)
            _check_topk('%s splits=%d' % (name, splits), 'groups', S, k, got, ro.allowed_mask(nq, nc, True, 4080, lists), g)
            if name.startswith('one'):
                assert (got[0][:, 1:] == -1).all()


def test_topk_infinities_and_nan():
    """+inf is listed; NaN (inf times a stored 0) and -inf never are, so a row whose every candidate is such a score is padding."""
    x = so.inf_rows()
    Q = C = Csr(x)
    S = _scores(Q, C, exact=False)
    assert np.isnan(S).any() and np.isposinf(S).any() and np.isneginf(S).any()
    for mode in ('plain', 'excl', 'groups'):
        for k in (1, 7, 8):
            groups = np.array([0, 1, 0, 1, 2, 2, 3, 3]) if mode == 'groups' else None
            got = _topk(mode, Q, C, k, 1, False, 0, None, groups)
            _check_topk('inf %s k=%d' % (mode, k), mode, S, k, got, None, groups)
            assert not np.isnan(got[1]).any() and not (np.isneginf(got[1]) & (got[0] >= 0)).any()
    # a query whose candidates all score NaN or -inf: padding only; one corpus row with -1 gives the one +inf entry
    col0 = np.array([1, 2, 0, np.inf, -1], np.float32)
    c = sp.csr_matrix((col0, np.zeros(5, np.int32), np.arange(6)), shape=(5, 3))
    q = sp.csr_matrix((np.array([-np.inf], np.float32), np.zeros(1, np.int32), np.array([0, 1])), shape=(1, 3))
    for n_c, want_i in ((4, []), (5, [4])):
        C = Csr(c[:n_c])
        for mode in ('plain', 'excl', 'groups'):
            got = _topk(mode, Csr(q), C, 7, 1, False, 0, None, np.arange(n_c) if mode == 'groups' else None)
            assert got[0][0].tolist() == want_i + [-1] * (7 - len(want_i)), (mode, got[0])
            assert np.isposinf(got[1][0, :len(want_i)]).all() and np.isneginf(got[1][0, len(want_i):]).all()


# ---------------------------------------------------------------------------------------------------------------------------
# thresholded pairs: dae_csr_similarity_pairs
# ---------------------------------------------------------------------------------------------------------------------------
def _pairs(Q, C, self_mode, tau, capacity, count0=0, check_ws=True):
    L = so.sp_layout(Q.n, C.n, C.nnz, C.F, 0, 0, _sms())
    ws_bytes = _query('dae_csr_similarity_pairs_workspace', Q.n, C.n, C.nnz, C.F)
    assert ws_bytes == L['total']
    ws, _ = _workspace(L, Q.n, C.n, 0)
    n_out = max(capacity, 1)
    i_out, j_out = Guarded(n_out, np.int32, SENT_I), Guarded(n_out, np.int32, SENT_I)
    s_out = Guarded(n_out, np.float32, SENT_V)
    cnt = Guarded(1, np.uint64, np.uint64(0x5A5A5A5A5A5A5A5A), np.uint64(count0))
    _call('dae_csr_similarity_pairs', *Q.args, *C.args, 1 if self_mode else 0, float(tau), ws.ptr, ws_bytes, cnt.ptr, capacity,
          i_out.ptr if capacity else None, j_out.ptr if capacity else None, s_out.ptr if capacity else None, _st())
    torch.cuda.synchronize()
    w = ws.get()
    if check_ws:
        _check_postings('pairs', C, L, w)
    return int(cnt.get()[0]) - count0, i_out.get(), j_out.get(), s_out.get()


def _check_triples(name, got, want, written):
    """The `written` slots hold distinct triples of `want`, with its score bits; all of them when written is its size."""
    i, j, s = got
    key = i[:written].astype(np.int64) * (1 << 32) + j[:written]
    assert np.unique(key).size == written, '%s: a pair listed twice' % name
    wk = want[0].astype(np.int64) * (1 << 32) + want[1]
    pos = np.searchsorted(wk, key)
    assert (pos < wk.size).all() and np.array_equal(wk[np.minimum(pos, wk.size - 1)], key), '%s: a pair outside the set' % name
    _same(name + ' scores', s[:written], want[2][pos])
    if written == wk.size:
        assert np.array_equal(np.sort(key), wk)


PAIR_DUPS = ((3, 127), (127, 128), (200, 255), (255, 256), (5, 2047), (2047, 2048), (4095, 4096), (2048, 4097))


@pytest.mark.parametrize('self_mode', [True, False])
@pytest.mark.parametrize('n', [2, 130, 2049, 4097])
def test_pairs_exact(self_mode, n):
    """Pairs on the 128-slot chunk and 2048-row range edges (duplicated rows), thresholds equal to exact scores (s >= tau), the
    capacity protocol on top of a non-zero counter start."""
    rng = np.random.default_rng(n + self_mode)
    c = so.edge_rows(rng, n, 30, dup=PAIR_DUPS)
    C = Csr(c)
    Q = C if self_mode else Csr(sp.vstack([c[max(0, n - 60):], so.dyadic_csr(rng, 7, 30, 0.3)]).tocsr())
    S = _scores(Q, C)
    pos = np.sort(S[np.tril_indices(Q.n, -1)] if self_mode else S.ravel())
    pos = pos[pos > 0]
    taus = [TINY] + ([float(pos[0]), float(pos[pos.size // 2]), float(pos[-1])] if pos.size else [])
    for tau in taus:
        want = ro.pairs_set(S, tau, self_mode)
        m = want[0].size
        for cap, c0 in ((m + 5, 3), (m, 0), (max(m - 1, 2) if m > 2 else 0, 11), (0, 5)):
            got_n, i, j, s = _pairs(Q, C, self_mode, tau, cap, c0, check_ws=cap == m)
            assert got_n == m, (tau, cap, got_n, m)
            first, end = min(c0, cap), min(c0 + m, cap)
            if cap:
                # slots below the counter's start and at or past its end stay untouched
                assert (i[:first] == SENT_I).all() and (i[end:] == SENT_I).all() and (s[end:].view(np.uint32) == SENT_V.view(np.uint32)).all()
                _check_triples('pairs n=%d tau=%r cap=%d' % (n, tau, cap), (i[first:end], j[first:end], s[first:end]), want, end - first)


# ---------------------------------------------------------------------------------------------------------------------------
# pair histogram: dae_csr_similarity_pair_hist
# ---------------------------------------------------------------------------------------------------------------------------
def _hist(X, labels, M, bins, h0, s0, check_ws=True):
    L = so.sp_layout(X.n, X.n, X.nnz, X.F, 0, 0, _sms())
    ws_bytes = _query('dae_csr_similarity_pair_hist_workspace', X.n, X.nnz, X.F)
    assert ws_bytes == L['total']
    ws, _ = _workspace(L, X.n, X.n, 0)
    hist = Guarded(2 * bins, np.uint64, np.uint64(0xA5A5A5A5A5A5A5A5), h0)
    sums = Guarded(2, np.float64, np.float64(-1234.5), s0)
    lab = _dev(np.asarray(labels, np.int32))
    _call('dae_csr_similarity_pair_hist', X.args[0], X.args[1], X.args[2], X.n, X.nnz, X.F, lab.data_ptr(), float(M), bins, ws.ptr,
          ws_bytes, hist.ptr, sums.ptr, _st())
    torch.cuda.synchronize()
    w = ws.get()
    if check_ws:
        _check_postings('hist', X, L, w)
    return hist.get().astype(np.int64).reshape(2, bins) - h0.astype(np.int64).reshape(2, bins), sums.get() - s0


@pytest.mark.parametrize('n', [2, 2047, 2048, 2049, 4097])
def test_pair_hist_exact(n):
    """Scores beyond +-M land in both end bins, all-zero rows fill the zero bin of each group, labels include -1."""
    rng = np.random.default_rng(n)
    x = so.edge_rows(rng, n, 24, dup=PAIR_DUPS)
    X = Csr(x)
    S = _scores(X, X)
    M = 2.0 ** -1
    low = S[np.tril_indices(n, -1)]
    if n > 100:
        assert (low > M).any() and (low < -M).any() and (low == 0).any()
    for bins in ((1 << 10, 1 << 24) if n in (2, 2049) else (1 << 10,)):
        for labels in (np.full(n, -1), np.zeros(n, np.int64), rng.integers(-1, 9, n), np.arange(n) % 2):
            h0 = rng.integers(0, 1 << 40, 2 * bins).astype(np.uint64)
            s0 = np.array([1.5, -2.25])
            hist, sums = _hist(X, labels, M, bins, h0, s0, check_ws=bins == 1 << 10)
            want_h, want_s, _, _ = host_histograms(S, labels, M, bins)
            _eq('hist n=%d bins=%d' % (n, bins), hist, want_h)
            _eq('sums n=%d' % n, sums, want_s)   # dyadic scores: the fp64 sums are exact in any order


def test_pair_hist_nan_and_inf_scores():
    """A NaN score is counted in bin 0 of its group and makes that group's sum NaN; +-inf land in the end bins."""
    x = so.inf_rows()
    X = Csr(x)
    S = _scores(X, X, exact=False)
    M, bins = 4.0, 1 << 10
    for labels in (np.zeros(8, np.int64), np.array([0, 1, 0, 1, 0, 1, 0, 1]), np.array([0, 0, 1, 0, 2, 2, -1, 0])):
        hist, sums = _hist(X, labels, M, bins, np.full(2 * bins, 3, np.uint64), np.array([0.5, 0.25]))
        want_h, want_s, _, _ = host_histograms(S, labels, M, bins)
        _eq('hist', hist, want_h)
        assert np.array_equal(sums, want_s, equal_nan=True), (sums, want_s)
    assert np.isnan(sums[0]) or np.isnan(sums[1])


# ---------------------------------------------------------------------------------------------------------------------------
# a hashed 2^24-column vocabulary: 10 241 scan tiles
# ---------------------------------------------------------------------------------------------------------------------------
def _hashed_corpus(rng, n=8193, F=1 << 24):
    """Every third row one entry from 40 shared columns (0 and F - 1 among them), every seventh row one more hashed column."""
    pool = np.concatenate([[0, F - 1], rng.choice(F, 38, replace=False)])
    rows, cols, vals = [], [], []
    for r in range(n):
        c = []
        if r % 3 == 0:
            c.append(int(pool[(r // 3) % pool.size]))
        if r % 7 == 0:
            c.append(int(rng.integers(0, F)))
        c = sorted(set(c))
        rows += [r] * len(c)
        cols += c
        vals += (rng.integers(1, 8, len(c)) * 0.125).tolist()
    x = sp.csr_matrix((np.array(vals, np.float32), (np.array(rows), np.array(cols))), shape=(n, F))
    x.sort_indices()
    return x


def test_hashed_vocabulary():
    rng = np.random.default_rng(24)
    x = _hashed_corpus(rng)
    X = Csr(x)
    n, F = X.n, X.F
    L = so.sp_layout(n, n, X.nnz, F, 0, 0, _sms())
    assert L['n_tiles'] == 10241 and 0 in x.indices and F - 1 in x.indices
    # top-k: the last rows as queries (a window reaching the one-row last range)
    r0, k = n - 45, 32
    Q = Csr(x[r0:])
    S = _scores(Q, X)
    got = _topk('plain', Q, X, k, 0, True, r0)
    _check_topk('hashed topk', 'plain', S, k, got, ro.allowed_mask(Q.n, n, True, r0), None)
    # pairs (self) and the histogram of every pair
    pi, pj, ps = so.sparse_self_pairs(x)
    keep = ps >= TINY
    want = (pi[keep], pj[keep], ps[keep])
    got_n, i, j, s = _pairs(X, X, True, TINY, want[0].size + 3)
    assert got_n == want[0].size > 1000
    _check_triples('hashed pairs', (i, j, s), want, got_n)
    labels = rng.integers(-1, 5, n)
    M, bins = 4.0, 1 << 12
    hist, sums = _hist(X, labels, M, bins, np.full(2 * bins, 17, np.uint64), np.array([3.0, -1.0]))
    want_h, want_s = so.hist_from_pairs(n, labels, pi, pj, ps, M, bins)
    _eq('hashed hist', hist, want_h)
    _eq('hashed sums', sums, want_s)


# ---------------------------------------------------------------------------------------------------------------------------
# random data: the same bits from every export, within the fp64 bound
# ---------------------------------------------------------------------------------------------------------------------------
def test_cross_export_bits_on_random_data():
    n, F, k = 2500, 3000, 32
    rng = np.random.default_rng(11)
    x = _tfidf(rng, n, F, 30, signed=False)
    X = Csr(x)
    S = _scores(X, X, exact=False)
    ref, bound = so.score_bound(x, x)
    # every positive score of the lower triangle, from the pairs export (self mode, the least threshold)
    want = ro.pairs_set(S, TINY, True)
    got_n, pi, pj, ps = _pairs(X, X, True, TINY, want[0].size)
    assert got_n == want[0].size
    _check_triples('pairs', (pi, pj, ps), want, got_n)
    P = np.zeros((n, n), np.float32)
    P[pi, pj] = ps
    worst = {'pairs': float(np.max(np.abs(ps - ref[pi, pj]) / bound[pi, pj]))}
    # top-k: every listed (i, j) with j < i and a positive score has the pairs' bits
    idx, val, _, _, _ = _topk('plain', X, X, k, 0, True, 0)
    _check_topk('topk', 'plain', S, k, (idx, val, None, None, 1), ro.allowed_mask(n, n, True, 0), None)
    m = (idx >= 0) & (idx < np.arange(n)[:, None]) & (val > 0)
    _eq('topk vs pairs bits', val[m].view(np.uint32), P[np.nonzero(m)[0], idx[m]].view(np.uint32))
    worst['topk'] = _ratio('cross topk', S, idx, val, ref, bound)
    # the histogram bins those same bits
    labels = rng.integers(-1, 5, n)
    M, bins = 2.0 ** int(np.ceil(np.log2(S.max() * 1.01))), 1 << 16
    hist, sums = _hist(X, labels, M, bins, np.zeros(2 * bins, np.uint64), np.zeros(2))
    want_h, want_s = so.hist_from_pairs(n, labels, pi.astype(np.int64), pj.astype(np.int64), ps, M, bins)
    _eq('hist', hist, want_h)
    mag = np.abs(ps).astype(np.float64).sum()
    assert (np.abs(sums - want_s) <= got_n * 2.0 ** -52 * mag).all(), (sums, want_s)
    print('\nworst |err| / bound: %s' % worst)
    assert max(worst.values()) <= 1.0


# ---------------------------------------------------------------------------------------------------------------------------
# which kernels ran
# ---------------------------------------------------------------------------------------------------------------------------
def _sp_mode(name):
    m = re.search(r'sp_topk_kernel<(.+?)>\(', name) or re.search(r'sp_topk_kernel<(.+)>', name)
    arg = m.group(1)
    t = re.search(r'(\d+)$', arg)
    return MODES[int(t.group(1))] if t else arg.split('::')[-1]


def _profile_exports():
    """Each export call in its own profiler session; returns [(export, kernel names in launch order, expected)]."""
    global _PROFILED
    rng = np.random.default_rng(1)
    expect = []
    _PROFILED = []
    X = Csr(so.dyadic_csr(rng, 3000, 3000, 0.01))
    _hist(X, np.zeros(3000), 4.0, 1024, np.zeros(2048, np.uint64), np.zeros(2), check_ws=False)
    expect.append(dict(mode='kSpHist', tiles=so.sp_layout(3000, 3000, X.nnz, 3000, 0, 0, _sms())['n_tiles'], merge=None))
    for nq, nc, F, splits in ((5, 5000, 400, 0), (5, 5000, 5000, 1), (4000, 3000, 50, 0)):
        C = Csr(so.dyadic_csr(rng, nc, F, 0.01))
        Q = Csr(so.dyadic_csr(rng, nq, F, 0.05))
        L = so.sp_layout(nq, nc, C.nnz, F, 7, splits, _sms())
        g = np.arange(nc) // 3
        _topk('plain', Q, C, 7, splits, check_ws=False)
        _topk('excl', Q, C, 7, splits, lists=Lists([[1, 2]], nq), check_ws=False)
        _topk('groups', Q, C, 7, splits, groups=g, check_ws=False)
        for mode, merge in (('kSpTopk', 'topk_merge_kernel'), ('kSpTopkExcl', 'topk_merge_kernel'),
                            ('kSpTopkGroups', 'topk_merge_groups_kernel')):
            expect.append(dict(mode=mode, tiles=L['n_tiles'], merge=merge if L['splits'] > 1 else None))
        _pairs(Q, C, False, 2.0 ** -6, 10, check_ws=False)
        expect.append(dict(mode='kSpPairs', tiles=L['n_tiles'], merge=None))
    record, _PROFILED = _PROFILED, None
    assert len(record) == len(expect), [r[0] for r in record]
    return [(export, names, want) for (export, names), want in zip(record, expect)]


def test_profiler_sees_every_dispatch():
    """The profiler runs in a process of its own: CUPTI's activity state is per process, and the profiler sessions of earlier
    tests in a long pytest process can leave later sessions without kernel records."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ('import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_sparse_ranking_kernels as t; '
            'print("RESULT " + json.dumps(t._profile_exports()))' % (here, os.path.dirname(here)))
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=600, cwd=os.path.dirname(here))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    record = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith('RESULT ')][-1][7:])
    seen_tiles, seen_merge = set(), set()
    for export, names, want in record:
        count = lambda s: sum(s in n for n in names)  # noqa: E731  (no kernel name here contains another)
        what = (export, [n[:80] for n in names])
        assert count('sp_count_kernel') == 1 and count('sp_scatter_kernel') == 1, what
        multi = want['tiles'] > 1
        seen_tiles.add(multi)
        assert count('sp_scan_tiles_kernel') == (2 if multi else 1), what
        assert count('sp_add_tile_offsets_kernel') == (1 if multi else 0), what
        modes = [_sp_mode(n) for n in names if 'sp_topk_kernel<' in n]
        assert modes == [want['mode']], (what, modes)
        merges = [m for m in ('topk_merge_kernel', 'topk_merge_groups_kernel') if count(m)]
        assert merges == ([want['merge']] if want['merge'] else []), (what, merges)
        seen_merge.add(want['merge'])
    assert seen_tiles == {False, True} and seen_merge == {None, 'topk_merge_kernel', 'topk_merge_groups_kernel'}
    assert {w['mode'] for _, _, w in record} == set(MODES)
