"""The dense ranking kernels through the C ABI (dae_similarity_topk_bf16x3 / _excl_ / _groups_, the long-list stages
dae_similarity_topk_bound_bf16x3 / _collect_bf16x3 / dae_pairs_sort / dae_similarity_topk_select, dae_similarity_pairs_bf16x3 and
dae_similarity_pair_hist_bf16x3) against the references of tests/ranking_kernel_oracle.py.

Harness.  Operands have ld above dim with bf16 NaN in [dim, ld) of hi and lo and a NaN row after the last, so only TMA's zero fill
can give the tile tails.  Every output has a guard region of sentinels that must survive.  The top-k workspace starts as
(+inf, n_corpus - 1) in every slot: a slot the kernel fails to write shows up in the partial lists, which are checked against the
model of each (row, split, half) list, and no index can leave the corpus.  Counters, row counts, histograms and sums start at
known non-zero values, since the contract accumulates.  On exact operands (gemm_kernel_oracle.exact_operands) every score is
known bit for bit, so lists, taus, pair sets, histograms and fp64 sums are compared exactly; random data scaled over 2^+-20 is
checked against fp64 within the per-element bound, and the exports must report the same bits for the same (i, j)."""
import ctypes
import functools
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import gemm_kernel_oracle as gk
import ranking_kernel_oracle as ro
from mining_kernel_oracle import bf16_split
from test_auroc_hist_host import host_histograms

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SENT_I = -7
SENT_V = np.float32(-7.25)
GUARD = 40
INF_BITS = 0x7F800000


_PROFILED = None   # _profile_exports: a list receiving (export, kernel names) for every export call


def _call(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    if _PROFILED is None:
        _cabi.call(name, *args)
        return
    # one profiler session around this export alone, so that each launch is attributed to the call that made it
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _cabi.call(name, *args)
        torch.cuda.synchronize()
    _PROFILED.append((name, {re.sub(r'\s+', '', e.name) for e in prof.events() if e.device_type.name == 'CUDA'}))


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


class Operand:
    """bf16 bit arrays [rows x dim] -> device hi / lo [rows + 1 x ld], ld > dim a multiple of 8, NaN outside the matrix."""

    def __init__(self, hi, lo):
        rows, dim = hi.shape
        self.ld = (dim + 8) // 8 * 8 + 8
        bufs = []
        for bits in (hi, lo):
            b = np.full((rows + 1, self.ld), gk.BF16_NAN, np.uint16)
            b[:rows, :dim] = bits
            bufs.append(_dev(b.view(np.int16)))
        self.hi, self.lo = bufs
        self.args = (self.hi.data_ptr(), self.lo.data_ptr(), self.ld)


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


def _same(name, got, want):
    """Bit equality of float32 arrays, +0.0 and -0.0 taken as equal (the sign of an exact zero sum is not part of the contract)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    bad = (got.view(np.uint32) != want.view(np.uint32)) & ~((got == 0) & (want == 0))
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError('%s: %d of %d differ; first %s: got %r want %r' % (name, int(bad.sum()), bad.size, i, got[i], want[i]))


def _eq(name, got, want):
    got, want = np.asarray(got), np.asarray(want)
    bad = got != want
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError('%s: %d of %d differ; first %s: got %r want %r' % (name, int(bad.sum()), bad.size, i, got[i], want[i]))


def _exact(nq, nc, dim, seed, dup=0, self_mode=False):
    """Exact operands and their fp32 scores; `dup` corpus rows copied from others (ties at different indices)."""
    rng = np.random.default_rng(seed)
    q = gk.exact_operands(rng, nq, dim)
    c = q if self_mode else gk.exact_operands(rng, nc, dim)
    if dup and not self_mode:
        src, dst = rng.integers(0, nc, dup), rng.integers(0, nc, dup)
        c[0][dst], c[1][dst] = c[0][src], c[1][src]
    s = gk.pair_exact(*q, *c)
    s32 = s.astype(np.float32)
    assert np.array_equal(s32.astype(np.float64), s)
    return q, c, s32


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
    """Per row: empty; the edge columns 0, 63, 64, 127, 128, N-1; a whole half; a whole tile; a whole split range; every column;
    a random subset."""
    rows = []
    edges = [c for c in (0, 63, 64, 127, 128, nc - 1) if 0 <= c < nc]
    for r in range(nq):
        kind = r % 7
        if kind == 0:
            cols = []
        elif kind == 1:
            cols = edges
        elif kind == 2:
            cols = range(64, min(128, nc))
        elif kind == 3:
            cols = range(128, min(256, nc))
        elif kind == 4:
            t0, t1 = ro.split_tiles(nc, splits, r % splits)
            cols = range(t0 * ro.BLOCK_N, min(t1 * ro.BLOCK_N, nc))
        elif kind == 5:
            cols = range(nc)
        else:
            cols = rng.choice(nc, rng.integers(0, nc // 2 + 1), replace=False)
        rows.append(list(cols))
    return rows


# ---------------------------------------------------------------------------------------------------------------------------
# register top-k: dae_similarity_topk_bf16x3 / _excl_ / _groups_
# ---------------------------------------------------------------------------------------------------------------------------
def _topk(mode, Q, C, nq, nc, dim, k, splits, exclude=False, diag=0, lists=None, groups=None):
    """One call; returns (idx, val, ws_val [nq, 2s, k], ws_idx) after checking every guard."""
    s = ro.topk_splits(nq, nc, splits, _sms())
    ws_bytes = _query('dae_similarity_topk_workspace', nq, nc, k, splits)
    assert ws_bytes == ro.topk_workspace_bytes(nq, k, s)
    n = nq * 2 * s * k
    init = np.concatenate([np.full(n, INF_BITS, np.int32), np.full(n, nc - 1, np.int32)])
    ws = Guarded(2 * n, np.int32, SENT_I, init)
    idx = Guarded(nq * k, np.int32, SENT_I)
    val = Guarded(nq * k, np.float32, SENT_V)
    args = [nq, nc, dim, *Q.args, *C.args, k, diag, 1 if exclude else 0, splits, ws.ptr, ws_bytes, idx.ptr, val.ptr]
    if mode == 'plain':
        assert lists is None and groups is None
        _call('dae_similarity_topk_bf16x3', *args, _st())
    else:
        L = lists if lists is not None else Lists([], nq)
        if mode == 'excl':
            _call('dae_similarity_topk_excl_bf16x3', *args, *L.args, _st())
        else:
            ex = L.args if lists is not None else (None, None, 0)
            g = _dev(np.asarray(groups, np.int32))
            _call('dae_similarity_topk_groups_bf16x3', *args, *ex, g.data_ptr(), _st())
    torch.cuda.synchronize()
    w = ws.get()
    return (idx.get().reshape(nq, k), val.get().reshape(nq, k), w[:n].view(np.float32).reshape(nq, 2 * s, k),
            w[n:].reshape(nq, 2 * s, k), s)


def _check_topk(name, mode, S, k, got, allowed, groups, rows=None):
    idx, val, wv, wi, s = got
    if mode == 'groups':
        want = ro.top_k_groups(S, k, allowed, groups)
    else:
        want = ro.top_k(S, k, allowed)
    _eq(name + ' idx', idx, want[0])
    _same(name + ' val', val, want[1])
    rows = np.arange(S.shape[0]) if rows is None else rows
    pv, pi = ro.partial_lists(S[rows], k, s, None if allowed is None else allowed[rows], groups if mode == 'groups' else None)
    _eq(name + ' partial idx', wi[rows], pi)
    _same(name + ' partial val', wv[rows], pv)


# (nq, nc, dim): 1, 63/64/65 and 127/128/129 rows on both sides, n_corpus below k, every dim of the issue
TOPK_SHAPES = [(1, 1, 1), (1, 20, 8), (63, 129, 63), (64, 128, 64), (65, 127, 65), (127, 65, 500), (128, 64, 8),
               (129, 63, 1), (129, 1000, 65), (65, 1300, 500)]
TOPK_SPLITS = [1, 2, 7, 32, 0]
TOPK_K = [1, 15, 16, 17, 31, 32]


@pytest.mark.parametrize('k', TOPK_K)
@pytest.mark.parametrize('mode', ['plain', 'excl', 'groups'])
def test_register_topk_exact(mode, k):
    for t, (nq, nc, dim) in enumerate(TOPK_SHAPES):
        rng = np.random.default_rng(1000 * k + t)
        q, c, S = _exact(nq, nc, dim, seed=t + 17 * k, dup=nc // 3)
        Q, C = Operand(*q), Operand(*c)
        for splits in (TOPK_SPLITS[t % 5], TOPK_SPLITS[(t + 2) % 5]):
            s = ro.topk_splits(nq, nc, splits, _sms())
            diag = [0, -5, 7, nc + 3, -nq][(t + splits) % 5]
            exclude = (t + k) % 3 != 0
            rows = _edge_lists(nq, nc, s, rng) if mode != 'plain' and t % 2 == 0 else None
            groups = rng.integers(0, max(1, nc // 3), nc) if mode == 'groups' else None
            got = _topk(mode, Q, C, nq, nc, dim, k, splits, exclude, diag, None if rows is None else Lists(rows, nq), groups)
            allowed = ro.allowed_mask(nq, nc, exclude, diag, rows)
            _check_topk('%s k=%d %s splits=%d' % (mode, k, (nq, nc, dim), splits), mode, S, k, got, allowed, groups)


@pytest.mark.parametrize('k', [16, 32])
def test_groups_identity_and_single_group(k):
    nq, nc, dim = 129, 700, 8
    q, c, S = _exact(nq, nc, dim, seed=k, dup=300)
    Q, C = Operand(*q), Operand(*c)
    rows = _edge_lists(nq, nc, 3, np.random.default_rng(k))
    L = Lists(rows, nq)
    allowed = ro.allowed_mask(nq, nc, True, 0, rows)
    ex = _topk('excl', Q, C, nq, nc, dim, k, 3, True, 0, L)
    gi = _topk('groups', Q, C, nq, nc, dim, k, 3, True, 0, L, np.arange(nc))
    for a, b in zip(ex[:4], gi[:4]):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))
    _check_topk('excl', 'excl', S, k, ex, allowed, None)
    one = np.zeros(nc, np.int64)
    got = _topk('groups', Q, C, nq, nc, dim, k, 3, True, 0, L, one)
    _check_topk('one group', 'groups', S, k, got, allowed, one)
    assert (got[0][:, 1:] == -1).all()
    # members of a group straddling halves, tiles and splits: column c and c + 64, c + 128, c + 300 share a label
    straddle = np.arange(nc) % 64
    got = _topk('groups', Q, C, nq, nc, dim, k, 3, False, 0, None, straddle)
    _check_topk('straddling groups', 'groups', S, k, got, None, straddle)


@pytest.mark.parametrize('k', [16, 32])
def test_long_exclusion_lists_cross_many_tiles(k):
    nq, nc, dim = 3, 20000, 8
    q, c, S = _exact(nq, nc, dim, seed=5, dup=5000)
    Q, C = Operand(*q), Operand(*c)
    rng = np.random.default_rng(k)
    rows = [np.sort(rng.choice(nc, 5000, replace=False)), np.arange(0, nc, 4), np.arange(3000, 8000)]
    for splits in (7, 32):
        for mode in ('excl', 'groups'):
            groups = rng.integers(0, 3000, nc) if mode == 'groups' else None
            got = _topk(mode, Q, C, nq, nc, dim, k, splits, False, 0, Lists(rows, nq), groups)
            _check_topk('%s splits=%d' % (mode, splits), mode, S, k, got, ro.allowed_mask(nq, nc, lists=rows), groups)


@pytest.mark.parametrize('k', [10, 32])
@pytest.mark.parametrize('mode', ['plain', 'excl', 'groups'])
def test_register_topk_past_three_grid_passes(mode, k):
    splits = ro.TOPK_MAX_SPLITS
    tiles_m = 3 * _sms() // splits + 1
    nq, nc, dim = tiles_m * ro.BLOCK_M - 5, splits * ro.BLOCK_N + 5, 8
    assert ro.work_items(nq, ro.topk_splits(nq, nc, splits, _sms())) > 3 * _sms()
    q, c, S = _exact(nq, nc, dim, seed=k, dup=1000)
    Q, C = Operand(*q), Operand(*c)
    rng = np.random.default_rng(k)
    rows = lists = groups = None
    if mode != 'plain':
        rows = [np.sort(rng.choice(nc, rng.integers(0, 300), replace=False)) for _ in range(nq)]
        lists = Lists(rows, nq)
    if mode == 'groups':
        groups = rng.integers(0, nc // 2, nc)
    got = _topk(mode, Q, C, nq, nc, dim, k, splits, True, 0, lists, groups)
    allowed = ro.allowed_mask(nq, nc, True, 0, rows)
    sample = None
    if mode == 'groups':   # the streamed-list model is a Python loop: every row of the first and last blocks, and a sample
        sample = np.unique(np.concatenate([np.arange(ro.BLOCK_M), np.arange(nq - ro.BLOCK_M, nq), rng.integers(0, nq, 64)]))
    _check_topk('%s k=%d' % (mode, k), mode, S, k, got, allowed, groups, sample)


# ---------------------------------------------------------------------------------------------------------------------------
# thresholded pairs: dae_similarity_pairs_bf16x3 (pairs_kernel<false>)
# ---------------------------------------------------------------------------------------------------------------------------
def _pairs(Q, C, nq, nc, dim, self_mode, tau, capacity, count0=0):
    n_out = max(capacity, 1)
    i_out, j_out = Guarded(n_out, np.int32, SENT_I), Guarded(n_out, np.int32, SENT_I)
    s_out = Guarded(n_out, np.float32, SENT_V)
    cnt = Guarded(1, np.uint64, np.uint64(0x5A5A5A5A5A5A5A5A), np.uint64(count0))
    _call('dae_similarity_pairs_bf16x3', nq, nc, dim, *Q.args, *C.args, 1 if self_mode else 0, float(tau), cnt.ptr, capacity,
          i_out.ptr if capacity else None, j_out.ptr if capacity else None, s_out.ptr if capacity else None, _st())
    torch.cuda.synchronize()
    return int(cnt.get()[0]) - count0, i_out.get(), j_out.get(), s_out.get()


def _check_triples(name, got, want, written):
    """The first `written` slots hold exactly the triples of `want` (any order, when written is all of them) or a subset."""
    i, j, s = got
    key = i[:written].astype(np.int64) * (1 << 32) + j[:written]
    assert np.unique(key).size == written, '%s: a pair listed twice' % name
    wk = want[0].astype(np.int64) * (1 << 32) + want[1]
    pos = np.searchsorted(wk, key)
    assert (pos < wk.size).all() and np.array_equal(wk[np.minimum(pos, wk.size - 1)], key), '%s: a pair outside the set' % name
    _same(name + ' scores', s[:written], want[2][pos])
    if written == wk.size:
        assert np.array_equal(np.sort(key), wk)


@pytest.mark.parametrize('self_mode', [True, False])
@pytest.mark.parametrize('shape', [(1, 1, 1), (2, 2, 8), (65, 127, 63), (129, 129, 500), (300, 1000, 65)])
def test_pairs_exact(self_mode, shape):
    nq, nc, dim = shape
    if self_mode:
        nc = nq
    q, c, S = _exact(nq, nc, dim, seed=nq + dim, dup=nc // 4, self_mode=self_mode)
    Q = Operand(*q)
    C = Q if self_mode else Operand(*c)
    vals = np.sort(S[np.tril_indices(nq, -1)] if self_mode else S.ravel())
    taus = [-1.0, float(vals[0]) if vals.size else 0.0, float(vals[vals.size // 2]) if vals.size else 0.0, -ro.FLT_MAX]
    for tau in taus:   # each tau equal to a score: s == tau qualifies; and a negative tau
        want = ro.pairs_set(S, tau, self_mode)
        n = want[0].size
        for cap, c0 in ((n + 5, 3), (n, 0), (max(n - 1, 0), 0), (0, 0)):
            got_n, i, j, s = _pairs(Q, C, nq, nc, dim, self_mode, tau, cap, c0)
            assert got_n == n, (tau, cap, got_n, n)
            first, end = min(c0, cap), min(c0 + n, cap)
            if cap:
                # slots below the counter's start and at or past its end stay untouched
                assert (i[:first] == SENT_I).all() and (i[end:] == SENT_I).all() and (s[end:].view(np.uint32) == SENT_V.view(np.uint32)).all()
                _check_triples('pairs tau=%r cap=%d' % (tau, cap), (i[first:end], j[first:end], s[first:end]), want, end - first)


def test_pairs_past_three_grid_passes():
    tm = 1
    while tm * (tm + 1) // 2 <= 3 * _sms():
        tm += 1
    n = tm * ro.BLOCK_M - 3
    q, _, S = _exact(n, n, 8, seed=3, self_mode=True)
    Q = Operand(*q)
    tau = float(np.quantile(S, 0.999))
    want = ro.pairs_set(S, tau, True)
    got_n, i, j, s = _pairs(Q, Q, n, n, 8, True, tau, want[0].size + 10)
    assert got_n == want[0].size
    _check_triples('self', (i[:got_n], j[:got_n], s[:got_n]), want, got_n)
    nq = 3 * _sms() // tm + 1
    nq = nq * ro.BLOCK_M
    q2, c2, S2 = _exact(nq, n, 8, seed=4)
    want = ro.pairs_set(S2, tau, False)
    got_n, i, j, s = _pairs(Operand(*q2), Operand(*c2), nq, n, 8, False, tau, want[0].size + 10)
    assert got_n == want[0].size
    _check_triples('corpus', (i[:got_n], j[:got_n], s[:got_n]), want, got_n)


# ---------------------------------------------------------------------------------------------------------------------------
# long lists: bound -> collect -> pairs sort -> select
# ---------------------------------------------------------------------------------------------------------------------------
def _bound(Q, C, nq, nc, dim, k, splits, exclude, diag, lists, groups):
    s = ro.topk_bound_splits(nq, nc, k, splits, _sms())
    ws_bytes = _query('dae_similarity_topk_bound_workspace', nq, nc, k, splits)
    assert ws_bytes == ro.topk_workspace_bytes(nq, ro.TOPK_MAX_K, s)
    n = nq * 2 * s * ro.TOPK_MAX_K
    ws = Guarded(2 * n, np.int32, SENT_I, np.concatenate([np.full(n, INF_BITS, np.int32), np.full(n, nc - 1, np.int32)]))
    tau = Guarded(nq, np.float32, SENT_V)
    ex = lists.args if lists is not None else (None, None, 0)
    g = None if groups is None else _dev(np.asarray(groups, np.int32))
    _call('dae_similarity_topk_bound_bf16x3', nq, nc, dim, *Q.args, *C.args, k, diag, 1 if exclude else 0, splits, ws.ptr, ws_bytes,
          *ex, None if g is None else g.data_ptr(), tau.ptr, _st())
    torch.cuda.synchronize()
    w = ws.get()
    return tau.get(), w[:n].view(np.float32).reshape(nq, 2 * s, 32), w[n:].reshape(nq, 2 * s, 32), s


def _collect(Q, C, nq, nc, dim, tau, exclude, diag, lists, capacity, count0=0, rc0=None):
    cap = max(capacity, 1)
    i_out, j_out, s_out = Guarded(cap, np.int32, SENT_I), Guarded(cap, np.int32, SENT_I), Guarded(cap, np.float32, SENT_V)
    cnt = Guarded(1, np.uint64, np.uint64(0x5A5A5A5A5A5A5A5A), np.uint64(count0))
    rc0 = np.zeros(nq, np.uint32) if rc0 is None else rc0
    rc = Guarded(nq, np.uint32, np.uint32(0xDEADBEEF), rc0)
    t = _dev(np.asarray(tau, np.float32))
    ex = lists.args if lists is not None else (None, None, 0)
    _call('dae_similarity_topk_collect_bf16x3', nq, nc, dim, *Q.args, *C.args, diag, 1 if exclude else 0, t.data_ptr(), *ex, cnt.ptr,
          rc.ptr, capacity, i_out.ptr, j_out.ptr, s_out.ptr, _st())
    torch.cuda.synchronize()
    return int(cnt.get()[0]) - count0, rc.get().astype(np.int64) - rc0, i_out.get(), j_out.get(), s_out.get()


def _sort(i, j, s, nc, key_bits=None):
    """dae_pairs_sort of (i, j, s) -> (pi, pj, ps) read back from the buffers `which` names, and which."""
    n = len(i)
    keys = np.asarray(i, np.uint64) * np.uint64(nc) + np.asarray(j, np.uint64)
    if key_bits is None:
        key_bits = max(1, int(keys.max()).bit_length()) if n else 1
    k0, k1 = _dev(keys.view(np.int64)), torch.full((max(n, 1),), -1, dtype=torch.int64, device=DEV)
    s0, s1 = _dev(np.asarray(s, np.float32)), torch.full((max(n, 1),), float('nan'), dtype=torch.float32, device=DEV)
    if n == 0:
        k0, s0 = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.float32, device=DEV)
    wsb = _query('dae_pairs_sort_workspace', n, key_bits)
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
    which = (ctypes.c_int32 * 1)(-1)
    _call('dae_pairs_sort', n, nc, key_bits, k0.data_ptr(), k1.data_ptr(), s0.data_ptr(), s1.data_ptr(), ws.data_ptr(), ws.numel(),
          ctypes.addressof(which), _st())
    torch.cuda.synchronize()
    w = which[0]
    assert w in (0, 1)
    ks, ss, free = (k0, s0, k1) if w == 0 else (k1, s1, k0)
    ij = free.cpu().numpy().view(np.int32)
    return ks.cpu().numpy()[:n].view(np.uint64), ss.cpu().numpy()[:n], ij[:n], ij[n:2 * n], w


def _select(pi, pj, ps, nq, k, groups=None):
    n = len(pi)
    idx, val = Guarded(nq * k, np.int32, SENT_I), Guarded(nq * k, np.float32, SENT_V)
    d = [_dev(np.asarray(a)) for a in (pi, pj, np.asarray(ps, np.float32))] if n else [None] * 3
    g = None if groups is None else _dev(np.asarray(groups, np.int32))
    _call('dae_similarity_topk_select', nq, n, *[None if a is None else a.data_ptr() for a in d], k,
          None if g is None else g.data_ptr(), idx.ptr, val.ptr, _st())
    torch.cuda.synchronize()
    return idx.get().reshape(nq, k), val.get().reshape(nq, k)


@pytest.mark.parametrize('k', [33, 256, 257, 1024])
@pytest.mark.parametrize('mode', ['plain', 'lists', 'groups'])
def test_long_lists_stage_by_stage(mode, k):
    nq, nc, dim = 65, 4200, 8
    q, c, S = _exact(nq, nc, dim, seed=k, dup=1500)
    Q, C = Operand(*q), Operand(*c)
    rng = np.random.default_rng(k)
    rows = lists = groups = None
    if mode != 'plain':
        rows = _edge_lists(nq, nc, 7, rng)
        lists = Lists(rows, nq)
    if mode == 'groups':
        groups = rng.integers(0, 2000, nc)
    exclude, diag = True, 11
    allowed = ro.allowed_mask(nq, nc, exclude, diag, rows)
    for splits in (1, 7):
        tau, wv, wi, s = _bound(Q, C, nq, nc, dim, k, splits, exclude, diag, lists, groups)
        pv, pi = ro.partial_lists(S, 32, s, allowed, groups, km=32)
        _eq('bound partial idx', wi, pi)
        _same('bound partial val', wv, pv)
        _same('tau', tau, ro.bound_tau(pv, pi, k, groups))
    want = ro.collect_set(S, tau, allowed)
    n = want[0].size
    rc0 = rng.integers(1, 1000, nq).astype(np.uint32)
    got_n, rc, i, j, sc = _collect(Q, C, nq, nc, dim, tau, exclude, diag, lists, n + 14, 9, rc0)
    assert got_n == n
    _eq('row_count', rc, np.bincount(want[0], minlength=nq))
    _check_triples('collect', (i[9:9 + n], j[9:9 + n], sc[9:9 + n]), want, n)
    _, ps, pi_, pj_, _ = _sort(i[9:9 + n], j[9:9 + n], sc[9:9 + n], nc)
    _eq('sorted i', pi_, want[0])
    _eq('sorted j', pj_, want[1])
    _same('sorted s', ps, want[2])
    idx, val = _select(pi_, pj_, ps, nq, k, groups)
    ref = ro.top_k_groups(S, k, allowed, groups) if groups is not None else ro.top_k(S, k, allowed)
    _eq('select idx', idx, ref[0])
    _same('select val', val, ref[1])


def test_bound_with_fewer_than_k_entries_and_collect_taus():
    nq, nc, dim = 130, 300, 8
    q, c, S = _exact(nq, nc, dim, seed=9, dup=100)
    Q, C = Operand(*q), Operand(*c)
    tau, wv, wi, s = _bound(Q, C, nq, nc, dim, 1024, 0, False, 0, None, None)
    assert s == ro.topk_bound_splits(nq, nc, 1024, 0, _sms()) and 2 * s * 32 < 1024
    assert (tau == np.float32(-ro.FLT_MAX)).all()
    pv, pi = ro.partial_lists(S, 32, s, km=32)
    _eq('partial idx', wi, pi)
    # an uploaded tau with -inf, NaN, -FLT_MAX, a score of the row (s == tau qualifies) and +FLT_MAX
    specials = [-np.inf, np.nan, -ro.FLT_MAX, ro.FLT_MAX]
    t = np.array([specials[r % 4] if r % 5 else S[r, r % nc] for r in range(nq)], np.float32)
    want = ro.collect_set(S, t)
    n = want[0].size
    got_n, rc, i, j, sc = _collect(Q, C, nq, nc, dim, t, False, 0, None, n)
    assert got_n == n
    _eq('row_count', rc, np.bincount(want[0], minlength=nq))
    _check_triples('collect', (i, j, sc), want, n)
    # capacity below the count: the count stays exact, nothing is written past capacity
    got_n, rc, i, j, sc = _collect(Q, C, nq, nc, dim, t, False, 0, None, n // 2)
    assert got_n == n
    _check_triples('collect capped', (i, j, sc), want, n // 2)


def test_collect_past_three_grid_passes():
    t = 1
    while t * t <= 3 * _sms():
        t += 1
    nq, nc = t * ro.BLOCK_M - 1, t * ro.BLOCK_M + 1
    q, c, S = _exact(nq, nc, 8, seed=12)
    tau = np.quantile(S, 0.995, axis=1).astype(np.float32)
    want = ro.collect_set(S, tau)
    n = want[0].size
    got_n, rc, i, j, sc = _collect(Operand(*q), Operand(*c), nq, nc, 8, tau, True, 0, None, n)
    want = ro.collect_set(S, tau, ro.allowed_mask(nq, nc, True, 0))
    assert got_n == want[0].size
    _eq('row_count', rc, np.bincount(want[0], minlength=nq))
    _check_triples('collect', (i[:got_n], j[:got_n], sc[:got_n]), want, got_n)


@pytest.mark.parametrize('n,nc,key_bits', [(0, 7, 1), (1, 7, 3), (5000, 1000, 20), (5000, 999, 23), (3_000_000, 100_003, 31)])
def test_pairs_sort(n, nc, key_bits):
    rng = np.random.default_rng(n)
    top = (1 << key_bits) - 1
    keys = np.unique(rng.integers(0, top + 1, int(n * 1.1) + 2, dtype=np.int64))
    rng.shuffle(keys)
    keys = keys[:n]
    if n:
        keys[0] = top   # the largest key the bits allow
    s = rng.standard_normal(n).astype(np.float32)
    ks, ss, pi, pj, _ = _sort(keys // nc, keys % nc, s, nc, key_bits)
    order = np.argsort(keys, kind='stable')
    _eq('keys', ks, keys[order].astype(np.uint64))
    _same('payload', ss, s[order])
    _eq('i', pi, (keys[order] // nc).astype(np.int32))
    _eq('j', pj, (keys[order] % nc).astype(np.int32))


def test_pairs_sort_reports_both_buffers():
    seen = set()
    n = 20000   # above the sort's single-tile size
    keys = np.arange(n, dtype=np.int64)[::-1].copy()
    for bits in range(15, 65, 3):
        ks, _, _, _, w = _sort(keys // 17, keys % 17, np.zeros(n, np.float32), 17, bits)
        _eq('keys bits=%d' % bits, ks, np.arange(n, dtype=np.uint64))
        seen.add(w)
    assert seen == {0, 1}


def _synthetic_pairs(nq, rng, L):
    """Sorted (i, j, s): the first and last rows empty, a row of > 2L candidates, all-equal scores, -0.0 before +0.0 at lower
    indices, and a group repeated across chunks (labels of j // 3 and j % 7 below)."""
    rows = []
    for r in range(nq):
        if r in (0, nq - 1) or r % 4 == 1:
            continue
        kind = r % 4
        if kind == 0:
            n = 2 * L + 300 + r
            j = np.sort(rng.choice(50_000, n, replace=False))
            s = rng.integers(-30, 30, n).astype(np.float32)
        elif kind == 2:
            j = np.arange(0, 3000, 2)
            s = np.full(j.size, 1.5, np.float32)
        else:
            j = np.arange(0, 2000, 1)
            s = np.where(j % 2 == 0, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
            s[j % 11 == 0] = 1.0
        rows.append((np.full(j.size, r, np.int32), j.astype(np.int32), s))
    return [np.concatenate([x[t] for x in rows]) for t in range(3)]


@pytest.mark.parametrize('k', [33, 256, 257, 1024])
def test_select_on_synthetic_rows(k):
    nq = 12
    rng = np.random.default_rng(k)
    pi, pj, ps = _synthetic_pairs(nq, rng, ro.rank_chunk(k))
    idx, val = _select(pi, pj, ps, nq, k)
    want = ro.select(pi, pj, ps, nq, k)
    _eq('idx', idx, want[0])
    _eq('val bits', val.view(np.uint32), want[1].view(np.uint32))   # stored bits: -0.0 stays -0.0
    for groups in (np.arange(50_000) // 3, np.arange(50_000) % 7):
        idx, val = _select(pi, pj, ps, nq, k, groups)
        want = ro.select(pi, pj, ps, nq, k, groups)
        _eq('groups idx', idx, want[0])
        _eq('groups val bits', val.view(np.uint32), want[1].view(np.uint32))
    idx, val = _select(pi[:0], pj[:0], ps[:0], nq, k)
    assert (idx == -1).all() and np.isneginf(val).all()


# ---------------------------------------------------------------------------------------------------------------------------
# pair histogram: dae_similarity_pair_hist_bf16x3
# ---------------------------------------------------------------------------------------------------------------------------
def _hist(X, n, dim, labels, M, bins, h0, s0):
    hist = Guarded(2 * bins, np.uint64, np.uint64(0xA5A5A5A5A5A5A5A5), h0)
    sums = Guarded(2, np.float64, np.float64(-1234.5), s0)
    lab = _dev(np.asarray(labels, np.int32))
    _call('dae_similarity_pair_hist_bf16x3', n, dim, *X.args, lab.data_ptr(), float(M), bins, hist.ptr, sums.ptr, _st())
    torch.cuda.synchronize()
    return hist.get().astype(np.int64).reshape(2, bins) - h0.astype(np.int64).reshape(2, bins), sums.get() - s0


def _edge_data(n, dim, seed):
    """Exact operands whose scores hit +-M = +-2^11 exactly (rows 0 / 1 / 2), exceed it, and fall on bin edges."""
    q, _, _ = _exact(n, n, dim, seed, self_mode=True)
    hi, lo = q[0].copy(), q[1].copy()
    e = gk.bf16_rn(np.array([32.0, -32.0, 0.0], np.float32))
    for r, sign in ((0, 0), (1, 0), (2, 1)):
        if r < n:
            hi[r] = e[2]
            lo[r] = e[2]
            hi[r, :min(2, dim)] = e[sign]
    s = gk.pair_exact(hi, lo, hi, lo)
    return (hi, lo), s.astype(np.float32)


@pytest.mark.parametrize('n', [2, 127, 128, 129])
@pytest.mark.parametrize('bins', [1 << 10, 1 << 24])
def test_pair_hist_exact(n, bins):
    dim = 8
    q, S = _edge_data(n, dim, seed=n)
    X = Operand(*q)
    M = 2.0 ** 11
    if n >= 3:
        assert S[1, 0] == M and S[2, 0] == -M
    rng = np.random.default_rng(n)
    for labels in (np.full(n, -1), np.zeros(n, np.int64), rng.integers(-1, 9, n), np.arange(n) % 2):
        h0 = rng.integers(0, 1 << 40, 2 * bins).astype(np.uint64)
        s0 = np.array([1.5, -2.25])
        hist, sums = _hist(X, n, dim, labels, M, bins, h0, s0)
        want_h, want_s, _, _ = host_histograms(S, labels, M, bins)
        _eq('hist', hist, want_h)
        _eq('sums', sums, want_s)   # exact scores: the fp64 sums are exact in any order


def test_pair_hist_past_three_grid_passes_and_nan_rows():
    tm = 1
    while tm * (tm + 1) // 2 <= 3 * _sms():
        tm += 1
    n, dim, bins, M = tm * ro.BLOCK_M - 7, 63, 1 << 12, 2.0 ** 14
    q, _, S = _exact(n, n, dim, seed=21, self_mode=True)
    labels = np.random.default_rng(0).integers(-1, 40, n)
    hist, sums = _hist(Operand(*q), n, dim, labels, M, bins, np.ones(2 * bins, np.uint64), np.zeros(2))
    want_h, want_s, _, _ = host_histograms(S, labels, M, bins)
    _eq('hist', hist, want_h)
    _eq('sums', sums, want_s)
    # a row holding NaN: each of its pairs goes to bin 0 and turns its group's fp64 sum into NaN
    hi, lo = q[0][:300].copy(), q[1][:300].copy()
    hi[37, 5] = gk.BF16_NAN
    lab = np.where(np.arange(300) < 150, 1, 2)
    lab[37] = 1
    S = gk.pair_exact(hi, lo, hi, lo).astype(np.float32)
    hist, sums = _hist(Operand(hi, lo), 300, dim, lab, M, bins, np.zeros(2 * bins, np.uint64), np.zeros(2))
    want_h, _, _, _ = host_histograms(S, lab, M, bins)
    _eq('hist with a NaN row', hist, want_h)
    assert hist[0, 0] >= 149 and hist[1, 0] >= 150   # 37 + 112 related, 150 unrelated NaN scores in bin 0
    assert np.isnan(sums).all()


# ---------------------------------------------------------------------------------------------------------------------------
# zero and NaN query rows
# ---------------------------------------------------------------------------------------------------------------------------
def test_zero_and_nan_query_rows():
    nq, nc, dim = 70, 500, 65
    q, c, _ = _exact(nq, nc, dim, seed=31, dup=100)
    hi, lo = q[0].copy(), q[1].copy()
    hi[[3, 64]] = 0
    lo[[3, 64]] = 0
    hi[[3]] |= np.uint16(0x8000)       # -0.0 entries: products and sums of signed zeros
    hi[[5, 69], 7] = gk.BF16_NAN
    S = gk.pair_exact(hi, lo, *c).astype(np.float32)
    assert np.isnan(S[5]).all() and (S[3] == 0).all()
    Q, C = Operand(hi, lo), Operand(*c)
    for mode in ('plain', 'excl', 'groups'):
        for k in (16, 32):
            groups = np.arange(nc) // 2 if mode == 'groups' else None
            got = _topk(mode, Q, C, nq, nc, dim, k, 2, False, 0, None, groups)
            _check_topk('%s k=%d' % (mode, k), mode, S, k, got, None, groups)
            assert (got[0][[5, 69]] == -1).all() and (got[0][3] == np.arange(k) * (2 if mode == 'groups' else 1)).all()
    tau, _, _, _ = _bound(Q, C, nq, nc, dim, 100, 0, False, 0, None, None)
    assert tau[5] == np.float32(-ro.FLT_MAX) and tau[69] == np.float32(-ro.FLT_MAX)
    n_all = int(np.sum(~np.isnan(S)))
    got_n, rc, i, j, sc = _collect(Q, C, nq, nc, dim, np.full(nq, -np.inf, np.float32), False, 0, None, n_all)
    assert got_n == n_all and rc[5] == 0 and rc[69] == 0 and rc[3] == nc
    assert not np.isin(i, [5, 69]).any()
    got_n, i, j, s = _pairs(Q, C, nq, nc, dim, False, -ro.FLT_MAX, n_all)
    assert got_n == n_all and not np.isin(i[:got_n], [5, 69]).any()
    _, ps, pi_, pj_, _ = _sort(*ro.collect_set(S, np.full(nq, -np.inf, np.float32)), nc)
    idx, val = _select(pi_, pj_, ps, nq, 100)
    assert (idx[[5, 69]] == -1).all() and (idx[3] == np.arange(100)).all()


# ---------------------------------------------------------------------------------------------------------------------------
# ordinary random data: the same bits from every export, within the fp64 bound
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H', [37, 500])
def test_cross_export_bits_on_random_data(H):
    n, k = 400, 32
    x = gk.scaled_operand(np.random.default_rng(H), n, H, row_spread=20, col_spread=0)
    hi, lo = bf16_split(x)
    X = Operand(hi, lo)
    ref, bound = gk.pair_bound(hi, lo, hi, lo, H)
    # every score of the lower triangle, from the pairs export (self mode, threshold -FLT_MAX)
    npairs = n * (n - 1) // 2
    got_n, pi, pj, ps = _pairs(X, X, n, n, H, True, -ro.FLT_MAX, npairs)
    assert got_n == npairs
    S = np.full((n, n), np.nan, np.float32)
    S[pi, pj] = ps
    low = np.tril_indices(n, -1)
    ratio = np.abs(S[low] - ref[low]) / bound[low]
    worst = {'pairs': float(ratio.max())}
    # top-k (query rows as the first operand, as the pairs export): every (i, j) with j < i has the pairs' bits
    idx, val, _, _, _ = _topk('plain', X, X, n, n, H, k, 0, True, 0)
    m = (idx >= 0) & (idx < np.arange(n)[:, None])
    rr = np.nonzero(m)[0]
    _eq('topk vs pairs bits', val[m].view(np.uint32), S[rr, idx[m]].view(np.uint32))
    jj = np.where(idx >= 0, idx, 0)
    worst['topk'] = float(np.max(np.where(idx >= 0, np.abs(val - ref[np.arange(n)[:, None], jj]) / bound[np.arange(n)[:, None], jj], 0)))
    assert ro.membership(ref, bound, idx, k, ro.allowed_mask(n, n, True, 0)) == []
    # collect with tau = -FLT_MAX lists every off-diagonal score: the lower triangle again has the pairs' bits
    got_n, rc, ci, cj, cs = _collect(X, X, n, n, H, np.full(n, -ro.FLT_MAX, np.float32), True, 0, None, n * (n - 1))
    assert got_n == n * (n - 1)
    C = np.full((n, n), np.nan, np.float32)
    C[ci, cj] = cs
    _eq('collect vs pairs bits', C[low].view(np.uint32), S[low].view(np.uint32))
    _eq('topk vs collect bits', val[idx >= 0].view(np.uint32), C[np.nonzero(idx >= 0)[0], idx[idx >= 0]].view(np.uint32))
    worst['collect'] = float(np.nanmax(np.abs(C - ref) / bound))
    # the histogram bins those same bits
    M = 2.0 ** int(np.ceil(np.log2(np.abs(ref).max() * 1.01)))
    labels = np.random.default_rng(1).integers(-1, 5, n)
    hist, sums = _hist(X, n, H, labels, M, 1 << 16, np.zeros(1 << 17, np.uint64), np.zeros(2))
    full = np.where(np.isnan(S), 0, S)
    want_h, want_s, rel, unrel = host_histograms(full + full.T, labels, M, 1 << 16)
    _eq('hist', hist, want_h)
    # fp64 sums in atomic order: not bit for bit, within n 2^-53 of the sum of magnitudes
    mag = np.array([np.abs(rel.astype(np.float64)).sum(), np.abs(unrel.astype(np.float64)).sum()])
    assert (np.abs(sums - want_s) <= npairs * 2.0 ** -52 * mag).all(), (sums, want_s)
    print('\nworst |err| / bound, H = %d: %s' % (H, worst))
    assert max(worst.values()) <= 1.0


# ---------------------------------------------------------------------------------------------------------------------------
# which kernels ran
# ---------------------------------------------------------------------------------------------------------------------------
INSTANTIATIONS = ['topk_kernel<16,false,false>', 'topk_kernel<32,false,false>', 'topk_kernel<16,true,false>',
                  'topk_kernel<32,true,false>', 'topk_kernel<16,true,true>', 'topk_kernel<32,true,true>', 'topk_merge_kernel',
                  'topk_merge_groups_kernel', 'pairs_kernel<false>', 'pairs_kernel<true>', 'pair_hist_kernel',
                  'topk_bound_kernel<false>', 'topk_bound_kernel<true>', 'topk_select_kernel<false>', 'topk_select_kernel<true>',
                  'pairs_decode_kernel']


def _profile_exports():
    """Each export call in its own profiler session (_call with _PROFILED set); returns [(export, kernel names, expected)]."""
    global _PROFILED
    nq, nc, dim = 130, 300, 8
    q, c, S = _exact(nq, nc, dim, seed=1)
    Q, C = Operand(*q), Operand(*c)
    g = np.arange(nc) // 3
    L = Lists([[1, 2]], nq)
    _PROFILED = []
    expect = []
    for k in (16, 32):
        _topk('plain', Q, C, nq, nc, dim, k, 0)
        _topk('excl', Q, C, nq, nc, dim, k, 0, lists=L)
        _topk('groups', Q, C, nq, nc, dim, k, 0, groups=g)
        expect += [['topk_kernel<%d,false,false>' % k, 'topk_merge_kernel'], ['topk_kernel<%d,true,false>' % k, 'topk_merge_kernel'],
                   ['topk_kernel<%d,true,true>' % k, 'topk_merge_groups_kernel']]
    _pairs(Q, C, nq, nc, dim, False, 0.0, 10)
    expect.append(['pairs_kernel<false>'])
    tau, _, _, _ = _bound(Q, C, nq, nc, dim, 40, 0, False, 0, None, None)
    _bound(Q, C, nq, nc, dim, 40, 0, False, 0, L, g)
    expect += [['topk_kernel<32,false,false>', 'topk_bound_kernel<false>'], ['topk_kernel<32,true,true>', 'topk_bound_kernel<true>']]
    want = ro.collect_set(S, tau)
    assert want[0].size > 0
    _collect(Q, C, nq, nc, dim, tau, False, 0, None, want[0].size)
    expect.append(['pairs_kernel<true>'])
    _, ps, pi, pj, _ = _sort(*want, nc)
    expect.append(['pairs_decode_kernel'])
    _select(pi, pj, ps, nq, 40)
    _select(pi, pj, ps, nq, 40, g)
    expect += [['topk_select_kernel<false>'], ['topk_select_kernel<true>']]
    _hist(Q, nq, dim, np.zeros(nq), 2.0 ** 14, 1024, np.zeros(2048, np.uint64), np.zeros(2))
    expect.append(['pair_hist_kernel'])
    record, _PROFILED = _PROFILED, None
    assert len(record) == len(expect), [r[0] for r in record]
    return [(export, sorted(names), want_k) for (export, names), want_k in zip(record, expect)]


def test_profiler_sees_every_instantiation():
    """The profiler runs in a process of its own: CUPTI's activity state is per process, and the profiler sessions of earlier
    tests in a long pytest process can leave later sessions without kernel records."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ('import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_ranking_kernels as t; '
            'print("RESULT " + json.dumps(t._profile_exports()))' % (here, os.path.dirname(here)))
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=600, cwd=os.path.dirname(here))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    record = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith('RESULT ')][-1][7:])
    bad = []
    for export, names, want_k in record:
        missing = [w for w in want_k if not any(w in n for n in names)]
        if missing:
            bad.append((export, missing, [n[:90] for n in names]))
    assert not bad, bad
    assert {w for _, _, want_k in record for w in want_k} == set(INSTANTIATIONS)
