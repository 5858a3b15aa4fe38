"""Host-side parts of the grouped top-k (dae_similarity_topk_groups_bf16x3, dae_csr_similarity_topk_groups): the exports' argument
checks before any CUDA call, the helpers' ValueErrors before any device work, recommend's read-group lists by hand, the oracle
against brute force and against a model of the kernels' streaming lists and merge, and the --top_k_dedup flag."""
import ctypes
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from topk_groups_oracle import brute_force_grouped, grouped_top_k, streamed_grouped

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FAKE = 1 << 20   # 16-byte aligned non-null stand-in for a device pointer: every call below fails validation before using it


def _dense(k=10, dim=64, ldq=64, ldc=64, ws_bytes=1 << 30, ex_indptr=FAKE, ex_indices=FAKE, ex_nnz=5, groups=FAKE, nq=300):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_similarity_topk_groups_bf16x3', nq, 500, dim, FAKE, FAKE, ldq, FAKE, FAKE, ldc, k, 0, 1, 1, FAKE, ws_bytes, FAKE,
               FAKE, ex_indptr, ex_indices, ex_nnz, groups, None)


def _sparse(k=10, fq=64, fc=64, ws_bytes=1 << 30, ex_indptr=FAKE, ex_indices=FAKE, ex_nnz=5, groups=FAKE):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_csr_similarity_topk_groups', FAKE, FAKE, FAKE, 300, 100, fq, FAKE, FAKE, FAKE, 500, 100, fc, k, 0, 1, 1, FAKE,
               ws_bytes, FAKE, FAKE, ex_indptr, ex_indices, ex_nnz, groups, None)


@pytest.mark.parametrize('call', [_dense, _sparse])
def test_export_argument_checks(call):
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='null pointer'):
        call(groups=None)
    with pytest.raises(_cabi.DaeError, match='null pointer'):
        call(ex_indptr=None)                       # lists announced (ex_nnz = 5) without their structure
    with pytest.raises(_cabi.DaeError, match='null pointer'):
        call(ex_indices=None)
    with pytest.raises(_cabi.DaeError, match='bad sizes'):
        call(ex_nnz=-1)
    for k in (0, 33):
        with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
            call(k=k)
    with pytest.raises(_cabi.DaeError, match='aligned'):
        call(groups=FAKE + 2)
    with pytest.raises(_cabi.DaeError, match='aligned'):
        call(ex_indptr=FAKE + 4)
    with pytest.raises(_cabi.DaeError, match='workspace'):
        call(ws_bytes=16)


def test_dense_export_checks_sizes_and_leading_dimensions():
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='bad sizes'):
        _dense(nq=0)
    with pytest.raises(_cabi.DaeError, match='leading dimensions'):
        _dense(ldq=60, dim=60)


def test_sparse_export_checks_features():
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='features'):
        _sparse(fq=64, fc=65)


def test_workspace_is_the_plain_one():
    from dae_rnn_news_recommendation_b200 import _cabi
    out = (ctypes.c_int64 * 1)()
    _cabi.call('dae_similarity_topk_workspace', 300, 500, 10, 1, ctypes.addressof(out))
    with pytest.raises(_cabi.DaeError, match='workspace'):
        _dense(ws_bytes=out[0] - 1)
    _cabi.call('dae_csr_similarity_topk_workspace', 300, 500, 100, 64, 10, 1, ctypes.addressof(out))
    with pytest.raises(_cabi.DaeError, match='workspace'):
        _sparse(ws_bytes=out[0] - 1)


def _no_device(monkeypatch):
    """Any device work fails the test: the checks must come first."""
    def boom(*a, **k):
        raise AssertionError('touched the device')
    monkeypatch.setattr(torch.Tensor, 'to', boom)
    monkeypatch.setattr(torch.Tensor, 'cuda', boom)
    from dae_rnn_news_recommendation_b200 import _cabi
    monkeypatch.setattr(_cabi, 'call', boom)


BAD_GROUPS = [
    (np.zeros(5, np.int32), 'shape'),                       # wrong length
    (np.zeros((6, 1), np.int32), 'shape'),                  # not 1-D
    (np.zeros(6, np.float32), 'integers'),                  # not integer
    (np.zeros(6, bool), 'integers'),
    (np.array([0, 1, -1, 2, 3, 4]), 'outside'),             # negative
    (np.array([0, 1, 2, 3, 4, 1 << 31], np.int64), 'outside'),
]


@pytest.mark.parametrize('groups, match', BAD_GROUPS)
def test_top_k_similar_rejects_groups_before_the_device(monkeypatch, groups, match):
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    _no_device(monkeypatch)
    x = np.zeros((4, 3), np.float32)
    c = np.zeros((6, 3), np.float32)
    with pytest.raises(ValueError, match=match):
        top_k_similar(x, k=2, corpus=c, groups=groups)
    with pytest.raises(ValueError, match=match):
        top_k_similar(sp.csr_matrix(x), k=2, corpus=sp.csr_matrix(c), groups=groups,
                      exclude=sp.csr_matrix((4, 6)))
    with pytest.raises(ValueError, match='shape'):
        top_k_similar(c, k=2, groups=np.zeros(4, np.int32))    # self mode: one label per row


@pytest.mark.parametrize('groups, match', BAD_GROUPS)
def test_recommend_rejects_groups_before_the_device(monkeypatch, groups, match):
    from dae_rnn_news_recommendation_b200.helpers import recommend
    _no_device(monkeypatch)
    emb = np.zeros((6, 3), np.float32)
    h = sp.csr_matrix(np.eye(2, 6, dtype=np.float32))
    with pytest.raises(ValueError, match=match):
        recommend(h, emb, k=2, groups=groups)


def test_read_group_lists_by_hand():
    """Users' read groups expanded to every member, over all articles and over candidate positions."""
    from dae_rnn_news_recommendation_b200.helpers import _read_group_lists
    groups = torch.tensor([4, 4, 1, 7, 7, 1, 9], dtype=torch.int32)   # groups 4: {0, 1}, 1: {2, 5}, 7: {3, 4}, 9: {6}
    # user 0 read 0 and 3 (and 1, same group as 0), user 1 nothing, user 2 read 5, user 3 read 6
    indptr = torch.tensor([0, 3, 3, 4, 5])
    indices = torch.tensor([0, 1, 3, 5, 6], dtype=torch.int32)
    ptr, ind = _read_group_lists(indptr, indices, groups, groups)
    assert ptr.tolist() == [0, 4, 4, 6, 7]
    assert ind.dtype == torch.int32 and ind.tolist() == [0, 1, 3, 4, 2, 5, 6]
    cand = torch.tensor([1, 2, 4, 6])                                  # candidate positions 0..3 hold articles 1, 2, 4, 6
    ptr, ind = _read_group_lists(indptr, indices, groups, groups[cand])
    assert ptr.tolist() == [0, 2, 2, 3, 4]
    assert ind.tolist() == [0, 2, 1, 3]
    ptr, ind = _read_group_lists(torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32), groups, groups)
    assert ptr.tolist() == [0, 0, 0] and ind.numel() == 0


def test_read_group_lists_against_a_loop():
    from dae_rnn_news_recommendation_b200.helpers import _read_group_lists
    rng = np.random.default_rng(0)
    n, u = 400, 60
    groups = rng.integers(0, 90, n).astype(np.int32)
    h = sp.random(u, n, density=0.02, format='csr', random_state=1)
    h.sort_indices()
    cand = np.sort(rng.choice(n, 250, replace=False))
    ptr, ind = _read_group_lists(torch.from_numpy(h.indptr.astype(np.int64)), torch.from_numpy(h.indices.astype(np.int32)),
                                 torch.from_numpy(groups), torch.from_numpy(groups[cand]))
    ptr, ind = ptr.numpy(), ind.numpy()
    for r in range(u):
        read = set(groups[h.indices[h.indptr[r]:h.indptr[r + 1]]].tolist())
        want = [p for p in range(cand.size) if groups[cand[p]] in read]
        assert ind[ptr[r]:ptr[r + 1]].tolist() == want


def _case(seed, nq, nc, n_groups, levels):
    rng = np.random.default_rng(seed)
    s = rng.integers(0, levels, (nq, nc)).astype(np.float32)          # few levels: many ties, inside and across groups
    groups = rng.integers(0, n_groups, nc)
    allowed = rng.random((nq, nc)) > 0.2
    return s, groups, allowed


@pytest.mark.parametrize('k', [1, 3, 10, 17])
def test_oracle_against_brute_force(k):
    for seed, n_groups, levels in ((0, 40, 5), (1, 3, 100), (2, 1, 7), (3, 200, 1000)):
        s, groups, allowed = _case(seed, 12, 150, n_groups, levels)
        for a in (None, allowed):
            got = grouped_top_k(s, groups, k, a)
            want = brute_force_grouped(s, groups, k, a)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize('parts, kmax', [(1, 16), (3, 16), (7, 32), (64, 32)])
def test_streaming_lists_and_merge_give_the_oracle(parts, kmax):
    """The two facts of the design: each part's streaming list of representatives (only the first k slots count) and the merge
    that skips taken groups give the global answer, whatever the cut."""
    for seed, n_groups, levels in ((4, 30, 6), (5, 5, 50), (6, 1, 3), (7, 300, 1000)):
        s, groups, allowed = _case(seed, 10, 300, n_groups, levels)
        for k in (1, 4, min(kmax, 11)):
            for a in (None, allowed):
                got = streamed_grouped(s, groups, k, parts, kmax=kmax, allowed=a)
                want = grouped_top_k(s, groups, k, a)
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (seed, k)


def test_shifted_out_slots_cannot_block_a_group():
    """Slots k..KMAX-1 hold shifted-out entries, all <= thr < any value offered: matching the group there neither drops the
    candidate nor changes the first k entries (the shift merely stops at that slot), so the lists are the same either way."""
    for seed, n_groups, levels in ((9, 20, 8), (10, 4, 30), (11, 60, 5)):
        s, groups, allowed = _case(seed, 10, 300, n_groups, levels)
        for k in (2, 5, 11):
            want = streamed_grouped(s, groups, k, 3, kmax=16, allowed=allowed)
            got = streamed_grouped(s, groups, k, 3, kmax=16, allowed=allowed, all_slots=True)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_identity_groups_are_the_plain_top_k():
    s, _, allowed = _case(8, 9, 120, 1, 4)
    for k in (1, 6):
        got = grouped_top_k(s, np.arange(120), k, allowed)
        order = [np.lexsort((np.flatnonzero(allowed[r]), -s[r, allowed[r]]))[:k] for r in range(9)]
        for r in range(9):
            assert got[0][r].tolist() == np.flatnonzero(allowed[r])[order[r]].tolist()


def test_top_k_dedup_flag(tmp_path):
    import main_autoencoder as cli
    p = cli.build_parser()
    F = cli.check_flags(p.parse_args(['--top_k', '5', '--top_k_dedup', '0.9']))
    assert F.top_k_dedup == 0.9
    assert cli.check_flags(p.parse_args(['--top_k', '5'])).top_k_dedup == 0.0
    with pytest.raises(AssertionError, match='--top_k_dedup needs --top_k'):
        cli.check_flags(p.parse_args(['--top_k_dedup', '0.9']))
    with pytest.raises(AssertionError):
        cli.check_flags(p.parse_args(['--top_k', '5', '--top_k_dedup', '-0.5']))
