"""Host half of the ranking kernels' references (tests/ranking_kernel_oracle.py): the partial-list model merges to the contract,
the exact operands sum exactly in any order, the restated split choice agrees with the library's workspace queries, and the
select oracle agrees with a brute-force sort on hand-made rows."""
import numpy as np
import pytest

import gemm_kernel_oracle as gk
import ranking_kernel_oracle as ro
from topk_groups_oracle import brute_force_grouped


def _query(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    return _cabi.query(name, *args)


def _exact_scores(rng, nq, nc, dim, dup=0):
    q = gk.exact_operands(rng, nq, dim)
    c = gk.exact_operands(rng, nc, dim)
    if dup:   # duplicated corpus rows: equal scores at different indices
        src = rng.integers(0, nc, dup)
        dst = rng.integers(0, nc, dup)
        c[0][dst], c[1][dst] = c[0][src], c[1][src]
    return np.asarray(gk.pair_exact(*q, *c), np.float32)


@pytest.mark.parametrize('k', [1, 15, 16, 17, 32])
@pytest.mark.parametrize('splits', [1, 2, 7])
@pytest.mark.parametrize('mode', ['plain', 'lists', 'groups', 'lists_groups'])
def test_partial_lists_merge_to_the_contract(k, splits, mode):
    rng = np.random.default_rng(k * 31 + splits)
    nq, nc = 9, 1000
    s = _exact_scores(rng, nq, nc, 3, dup=300)
    allowed = None
    if 'lists' in mode:
        allowed = ro.allowed_mask(nq, nc, exclude=True, diag_offset=5,
                                  lists=[np.sort(rng.choice(nc, rng.integers(0, 400), replace=False)) for _ in range(nq)])
        allowed[0] = False                       # a row without candidates
    groups = rng.integers(0, 120, nc) if 'groups' in mode else None
    val, idx = ro.partial_lists(s, k, splits, allowed, groups)
    got = ro.merge_lists(val, idx, k, groups)
    if groups is None:
        want = ro.top_k(s, k, allowed)
    else:
        want = ro.top_k_groups(s, k, allowed, groups)
        assert np.array_equal(want[0], brute_force_grouped(s, groups, k, allowed)[0])
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
    # the lists are those of the split ranges: an entry of list 2 sp + h lies in that half of that split's tiles
    for sp in range(splits):
        for h in range(2):
            cols = set(ro.half_columns(nc, splits, sp, h).tolist())
            assert set(idx[:, 2 * sp + h].ravel().tolist()) - {-1} <= cols


def test_identity_groups_are_the_plain_lists():
    rng = np.random.default_rng(3)
    s = _exact_scores(rng, 5, 700, 2, dup=200)
    for k in (1, 16, 32):
        a = ro.partial_lists(s, k, 3)
        b = ro.partial_lists(s, k, 3, groups=np.arange(700))
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[0], b[0])


@pytest.mark.parametrize('dim', [1, 8, 63, 500])
def test_exact_operands_sum_exactly_in_any_order(dim):
    rng = np.random.default_rng(dim)
    (ah, al), (bh, bl) = gk.exact_operands(rng, 40, dim), gk.exact_operands(rng, 1, dim)
    a_hi, a_lo, b_hi, b_lo = (gk.bf16_value(x) for x in (ah, al, bh, bl))
    terms = a_hi * b_hi + a_hi * b_lo + a_lo * b_hi          # per-k fp64 terms, each a multiple of 2^-4
    assert np.array_equal(terms.astype(np.float32).astype(np.float64), terms)
    want = gk.pair_exact(ah, al, bh, bl)[:, 0]
    for got in gk.fl32_sum_orders(terms):
        assert np.array_equal(got.astype(np.float64), want)
    # the three products summed separately (the kernel's per-k16-step order) agree as well
    assert np.array_equal(gk.emulate_bf16x3(ah, al, bh, bl)[:, 0].astype(np.float64), want)
    assert np.max(np.abs(want)) < 2 ** 15


SHAPES = [(1, 1), (1, 129), (65, 1000), (129, 4096), (1000, 50000), (300, 200000)]


@pytest.mark.parametrize('nq,nc', SHAPES)
def test_restated_splits_agree_with_the_workspace_queries(nq, nc):
    for k in (1, 16, 17, 32):
        for splits in list(range(1, 40)) + [64, 1000]:
            want = ro.topk_workspace_bytes(nq, k, ro.topk_splits(nq, nc, splits))
            assert _query('dae_similarity_topk_workspace', nq, nc, k, splits) == want, (nq, nc, k, splits)
    for k in (1, 32, 33, 256, 257, 1000, 1024):
        for splits in list(range(1, 40)) + [1000]:
            want = ro.topk_workspace_bytes(nq, ro.TOPK_MAX_K, ro.topk_bound_splits(nq, nc, k, splits))
            assert _query('dae_similarity_topk_bound_workspace', nq, nc, k, splits) == want, (nq, nc, k, splits)


def test_rank_chunk_and_splits_by_hand():
    assert [ro.rank_chunk(k) for k in (1, 33, 256, 257, 512, 513, 1024)] == [256, 256, 256, 512, 512, 1024, 1024]
    assert ro.topk_splits(100, 100, 7) == 1                 # one column tile
    assert ro.topk_splits(100, 10000, 0, sms=132) == 19     # 79 tiles // 4
    assert ro.topk_splits(100, 100000, 0, sms=132) == 32
    assert ro.topk_bound_splits(100, 100000, 1024, 1) == 32
    assert ro.topk_bound_splits(100, 1000, 1024, 1) == 8     # capped by the 8 column tiles
    assert [ro.split_tiles(1000, 3, s) for s in range(3)] == [(0, 2), (2, 5), (5, 8)]
    assert ro.half_columns(200, 1, 0, 1).tolist() == list(range(64, 128)) + list(range(192, 200))


def _hand_pairs():
    """(pi, pj, ps) sorted by (i, j) over 6 rows: rows 1 and 3 empty, row 0 with +-0.0 ties, row 2 longer than 2L = 512, row 5
    the last, all-equal scores in row 4."""
    rows = []
    rows += [(0, 3, 0.0), (0, 5, -0.0), (0, 7, 1.0), (0, 9, -0.0), (0, 11, 0.0), (0, 12, -1.0)]
    rng = np.random.default_rng(0)
    for j in range(1500):
        rows.append((2, j, float(rng.integers(-20, 20))))
    rows += [(4, j, 2.5) for j in range(0, 40, 3)]
    rows += [(5, 0, -3.0), (5, 99, 7.0)]
    pi = np.array([r[0] for r in rows], np.int32)
    pj = np.array([r[1] for r in rows], np.int32)
    ps = np.array([r[2] for r in rows], np.float32)
    return pi, pj, ps


@pytest.mark.parametrize('k', [1, 3, 5, 33, 600, 1024])
def test_select_oracle_against_brute_force(k):
    pi, pj, ps = _hand_pairs()
    got = ro.select(pi, pj, ps, 6, k)
    want = ro.select_brute(pi, pj, ps, 6, k)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
    assert (got[0][1] == -1).all() and (got[0][3] == -1).all()


def test_select_keeps_the_stored_zero_bits():
    pi, pj, ps = _hand_pairs()
    idx, val = ro.select(pi, pj, ps, 6, 6)
    assert idx[0].tolist() == [7, 3, 5, 9, 11, 12]
    assert val[0].view(np.uint32).tolist() == np.array([1.0, 0.0, -0.0, -0.0, 0.0, -1.0], np.float32).view(np.uint32).tolist()
    t_idx, t_val = ro.top_k(np.array([[0.0, -0.0, -0.0, 0.0, -np.inf, np.nan]], np.float32), 6)
    assert t_idx[0].tolist() == [0, 1, 2, 3, -1, -1]
    assert t_val[0].view(np.uint32).tolist() == np.array([0.0, -0.0, -0.0, 0.0, -np.inf, -np.inf], np.float32).view(np.uint32).tolist()


def test_bound_and_collect_by_hand():
    val = np.array([[[5.0, 3.0, -np.inf], [4.0, 3.0, 2.0]]], np.float32)
    idx = np.array([[[1, 7, -1], [2, 8, 9]]], np.int32)
    assert ro.bound_tau(val, idx, 3)[0] == 3.0
    assert ro.bound_tau(val, idx, 5)[0] == 2.0
    assert ro.bound_tau(val, idx, 6)[0] == -ro.FLT_MAX
    groups = np.zeros(10, np.int64)
    groups[[2, 8]] = 1
    assert ro.bound_tau(val, idx, 2, groups)[0] == 4.0
    assert ro.bound_tau(val, idx, 3, groups)[0] == -ro.FLT_MAX
    s = np.array([[1.0, np.nan, -np.inf, 3.4e38], [0.0, -1.0, 2.0, np.nan]], np.float32)
    i, j, v = ro.collect_set(s, np.array([np.nan, 0.0], np.float32))
    assert list(zip(i.tolist(), j.tolist())) == [(0, 0), (0, 3), (1, 0), (1, 2)]
    i, j, v = ro.pairs_set(np.array([[1, 2], [2, 1]], np.float32), 1.0, True)
    assert list(zip(i.tolist(), j.tolist())) == [(1, 0)]


def test_membership_rule():
    ref = np.array([[4.0, 3.0, 2.99, 1.0]])
    bound = np.full_like(ref, 0.01)
    assert ro.membership(ref, bound, np.array([[0, 1]]), 2) == []
    assert ro.membership(ref, bound, np.array([[0, 2]]), 2) == []       # within the bounds of the k-th
    assert ro.membership(ref, bound, np.array([[1, 2]]), 2) != []       # 0 beats the k-th by far more than the bounds
    assert ro.membership(ref, bound, np.array([[0, 3]]), 2) != []


def test_nan_scores_go_to_bin_zero_on_the_host():
    from dae_rnn_news_recommendation_b200.helpers import score_bins
    assert score_bins(np.array([np.nan, -np.inf, np.inf, -1.0, 1.0], np.float32), 1.0, 1024).tolist() == [0, 0, 1023, 0, 1023]
