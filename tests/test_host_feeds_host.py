"""HostFeed, the one packed host buffer of a training step, without a GPU: its byte layout against a NumPy unpacker, the corrupted
values of a non-canonical batch, and the feed checks of TrainEngine.run_feed / run_feeds that come before any device work.
Pinning needs CUDA, so torch.Tensor.pin_memory returns the tensor itself here."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from helpers import random_csr


@pytest.fixture(autouse=True)
def _no_pinning(monkeypatch):
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self, *a, **k: self)


def _feed(*a, **k):
    from dae_rnn_news_recommendation_b200.engine import HostFeed
    return HostFeed(*a, **k)


def unpack(f):
    """(indptr, indices, values, values_c, labels) rebuilt from the bytes of f.host and the layout HostFeed documents:
    [indptr int64[B+1] | indices int32[nnz] | values f32[nnz] | corrupted values f32[nnz] | labels f32[B]], each part 16-byte aligned."""
    hb = f.host.numpy()
    B = f.B
    indptr = hb[0:8 * (B + 1)].view(np.int64)
    n = int(indptr[-1])
    part = lambda off, cnt, dt: hb[off:off + 4 * cnt].view(dt)
    return (indptr, part(f.off_indices, n, np.int32), part(f.off_values, n, np.float32), part(f.off_values_c, n, np.float32),
            part(f.off_labels, B, np.float32))


def _dense(indptr, indices, values, shape):
    return sp.csr_matrix((values, indices, indptr), shape=shape).toarray()


@pytest.mark.parametrize('B,nnz_row,cap_extra,labelled', [(64, 12, 0, True), (63, 5, 37, True), (7, 3, 1, False), (1, 1, 0, True),
                                                          (5, 0, 3, True)])
def test_layout_offsets_alignment_and_contents(B, nnz_row, cap_extra, labelled):
    x = random_csr(B, 300, nnz_row, kind='tfidf', seed=B)
    if nnz_row == 0:
        x = sp.csr_matrix((B, 300), dtype=np.float32)
    xc = (x.data * (np.arange(x.nnz) % 3 != 0)).astype(np.float32)
    lab = np.arange(B, dtype=np.float32) % 4 if labelled else None
    cap = x.nnz + cap_extra
    f = _feed(x, xc, lab, cap_nnz=cap)
    al = lambda n: (n + 15) // 16 * 16
    assert (f.B, f.nnz, f.F, f.cap_nnz, f.has_labels) == (B, cap, 300, cap, labelled)
    assert f.off_indptr == 0
    assert f.off_indices == al(8 * (B + 1))
    assert f.off_values == f.off_indices + al(4 * cap)
    assert f.off_values_c == f.off_values + al(4 * cap)
    assert f.off_labels == f.off_values_c + al(4 * cap)
    assert f.nbytes == f.off_labels + al(4 * B) == f.host.numel()
    assert all(o % 16 == 0 for o in (f.off_indices, f.off_values, f.off_values_c, f.off_labels, f.nbytes))
    assert f.host.dtype == torch.uint8
    indptr, indices, values, values_c, labels = unpack(f)
    assert np.array_equal(indptr, x.indptr) and np.array_equal(indices, x.indices)
    assert np.array_equal(values, x.data.astype(np.float32)) and np.array_equal(values_c, xc)
    assert np.array_equal(labels, lab if labelled else np.zeros(B, np.float32))
    # without a cap the layout is sized by the batch itself
    g = _feed(x, xc, lab)
    assert g.cap_nnz is None and g.nnz == x.nnz and g.nbytes == al(8 * (B + 1)) + 3 * al(4 * x.nnz) + al(4 * B)
    assert all(np.array_equal(u, v) for u, v in zip(unpack(g), unpack(f)))


def test_clean_values_stand_in_for_absent_corruption():
    x = random_csr(16, 100, 6, kind='tfidf', seed=3)
    _, _, values, values_c, _ = unpack(_feed(x, None, None, cap_nnz=x.nnz + 5))
    assert np.array_equal(values_c, values) and np.array_equal(values, x.data.astype(np.float32))


def test_cap_below_the_batch_is_refused():
    x = random_csr(8, 100, 6, seed=4)
    with pytest.raises(AssertionError):
        _feed(x, None, None, cap_nnz=x.nnz - 1)


def test_corrupted_values_follow_their_columns_in_an_unsorted_batch():
    """A row stored with columns [5, 2] and corrupted values [50, 20]: the feed holds columns [2, 5], so its corrupted values must be
    [20, 50] (column 2 trains on 20)."""
    x = sp.csr_matrix((np.array([1.0, 2.0], np.float32), np.array([5, 2]), np.array([0, 2])), shape=(1, 8))
    assert not x.has_sorted_indices
    indptr, indices, values, values_c, _ = unpack(_feed(x, np.array([50.0, 20.0]), None, cap_nnz=4))
    assert indices.tolist() == [2, 5] and values.tolist() == [2.0, 1.0] and values_c.tolist() == [20.0, 50.0]


def test_corrupted_values_of_shuffled_rows_land_on_the_callers_columns():
    rng = np.random.default_rng(7)
    x = random_csr(40, 500, 15, kind='tfidf', seed=8)
    perm = np.concatenate([x.indptr[r] + rng.permutation(x.indptr[r + 1] - x.indptr[r]) for r in range(40)]).astype(np.int64)
    xs = sp.csr_matrix((x.data[perm], x.indices[perm], x.indptr), shape=x.shape)      # the same matrix, entries shuffled in each row
    xs.has_sorted_indices = False
    xc = rng.random(xs.nnz).astype(np.float32) + 1.0                                    # distinct corrupted values
    want = _dense(xs.indptr, xs.indices, xc, xs.shape)
    indptr, indices, values, values_c, _ = unpack(_feed(xs, xc, None, cap_nnz=xs.nnz + 9))
    assert np.array_equal(indices, x.indices)
    assert np.array_equal(_dense(indptr, indices, values_c, x.shape), want)
    assert np.array_equal(_dense(indptr, indices, values, x.shape), x.toarray())


def test_duplicate_entries_sum_their_corrupted_values_as_their_values():
    """A duplicate (row, column) entry is summed into one; its corrupted values are summed the same way."""
    x = sp.csr_matrix((np.array([1, 2, 4, 8], np.float32), np.array([3, 3, 1, 0]), np.array([0, 3, 4])), shape=(2, 6))
    indptr, indices, values, values_c, _ = unpack(_feed(x, np.array([10, 0, 40, 80]), None, cap_nnz=6))
    assert indptr.tolist() == [0, 2, 3] and indices.tolist() == [1, 3, 0]
    assert values.tolist() == [4.0, 3.0, 8.0] and values_c.tolist() == [40.0, 10.0, 80.0]


def test_other_input_formats_keep_their_entry_order():
    rng = np.random.default_rng(9)
    x = random_csr(12, 60, 8, kind='tfidf', seed=10)
    dense = x.toarray()
    xc = rng.random(x.nnz).astype(np.float32) + 1.0
    want = _dense(x.indptr, x.indices, xc, x.shape)
    # ndarray: one value per nonzero in row-major order (that is the canonical CSR order)
    assert np.array_equal(unpack(_feed(dense, xc, None))[3], xc)
    # COO with its entries reversed, and CSC: values follow the matrix's own storage order
    coo = x.tocoo()
    rev = sp.coo_matrix((coo.data[::-1], (coo.row[::-1], coo.col[::-1])), shape=x.shape)
    ip, ix, _, vc, _ = unpack(_feed(rev, xc[::-1], None))
    assert np.array_equal(_dense(ip, ix, vc, x.shape), want)
    csc = x.tocsc()
    vc_csc = sp.csc_matrix((sp.csr_matrix((xc, x.indices, x.indptr), shape=x.shape)).tocsc())
    assert np.array_equal(vc_csc.indices, csc.indices) and np.array_equal(vc_csc.indptr, csc.indptr)
    ip, ix, _, vc, _ = unpack(_feed(csc, vc_csc.data, None))
    assert np.array_equal(_dense(ip, ix, vc, x.shape), want)


def test_corrupted_values_of_the_wrong_length_are_refused():
    x = random_csr(6, 40, 5, seed=11)
    for xs in (x, x.tocoo()):
        with pytest.raises(ValueError, match='x_corr_values'):
            _feed(xs, np.ones(x.nnz + 1, np.float32), None)


# ---- TrainEngine's feed checks: they run before any device work --------------------------------------------------------------------
def _bare_engine(strategy):
    """A TrainEngine without a device: only the attributes its feed checks read."""
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200.engine import TrainEngine
    eng = TrainEngine.__new__(TrainEngine)
    eng.strategy = _cabi.STRATEGY[strategy]
    return eng


@pytest.mark.parametrize('rows', [4, 5, 3001])
def test_stacked_explicit_feed_of_a_row_count_not_a_multiple_of_three_is_refused(rows):
    x = random_csr(rows, 50, 4, seed=rows)
    eng = _bare_engine('explicit')
    capped = _feed(x, None, None, cap_nnz=x.nnz + 2)
    for f in (_feed(x, None, None), capped):
        with pytest.raises(ValueError, match='multiple of 3'):
            eng.run_feed(f)
    with pytest.raises(ValueError, match='multiple of 3'):
        eng.run_feeds([capped, capped])


@pytest.mark.parametrize('strategy', ['batch_all', 'batch_hard'])
def test_triplet_strategies_refuse_feeds_without_labels(strategy):
    x = random_csr(16, 50, 4, seed=2)
    eng = _bare_engine(strategy)
    f = _feed(x, None, None, cap_nnz=x.nnz)
    with pytest.raises(ValueError, match='labels'):
        eng.run_feed(f)
    with pytest.raises(ValueError, match='labels'):
        eng.run_feeds([f, f])


def test_run_feeds_refuses_mixed_layouts():
    eng = _bare_engine('batch_all')
    x, y = random_csr(16, 50, 4, seed=3), random_csr(16, 50, 4, seed=4)
    lab = np.zeros(16, np.float32)
    cap = max(x.nnz, y.nnz)
    a = _feed(x, None, lab, cap_nnz=cap)
    mixed = [
        [a, _feed(y, None, lab, cap_nnz=cap + 1)],                   # another cap_nnz
        [a, _feed(y, None, None, cap_nnz=cap)],                      # labels absent
        [a, _feed(y, None, lab)],                                    # no common layout at all
        [_feed(x, None, lab), _feed(x, None, lab)],                  # feeds without a cap
        [a, _feed(random_csr(17, 50, 4, seed=5)[:15], None, np.zeros(15, np.float32), cap_nnz=cap)],   # another batch size
        [a, _feed(sp.csr_matrix(y.toarray()[:, :49]), None, lab, cap_nnz=cap)],                   # another feature count
    ]
    for feeds in mixed:
        with pytest.raises(AssertionError, match='one common layout'):
            eng.run_feeds(feeds)
    assert eng.run_feeds([]) == []
