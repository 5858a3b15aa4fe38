"""CPU checks of tests/batch_prepare_oracle.py, the exact reference the batch preparation and masking-noise kernels are compared
with bit for bit (tests/test_gpu_batch_prepare.py): its class segments, data weights and N_valid equal the B^3 mask reductions of
oracle.dae_oracle, with NaN and +-0.0 labels classed as torch.eq (the reference's tf.equal) classes them; its Philox stream equals
a per-quad restatement; and dae_batch_prepare_explicit refuses blocks whose row ids overflow int32 before any device work."""
import numpy as np
import pytest
import torch

import batch_prepare_oracle as bo
from salt_pepper_oracle import philox4x32_10

SMALL = [1, 2, 3, 7, 31, 64]


def _same_class(lab):
    """B x B: rows i, j share a class by the oracle's segments (of the sorted batch)."""
    lo, hi = bo.segments(lab)
    j = np.arange(lab.shape[0])
    return (j[None, :] >= lo[:, None]) & (j[None, :] < hi[:, None])


@pytest.mark.parametrize('kind', bo.LABEL_KINDS)
@pytest.mark.parametrize('B', SMALL)
def test_segments_are_the_classes_of_torch_eq(kind, B):
    """Row i's segment holds exactly the rows whose label == its own under IEEE equality, plus i itself: -0.0 == +0.0, and a NaN
    row is alone.  The order puts every NaN after every other label and keeps each class contiguous."""
    perm = np.random.default_rng(B).permutation(B + 5).astype(np.int32)
    lab_b = bo.batch_labels(B, kind, seed=B)
    labels_all = bo.scatter_labels(B + 5, perm, 3, lab_b)
    rows, lab, lo, hi, w, st = bo.prepare(perm, 3, B, labels_all, bo.STRATEGY_BATCH_ALL)
    assert sorted(rows.tolist()) == sorted(perm[3:3 + B].tolist())
    assert np.array_equal(lab.view(np.uint32), labels_all[rows].view(np.uint32))        # the labels' own bits
    t = torch.from_numpy(lab)
    eq = (t[:, None] == t[None, :]).numpy() | np.eye(B, dtype=bool)
    assert np.array_equal(_same_class(lab), eq)
    nan = np.isnan(lab)
    assert not (nan[:-1] & ~nan[1:]).any()                                              # NaN rows last ...
    assert np.all(np.diff(rows[nan]) > 0)                                               # ... in row-id order
    fin = lab[~nan] + np.float32(0.0)
    assert np.all(fin[1:] >= fin[:-1])
    same = fin[:-1] == fin[1:]
    assert np.all(np.diff(rows[~nan])[same] > 0)                                        # ties by row id


@pytest.mark.parametrize('kind', bo.LABEL_KINDS)
@pytest.mark.parametrize('B', [3, 17, 40])
def test_closed_form_equals_the_b3_mask_reductions(kind, B):
    """Weights and N_valid against oracle.dae_oracle.batch_all_triplet_loss's three axis reductions of the B^3 valid-triplet mask
    (in the sorted batch); both are exact integers, so they are compared for equality."""
    from oracle.dae_oracle import batch_all_triplet_loss, triplet_mask
    perm = np.random.default_rng(B + 1).permutation(B).astype(np.int32)
    labels_all = bo.scatter_labels(B, perm, 0, bo.batch_labels(B, kind, seed=B + 2))
    rows, lab, lo, hi, w, st = bo.prepare(perm, 0, B, labels_all, bo.STRATEGY_BATCH_ALL)
    t = torch.from_numpy(lab)
    E = torch.randn(B, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(B))
    _, w_ref, _, _ = batch_all_triplet_loss(t, E)
    nv = float(triplet_mask(t).sum())
    assert np.array_equal(w.astype(np.float64), w_ref.numpy())
    assert st[bo.STAT_N_VALID] == nv and st[bo.STAT_SUM_W] == 3.0 * nv
    assert np.count_nonzero(st) == (2 if nv else 0)
    _, wh, _, _, wh_w, sth = bo.prepare(perm, 0, B, labels_all, bo.STRATEGY_BATCH_HARD)
    assert not wh_w.any() and not sth.any()


def test_weights_round_once_from_fp64():
    """At B = 262 144 in two classes the fp64 weights exceed 2^24: fp32 holds them rounded once."""
    B = 262144
    lab = np.zeros(B, np.float32)
    lab[:100003] = 1.0
    rows, l, lo, hi, w, st = bo.prepare(None, 0, B, lab, bo.STRATEGY_BATCH_ALL)
    w64, NV = bo.closed_form(lo, hi, B)
    assert w64.max() > 2 ** 24 and np.array_equal(w, w64.astype(np.float32))
    n = np.array([100003.0, B - 100003.0])
    assert NV == float(np.sum(n * (n - 1) * (B - n)))


def test_strategy_none_keeps_the_permutation():
    perm = np.array([5, 2, 9, 0, 7], np.int32)
    rows, lab, lo, hi, w, st = bo.prepare(perm, 1, 3, np.full(10, np.nan, np.float32), bo.STRATEGY_NONE)
    assert rows.tolist() == [2, 9, 0] and not lab.any() and not lo.any() and (hi == 3).all() and (w == 1).all()
    assert st[bo.STAT_SUM_W] == 3.0 and np.count_nonzero(st) == 1


@pytest.mark.parametrize('seed,epoch', [(0, 0), (7, 3), ((0x1234 << 32) | 0x9abc, (5 << 32) | 11)])
def test_mask_uniforms_equal_a_per_quad_loop(seed, epoch):
    nnz = 23
    u = bo.mask_uniforms(nnz, seed, epoch)
    for p in range(nnz):
        q = p // 4
        c = philox4x32_10((q & 0xFFFFFFFF, q >> 32, epoch & 0xFFFFFFFF, epoch >> 32), (seed & 0xFFFFFFFF, seed >> 32))
        assert u[p] == (int(c[p % 4]) >> 8) / 16777216.0
    assert u.dtype == np.float64 and (u < 1.0).all() and (u >= 0.0).all()


def test_mask_uniforms_quad_index_high_word():
    """The quad index's high word is the counter's second word: quad 2^32 + q differs from quad q."""
    q = (1 << 32) + 5
    c = philox4x32_10((q & 0xFFFFFFFF, q >> 32, 0, 0), (1, 0))
    d = philox4x32_10((5, 0, 0, 0), (1, 0))
    assert [int(x) for x in c] != [int(x) for x in d]


def test_mask_values_keeps_bits_and_compares_with_ge():
    vals = np.array([np.nan, -0.0, 1.5, -2.0, np.inf, 3.0, 4.0], np.float32)
    vals[0] = np.uint32(0xffc01234).view(np.float32)
    u = bo.mask_uniforms(vals.shape[0], 9, 2)
    frac = np.float32(u[3])                         # u is k * 2^-24: exact in fp32
    out = bo.mask_values(vals, None, frac, 9, 2)
    keep = u >= u[3]
    assert keep[3]
    assert np.array_equal(out.view(np.uint32), np.where(keep, vals, np.float32(0.0)).view(np.uint32))
    out = bo.mask_values(vals, np.array([0, 1, 255, 0, 1, 255, 0], np.uint8), 0.5)
    assert np.array_equal(out.view(np.uint32), np.array([0, vals[1].view(np.uint32), vals[2].view(np.uint32), 0,
                                                         vals[4].view(np.uint32), vals[5].view(np.uint32), 0], np.uint32))
    assert (bo.mask_values(vals, None, 0.0).view(np.uint32) == vals.view(np.uint32)).all()
    assert not bo.mask_values(vals, None, 1.0).view(np.uint32).any()


def test_batch_prepare_explicit_refuses_int32_overflow():
    """r + 2 n_each must fit in int32: n_each above (2^31 - 1) / 3 is refused before any device work (no pointer is used)."""
    from dae_rnn_news_recommendation_b200 import _cabi
    FAKE = 1 << 20
    lim = (2 ** 31 - 1) // 3
    for n_each in (lim + 1, 2 ** 40):
        with pytest.raises(_cabi.DaeError, match='dae_batch_prepare_explicit.*int32'):
            _cabi.call('dae_batch_prepare_explicit', None, 0, None, 4, n_each, FAKE, FAKE, None)
