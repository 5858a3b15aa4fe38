"""Large triplet batches, host side: the chunked batch_all oracle against the materialising one (fp64), and the B cap of the C
exports, checked before any CUDA call (no GPU needed)."""
import numpy as np
import pytest
import torch

from oracle.chunked_oracle import batch_all_triplet_loss_chunked, _batch_hard_on
from oracle.dae_oracle import batch_all_triplet_loss, batch_hard_triplet_loss


def _labels(B, n_classes, seed):
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, n_classes, B).astype(np.float32)
    lab[rng.integers(0, B)] = 1000.0     # a singleton class
    return lab


@pytest.mark.parametrize('n_classes', [1, 2, 4, 37])
@pytest.mark.parametrize('pos_only', [False, True])
def test_chunked_oracle_equals_materialising_oracle(n_classes, pos_only):
    B, H = 120 if n_classes < 37 else 300, 7
    lab = torch.from_numpy(_labels(B, n_classes, seed=n_classes))
    E0 = torch.from_numpy(np.random.default_rng(3).normal(0.0, 1.5, (B, H)))
    E1 = E0.clone().requires_grad_(True)
    want = batch_all_triplet_loss(lab, E1, pos_triplets_only=pos_only)
    (gw,) = torch.autograd.grad(want[0], E1)
    E2 = E0.clone().requires_grad_(True)
    got = batch_all_triplet_loss_chunked(lab, E2, pos_triplets_only=pos_only, block_elems=5000)   # many blocks per class
    (gg,) = torch.autograd.grad(got[0], E2)
    assert float(got[0].detach()) == pytest.approx(float(want[0]), rel=1e-12, abs=1e-300)
    np.testing.assert_allclose(got[1].numpy(), want[1].numpy(), rtol=0, atol=0)
    assert got[2] == pytest.approx(float(want[2]), rel=1e-12, abs=0)
    assert got[3] == int(want[3])
    np.testing.assert_allclose(gg.numpy(), gw.numpy(), rtol=1e-10, atol=1e-13 * float(gw.abs().max() + 1))
    # G = d loss / d S: its symmetric part reproduces the gradient, and every row sums to zero
    S = E0 @ E0.t()
    Sl = S.clone().requires_grad_(True)
    d = -Sl[:, :, None] + Sl[:, None, :]
    from oracle.dae_oracle import triplet_mask
    valid = triplet_mask(lab).to(d.dtype)
    pos = ((valid * d) > 1e-16).to(d.dtype)
    mask, n = (pos, pos.sum()) if pos_only else (valid, valid.sum())
    (gs,) = torch.autograd.grad((torch.nn.functional.softplus(d) * mask).sum() / (n + 1e-16), Sl)
    np.testing.assert_allclose(got[4].numpy(), gs.numpy(), rtol=1e-10, atol=1e-15)
    assert float(got[4].sum(1).abs().max()) < 1e-12


def test_batch_hard_on_device_matches_oracle():
    B, H = 200, 9
    lab = torch.from_numpy(_labels(B, 5, seed=9))
    E = torch.from_numpy(np.random.default_rng(4).normal(0.0, 1.0, (B, H)))
    a, b = _batch_hard_on(lab, E), batch_hard_triplet_loss(lab, E)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(np.asarray(x), np.asarray(y))


def _ptrs(n):
    return [8 * (k + 1) for k in range(n)]     # non-null dummies: the argument checks fail before any CUDA call


def test_prepare_rejects_batches_above_the_cap():
    from dae_rnn_news_recommendation_b200 import _cabi
    assert _cabi.MAX_TRIPLET_BATCH == 32768
    B = _cabi.MAX_TRIPLET_BATCH + 1
    perm, labels, rows, labs, lo, hi, w, stats = _ptrs(8)
    for strategy in (1, 2):
        with pytest.raises(_cabi.DaeError) as e:
            _cabi.call('dae_batch_prepare', perm, 0, None, B, labels, strategy, rows, labs, lo, hi, w, stats, None)
        assert '32768' in str(e.value) and str(B) in str(e.value)
        with pytest.raises(_cabi.DaeError) as e:
            _cabi.call('dae_batch_prepare_next', perm, 10 ** 6, B, 8, B, labels, strategy, rows, labs, lo, hi, w, stats, None)
        assert '32768' in str(e.value)


def test_batch_all_rejects_batches_above_the_cap():
    from dae_rnn_news_recommendation_b200 import _cabi
    B = _cabi.MAX_TRIPLET_BATCH + 1
    S, lo, hi, G, stats = _ptrs(5)
    with pytest.raises(_cabi.DaeError) as e:
        _cabi.call('dae_triplet_batch_all', S, B, B, lo, hi, G, B, stats, 0, None, None, 0, None)
    assert '32768' in str(e.value) and str(B) in str(e.value)

