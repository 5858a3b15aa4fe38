"""Block mining without a GPU: the block oracles against the materialising fp64 oracle, the argument checks of the block-mining C
exports, and the host-side validation of mining_block_rows."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]


def _case(kind, B=200, H=6, seed=0):
    rng = np.random.default_rng(seed)
    E = rng.integers(-2, 3, (B, H)).astype(np.float64)      # small integers: exact dot products, many exact ties
    lab = rng.integers(0, 5, B).astype(np.float32)
    if kind == 'zero_row':
        E[17] = 0.0
    elif kind == 'singleton':
        lab[5] = 99.0
    elif kind == 'one_class':
        lab[:] = 2.0
    elif kind == 'real':
        E = rng.normal(0.0, 0.7, (B, H))
    return torch.from_numpy(lab), E


@pytest.mark.parametrize('kind', ['ties', 'zero_row', 'singleton', 'one_class', 'real'])
@pytest.mark.parametrize('block_rows', [7, 64, 200])
def test_batch_hard_block_oracle_matches_materialising(kind, block_rows):
    from oracle.dae_oracle import batch_hard_triplet_loss
    from block_oracle import batch_hard_triplet_loss_chunked
    lab, E0 = _case(kind, seed=len(kind))
    E1 = torch.tensor(E0, requires_grad=True)
    l1, w1, f1, n1 = batch_hard_triplet_loss(lab, E1)
    g1, = torch.autograd.grad(l1, E1)
    E2 = torch.tensor(E0, requires_grad=True)
    l2, w2, f2, n2, C = batch_hard_triplet_loss_chunked(lab, E2, block_rows)
    g2, = torch.autograd.grad(l2, E2)
    assert abs(float(l2.detach()) - float(l1.detach())) <= 1e-10 * max(1.0, abs(float(l1.detach())))
    assert torch.equal(w2, w1.to(w2.dtype))
    assert float(f2) == pytest.approx(float(f1), abs=1e-12) and float(n2) == float(n1)
    scale = max(1.0, float(g1.abs().max()))
    assert float((g2 - g1).abs().max()) <= 1e-10 * scale
    assert float((C - g1).abs().max()) <= 1e-10 * scale


@pytest.mark.parametrize('kind', ['ties', 'singleton', 'one_class', 'real'])
def test_batch_all_block_oracle_matches_materialising(kind):
    from oracle.dae_oracle import batch_all_triplet_loss
    from block_oracle import batch_all_triplet_loss_block
    lab, E0 = _case(kind, B=90, seed=3 + len(kind))
    E1 = torch.tensor(E0, requires_grad=True)
    l1, w1, f1, n1 = batch_all_triplet_loss(lab, E1)
    g1, = torch.autograd.grad(l1, E1)
    E2 = torch.tensor(E0, requires_grad=True)
    l2, w2, f2, n2, C = batch_all_triplet_loss_block(lab, E2, block_elems=5000)
    g2, = torch.autograd.grad(l2, E2)
    assert abs(float(l2.detach()) - float(l1.detach())) <= 1e-10 * max(1.0, abs(float(l1.detach())))
    assert torch.allclose(w2, w1.to(w2.dtype), rtol=0, atol=0)
    assert float(n2) == float(n1) and float(f2) == pytest.approx(float(f1), abs=1e-12)
    scale = max(1.0, float(g1.abs().max()))
    assert float((g2 - g1).abs().max()) <= 1e-10 * scale
    assert float((C - g1).abs().max()) <= 1e-10 * scale


def test_max_blocked_batch():
    from dae_rnn_news_recommendation_b200 import _cabi
    assert _cabi.MAX_BLOCKED_BATCH == 262144
    text = (ROOT / 'include' / 'dae_sm100.h').read_text()
    assert int(re.search(r'#define DAE_MAX_BLOCKED_BATCH (\d+)', text).group(1)) == _cabi.MAX_BLOCKED_BATCH


def _refused(name, *args, match=None):
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError) as e:
        _cabi.call(name, *args)
    assert name in str(e.value)
    if match:
        assert match in str(e.value), str(e.value)


P = 256   # a non-null stand-in pointer: every call below is refused by its argument checks, before any CUDA call


def test_blocked_exports_reject_out_of_range_arguments():
    big = 262145
    _refused('dae_batch_prepare_blocked', P, 0, None, big, P, 1, P, P, P, P, P, P, None, match='262144')
    _refused('dae_batch_prepare_next_blocked', P, big + 10, 0, P, big, P, 2, P, P, P, P, P, P, None, match='262144')
    B = 1000
    # dae_triplet_batch_all_rows(S_blk, lds, row0, n_rows, B, seg_lo, seg_hi, G_blk, ldg, stats, pos_only, g_hi, g_lo, ld_split, stream)
    _refused('dae_triplet_batch_all_rows', P, big, 0, 128, big, P, P, P, big, P, 0, P, P, big + 7, None, match='262144')
    _refused('dae_triplet_batch_all_rows', P, B, 896, 128, B, P, P, P, B, P, 0, P, P, 1008, None, match='outside')
    _refused('dae_triplet_batch_all_rows', P, B, -128, 128, B, P, P, P, B, P, 0, P, P, 1008, None)
    _refused('dae_triplet_batch_all_rows', P, B - 1, 0, 128, B, P, P, P, B, P, 0, P, P, 1008, None)
    _refused('dae_triplet_batch_all_rows', P, B, 0, 128, B, P, P, P, B - 1, P, 0, P, P, 1008, None)
    _refused('dae_triplet_batch_all_rows', P, B, 0, 128, B, P, P, P, B, P, 0, P, P, B - 1, None)
    # dae_triplet_batch_hard_rows(S_blk, lds, row0, n_rows, B, labels, G_blk, ldg, weight, stats, stream)
    _refused('dae_triplet_batch_hard_rows', P, big, 0, 128, big, P, P, big, P, P, None, match='262144')
    _refused('dae_triplet_batch_hard_rows', P, B, 900, 128, B, P, P, B, P, P, None, match='outside')
    _refused('dae_triplet_batch_hard_rows', P, B, 0, 0, B, P, P, B, P, P, None)
    _refused('dae_triplet_batch_hard_rows', P, B - 1, 0, 128, B, P, P, B, P, P, None)
    _refused('dae_triplet_batch_hard_rows', P, B, 0, 128, B, P, P, B - 1, P, P, None)
    # dae_triplet_batch_hard_finish(weight, B, stats, dE2, H, ld, stream)
    _refused('dae_triplet_batch_hard_finish', P, big, P, None, 0, 0, None)
    _refused('dae_triplet_batch_hard_finish', P, B, P, P, 16, 15, None)


@pytest.mark.parametrize('R', [0, 100, 64, 32768 + 128, 1000.5, -128, True])
def test_bad_mining_block_rows_raise_in_the_ctor(R):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder
    from dae_rnn_news_recommendation_b200.engine import TrainEngine
    with pytest.raises(ValueError):
        DenoisingAutoencoder(model_name='bad', main_dir='bad', mining_block_rows=R)
    with pytest.raises(ValueError):
        TrainEngine(100, 10, mining_block_rows=R)


@pytest.mark.parametrize('R', [None, 128, 4096, 32768])
def test_good_mining_block_rows_are_kept_and_not_written_to_the_parameter_file(R):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder
    m = DenoisingAutoencoder(model_name='ok', main_dir='ok', mining_block_rows=R)
    assert m.mining_block_rows == R
    m._write_parameter_to_file(False)
    assert 'mining_block_rows' not in Path(m.parameter_file).read_text()


def test_cli_flag():
    import main_autoencoder
    F = main_autoencoder.build_parser().parse_args(['--mining_block_rows', '4096'])
    assert F.mining_block_rows == 4096
    assert main_autoencoder.build_parser().parse_args([]).mining_block_rows == 0
