"""Host-side parts of the top-k recommendation: argument checks of the C entry points (before any CUDA call), the label precision
metric and the CLI flag."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FAKE = 1 << 20   # 16-byte aligned non-null stand-in for a device pointer: every call below fails validation before using it


def _topk(k=10, ldq=64, ldc=64, dim=64, ws_bytes=1 << 30, splits=1):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_similarity_topk_bf16x3', 300, 500, dim, FAKE, FAKE, ldq, FAKE, FAKE, ldc, k, 0, 1, splits, FAKE, ws_bytes,
               FAKE, FAKE, None)


@pytest.mark.parametrize('k', [0, 33, -1])
def test_k_outside_the_limit_is_rejected(k):
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
        _topk(k=k)
    out = (ctypes.c_int64 * 1)()
    with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
        _cabi.call('dae_similarity_topk_workspace', 300, 500, k, 1, ctypes.addressof(out))


@pytest.mark.parametrize('ldq,ldc,dim', [(36, 64, 37), (64, 60, 37), (68, 64, 64), (64, 72, 70)])
def test_bad_leading_dimensions_are_rejected(ldq, ldc, dim):
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='leading dimensions'):
        _topk(ldq=ldq, ldc=ldc, dim=dim)


def test_short_workspace_is_rejected():
    from dae_rnn_news_recommendation_b200 import _cabi
    out = (ctypes.c_int64 * 1)()
    _cabi.call('dae_similarity_topk_workspace', 300, 500, 10, 2, ctypes.addressof(out))
    assert out[0] == 300 * 2 * 2 * 10 * 8          # 2 splits x 2 column halves -> 4 lists of 10 (score, index) pairs per row
    with pytest.raises(_cabi.DaeError, match='workspace'):
        _topk(k=10, splits=2, ws_bytes=out[0] - 1)


def test_top_k_similar_rejects_k_before_touching_the_device():
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
        top_k_similar(np.zeros((4, 3), np.float32), k=33)


def test_label_precision_at_k_by_hand():
    from dae_rnn_news_recommendation_b200.helpers import label_precision_at_k
    corpus_labels = np.array([0, 0, 1, 1, -1, 2])
    index = np.array([[1, 2, 4],       # query label 0: corpus 1 matches, 2 and 4 do not            -> 1/3
                      [3, 2, -1],      # label 1: both returned neighbours match, padding skipped   -> 2/2
                      [0, 1, 5],       # label -1: query skipped
                      [-1, -1, -1],    # label 2, no neighbour at all: skipped
                      [5, 0, -1]])     # label 2: 5 matches, 0 does not                             -> 1/2
    query_labels = np.array([0, 1, -1, 2, 2])
    assert label_precision_at_k(index, query_labels, corpus_labels) == pytest.approx((1 / 3 + 1 + 1 / 2) / 3)
    assert np.isnan(label_precision_at_k(index[2:4], query_labels[2:4], corpus_labels))


def test_top_k_flag():
    import main_autoencoder as cli
    assert cli.build_parser().parse_args([]).top_k == 0
    F = cli.check_flags(cli.build_parser().parse_args(['--top_k', '5']))
    assert F.top_k == 5
    with pytest.raises(AssertionError):
        cli.check_flags(cli.build_parser().parse_args(['--top_k', '33']))
