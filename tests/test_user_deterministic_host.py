"""The user encoders' deterministic mode without a GPU (DESIGN 4.21): the keyword's checks, --user_deterministic's flag rules, the
new exports' argument checks, and the NumPy restatements of the fixed-order sums against exact sums."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import user_deterministic_oracle as do  # noqa: E402
from dae_rnn_news_recommendation_b200 import _cabi  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import UserAttention, UserGRU, UserLSTM  # noqa: E402

CELLS = (UserGRU, UserLSTM, UserAttention)


@pytest.mark.parametrize('cls', CELLS)
def test_deterministic_keyword(cls):
    assert cls(8, device='cpu').deterministic is False
    assert cls(8, device='cpu', deterministic=True).deterministic is True
    for bad in (1, 0, 'yes', None, np.bool_(True), 1.0):
        with pytest.raises(ValueError, match='deterministic'):
            cls(8, device='cuda:0', deterministic=bad)   # refused before any device work


@pytest.mark.parametrize('cls', CELLS)
def test_deterministic_is_not_saved(cls, tmp_path):
    m = cls(8, device='cpu', deterministic=True)
    m.save(tmp_path / 'm.npz')
    assert 'deterministic' not in np.load(tmp_path / 'm.npz').files
    assert cls.load(tmp_path / 'm.npz', device='cpu').deterministic is False


def test_user_deterministic_flag(tmp_path):
    import main_autoencoder as cli
    s = tmp_path / 's.npz'
    np.savez(s, indptr=np.array([0, 1]), items=np.array([0]))
    p = cli.build_parser()
    base = ['--top_k', '5', '--user_sequences', str(s)]
    assert cli.check_flags(p.parse_args(base + ['--user_deterministic'])).user_deterministic
    F = cli.check_flags(p.parse_args(base))
    assert not F.user_deterministic and not F.deterministic
    assert not cli.check_flags(p.parse_args(base + ['--deterministic', '--seed', '1'])).user_deterministic
    with pytest.raises(AssertionError, match='--user_deterministic needs --user_sequences'):
        cli.check_flags(p.parse_args(['--top_k', '5', '--user_deterministic']))
    assert '--user_deterministic' in p.format_help()


def _refuses(name, *args, match=None):
    with pytest.raises(_cabi.DaeError, match=match or name):
        _cabi.call(name, *args)


def test_new_exports_refuse_bad_arguments_without_gpu():
    P = 8   # any non-null fake pointer: the checks run before any device work
    loss = ('dae_seq_rank_loss_det', P, 4, P, 4, 4, P, P, 10, 1.0, P, 4)
    _refuses(*loss, None, None)                                        # loss_slots NULL
    _refuses(*loss[:8], 0, 1.0, P, 4, P, None)                         # n_pos = 0
    _refuses('dae_seq_rank_loss_det', P, 4, P, 4, 4, P, P, 10, 1.0, P, 4, 12, None, match='aligned')
    g = ('dae_seq_rank_loss_grad_det', P, 4, P, 4, 4, P, P, 10, 1.0, P, 4, P)
    _refuses(*g, P, P, None, None)
    _refuses(*g, P, P, 6, None, match='misaligned')
    imp = (P, 4, P, 4, 4, P, 10, P, P, P, 1.0, P, 4)
    _refuses('dae_impression_rank_loss_det', *imp, None, None)
    _refuses('dae_impression_rank_loss_det', P, 2, P, 4, 4, P, 10, P, P, P, 1.0, P, 4, P, None)   # ld_h < H
    _refuses('dae_impression_rank_loss_grad_det', *imp, P, P, None, P, None)
    sm = (P, 4, P, 4, 4, P, 10, P, P, P, P)
    _refuses('dae_impression_softmax_loss_det', *sm, 33, 0, 0, 1.0, P, 4, P, P, None)           # K > 32
    _refuses('dae_impression_softmax_loss_det', *sm, 2, 0, 0, 1.0, P, 4, P, None, None)         # no workspace
    _refuses('dae_impression_softmax_loss_grad_det', *sm, 2, 0, 0, 1.0, P, 4, P, P, P, P, None, None)
    _refuses('dae_loss_slots_sum', None, 4, P, None)
    _refuses('dae_loss_slots_sum', P, -1, P, None)
    _refuses('dae_loss_slots_sum', 4, 4, P, None, match='aligned')
    ws = 256
    o = ('dae_ordered_rows', P, P, P, 10, P, 4, P, 5, P, 4)
    _refuses(*o, 0, 4, P, 4, ws, 1 << 20, None)                        # n_slots = 0
    _refuses(*o, 3, 5, P, 4, ws, 1 << 20, None)                        # ld_dst < cols
    _refuses(*o, 3, 4, None, 4, ws, 1 << 20, None)                     # dst NULL
    _refuses('dae_ordered_rows', None, P, P, 10, P, 4, P, 5, P, 4, 3, 4, P, 4, ws, 1 << 20, None)   # triples NULL, n_a > 0
    _refuses(*o, 3, 4, P, 4, ws + 8, 1 << 20, None, match='aligned')
    _refuses('dae_ordered_rows', P, P, P, -1, P, 4, P, 5, P, 4, 3, 4, P, 4, ws, 1 << 20, None)
    _refuses('dae_ordered_rows_workspace', -1, 0, 4, P, match='dae_ordered_rows_workspace')
    _refuses('dae_ordered_rows_workspace', 0, 0, 0, P, match='dae_ordered_rows_workspace')
    _refuses('dae_ordered_rows_workspace', 1 << 30, 1 << 30, 4, P, match='dae_ordered_rows_workspace')


def test_ordered_rows_workspace_of_no_terms():
    assert _cabi.query('dae_ordered_rows_workspace', 0, 0, 7) == 0   # keys / values: 16 bytes per term, no sort scratch


def test_slot_sum_order_and_bound():
    rng = np.random.default_rng(0)
    for n in (0, 1, 255, 256, 257, 5000):
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)
        got = do.slot_sum(x, 0.25)
        assert abs(got - (0.25 + math.fsum(x))) <= do.slot_sum_bound(x) + np.finfo(np.float64).eps * abs(got)
    x = np.array([1.0, 1e16, -1e16] + [0.0] * 300)   # slots 0, 1, 2 go to three partials: 1 + 1e16 rounds only at level 2
    assert do.slot_sum(x) == (1.0 + 1e16) - 1e16


def test_ordered_rows_restatement():
    rng = np.random.default_rng(1)
    n_slots, cols = 6, 5
    src_a, src_b = rng.standard_normal((4, cols)).astype(np.float32), rng.standard_normal((3, cols)).astype(np.float32)
    a_slot, a_row, a_coef = np.array([2, -1, 2, 0]), np.array([0, 1, 3, 2]), np.array([0.5, 9.0, -1.25, 2.0], np.float32)
    b_slot = np.array([2, 5, -1])
    got = do.ordered_rows(a_slot, a_row, a_coef, src_a, b_slot, src_b, n_slots)
    want = np.zeros((n_slots, cols), np.float32)
    want[2] = ((np.float32(0.5) * src_a[0] + np.float32(-1.25) * src_a[3]).astype(np.float32) + src_b[0]).astype(np.float32)
    want[0] = np.float32(2.0) * src_a[2]
    want[5] = src_b[1]
    assert np.array_equal(got, want)
    exact = do.ordered_rows_fp64(a_slot, a_row, a_coef, src_a, b_slot, src_b, n_slots)
    assert np.abs(got - exact).max() <= 4 * np.finfo(np.float32).eps * np.abs(exact).max()
    # many terms on one slot: within the float32 bound of the exact sum
    n = 3000
    a = rng.standard_normal((n, cols)).astype(np.float32)
    c = rng.standard_normal(n).astype(np.float32)
    got = do.ordered_rows(np.zeros(n, np.int64), np.arange(n), c, a, [], a[:0], 1)
    exact = np.array([math.fsum(float(c[i]) * float(a[i, j]) for i in range(n)) for j in range(cols)])
    bound = (n + 1) * np.finfo(np.float32).eps * (np.abs(c[:, None].astype(np.float64) * a).sum(0))
    assert (np.abs(got[0] - exact) <= bound).all()
