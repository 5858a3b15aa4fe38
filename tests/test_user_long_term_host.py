"""Long-term user vectors (user_model.UserGRU / UserLSTM with long_term_users, DESIGN 4.18) without a GPU: the row export's
argument checks, the constructor, the table's layout and its mask draw, save / load, fit's row-count check, the learning-check
generator and the CLI's --user_long_term flags."""
import os
import sys

import numpy as np
import pytest
import torch

from dae_rnn_news_recommendation_b200 import _cabi
from dae_rnn_news_recommendation_b200.synth import make_long_term_impressions
from dae_rnn_news_recommendation_b200.user_model import LONG_TERM_LEARNING_RATE, UserAttention, UserGRU, UserLSTM, check_impressions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 0x1000   # a non-NULL pointer that no check dereferences


def _rows_args(**change):
    a = dict(table=P, ld=8, cols=8, rows=P, n=4, grad=P, ld_grad=8, slot1=P, slot2=P, counts=P, opt=_cabi.OPT['adam'], lr=0.1,
             momentum=0.5, stream=None)
    a.update(change)
    return list(a.values())


@pytest.mark.parametrize('change', [dict(table=None), dict(rows=None), dict(grad=None), dict(n=-1), dict(cols=0), dict(ld=7),
                                    dict(ld_grad=7), dict(opt=4), dict(opt=-1), dict(slot2=None), dict(counts=None),
                                    dict(opt=_cabi.OPT['momentum'], slot1=None), dict(opt=_cabi.OPT['ada_grad'], slot1=None)])
def test_rows_step_bad_arguments(change):
    with pytest.raises(_cabi.DaeError, match='dae_rows_optimizer_step'):
        _cabi.call('dae_rows_optimizer_step', *_rows_args(**change))


def test_rows_step_empty_list_is_a_no_op_without_gpu():
    """n = 0 returns before any CUDA call; SGD needs neither slots nor counts."""
    _cabi.call('dae_rows_optimizer_step', *_rows_args(n=0))
    _cabi.call('dae_rows_optimizer_step', *_rows_args(n=0, opt=_cabi.OPT['gradient_descent'], slot1=None, slot2=None, counts=None))


@pytest.mark.parametrize('cls', [UserGRU, UserLSTM])
def test_table_layout_and_slots(cls):
    for opt, s1, s2 in (('adam', 0.0, True), ('ada_grad', 0.1, False), ('momentum', 0.0, False), ('gradient_descent', None, False)):
        m = cls(6, long_term_users=11, opt=opt, device='cpu')
        assert m._lt.shape == (12, 6) and not m._lt.any() and m.long_term.shape == (11, 6)
        assert m.long_term.data_ptr() == m._lt.data_ptr()                      # a view: writes reach the model
        assert (m._lt_slot1 is None) == (s1 is None) and (m._lt_slot2 is not None) == s2
        if s1 is not None:
            assert (m._lt_slot1 == s1).all()
        assert m._lt_count.dtype == torch.int32 and m._lt_count.shape == (12,)
        assert sorted(m.state_dict()) == sorted(('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0'))
    m = cls(6, device='cpu')
    assert m.long_term is None and m.long_term_users is None
    assert m.long_term_learning_rate == LONG_TERM_LEARNING_RATE


def test_constructor_checks():
    for kw in (dict(long_term_users=0), dict(long_term_users=2.5), dict(long_term_users=True), dict(long_term_users=5, long_term_mask=1.5),
               dict(long_term_users=5, long_term_mask=-0.1), dict(long_term_users=5, long_term_learning_rate=0.0)):
        with pytest.raises(ValueError, match='long_term'):
            UserGRU(4, device='cpu', **kw)
    with pytest.raises(TypeError):
        UserAttention(4, long_term_users=5, device='cpu')
    m = UserLSTM(4, long_term_users=5, long_term_mask=0.2, long_term_learning_rate=0.07, device='cpu')
    assert (m.long_term_mask, m.long_term_learning_rate) == (0.2, 0.07)


def test_mask_draw_keyed_by_seed_epoch_user():
    m = UserGRU(4, long_term_users=20000, long_term_mask=0.3, seed=5, device='cpu')
    k0, k1 = m.long_term_kept(0).copy(), m.long_term_kept(1).copy()
    assert k0.shape == (20000,) and abs(k0.mean() - 0.7) < 0.02 and abs(k1.mean() - 0.7) < 0.02
    assert (k0 != k1).any()
    m2 = UserGRU(4, long_term_users=20000, long_term_mask=0.3, seed=5, batch_users=7, device='cpu')
    assert np.array_equal(m2.long_term_kept(1), k1) and np.array_equal(m2.long_term_kept(0), k0)
    assert not UserGRU(4, long_term_users=50, long_term_mask=1.0, device='cpu').long_term_kept(0).any()
    assert UserGRU(4, long_term_users=50, long_term_mask=0.0, device='cpu').long_term_kept(0).all()


def test_fit_refuses_more_users_than_rows_before_device_work():
    m = UserGRU(4, long_term_users=3, device='cpu')
    indptr = np.array([0, 2, 4, 6, 8], np.int64)
    with pytest.raises(ValueError, match='4 users.*3 rows'):
        m.fit((indptr, np.zeros(8, np.int32)), np.zeros((5, 4), np.float32))


@pytest.mark.parametrize('cls', [UserGRU, UserLSTM])
def test_save_load_round_trip_and_old_files(cls, tmp_path):
    m = cls(5, max_len=7, seed=3, long_term_users=9, device='cpu')
    m.long_term.copy_(torch.arange(45, dtype=torch.float32).view(9, 5))
    m.save(tmp_path / 'a.npz')
    z = np.load(tmp_path / 'a.npz')
    assert int(z['long_term_users']) == 9 and z['long_term'].shape == (9, 5)
    m2 = cls.load(tmp_path / 'a.npz', device='cpu')
    assert m2.long_term_users == 9 and m2.max_len == 7
    assert torch.equal(m2.long_term, m.long_term) and not m2._lt[9].any()
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k])
    with pytest.raises(ValueError, match='long-term table of shape'):
        cls.load(tmp_path / 'a.npz', long_term_users=4, device='cpu')
    assert cls.load(tmp_path / 'a.npz', long_term_users=None, device='cpu').long_term is None
    cls(5, seed=3, device='cpu').save(tmp_path / 'old.npz')                  # a file written without a table
    old = cls.load(tmp_path / 'old.npz', device='cpu')
    assert old.long_term is None and 'long_term' not in np.load(tmp_path / 'old.npz').files
    assert cls.load(tmp_path / 'old.npz', long_term_users=6, device='cpu').long_term.shape == (6, 5)
    torch_cell = (torch.nn.GRU if cls is UserGRU else torch.nn.LSTM)(5, 5)
    torch_cell.load_state_dict(m2.state_dict())


def test_learning_generator_hides_the_signal_before_the_window():
    labels = np.random.default_rng(0).integers(0, 6, 600)
    indptr, items, train, test = make_long_term_impressions(50, labels, window=4, history=(10, 20), shown=5, seed=1)
    lens = np.diff(indptr)
    assert ((lens >= 14) & (lens <= 24)).all()
    for imp in (train, test):
        share = []
        imp = check_impressions(imp, 600, 'test', indptr)
        assert np.array_equal(imp['time'], lens) and np.array_equal(imp['user'], np.arange(50))
        for u in range(50):
            s = items[indptr[u]:indptr[u + 1]]
            window, before = labels[s[-4:]], labels[s[:-4]]
            assert (window == window[0]).all()
            shown = imp['items'][imp['indptr'][u]:imp['indptr'][u + 1]]
            ck = imp['clicked'][imp['indptr'][u]:imp['indptr'][u + 1]].astype(bool)
            home = labels[shown[ck]][0]
            assert ck.sum() == 1 and home != window[0]
            assert (labels[shown[~ck]] != home).all() and (labels[shown[~ck]] == window[0]).sum() == 2
            share.append((before == home).mean())
        assert np.mean(share) > 0.55                                         # the home class dominates the earlier reads


def test_long_term_flags(tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    s = tmp_path / 's.npz'
    np.savez(s, indptr=np.array([0, 1]), items=np.array([0]))
    p = cli.build_parser()
    base = ['--top_k', '5', '--user_sequences', str(s)]
    F = cli.check_flags(p.parse_args(base + ['--user_long_term']))
    assert F.user_long_term and F.user_long_term_mask == 0.5 and F.user_long_term_lr is None
    F = cli.check_flags(p.parse_args(base + ['--user_cell', 'lstm', '--user_long_term', '--user_long_term_mask', '0.25',
                                             '--user_long_term_lr', '0.05']))
    assert (F.user_long_term_mask, F.user_long_term_lr) == (0.25, 0.05)
    assert not cli.check_flags(p.parse_args(base)).user_long_term
    with pytest.raises(AssertionError, match='--user_long_term needs --user_sequences'):
        cli.check_flags(p.parse_args(['--top_k', '5', '--user_long_term']))
    with pytest.raises(AssertionError, match='needs --user_cell gru or lstm'):
        cli.check_flags(p.parse_args(base + ['--user_cell', 'attention', '--user_long_term']))
    for extra in (['--user_long_term_mask', '0.3'], ['--user_long_term_lr', '0.1']):
        with pytest.raises(AssertionError, match='needs --user_long_term'):
            cli.check_flags(p.parse_args(base + extra))
    with pytest.raises(AssertionError, match='mask must lie'):
        cli.check_flags(p.parse_args(base + ['--user_long_term', '--user_long_term_mask', '1.5']))
    with pytest.raises(AssertionError, match='lr must be > 0'):
        cli.check_flags(p.parse_args(base + ['--user_long_term', '--user_long_term_lr', '0']))
