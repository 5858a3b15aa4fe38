"""CPU checks of the article encoder fine-tuned through the user encoders' losses (user_model.ArticleEncoder, DESIGN 4.19): the fp64
joint oracle against the frozen-embedding oracles and central differences, the compaction's restatement, the argument checks and
the CLI flags."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import impression_oracle as io_
import user_article_oracle as ao
import user_attention_oracle as uo
import user_gru_oracle as go
import user_lstm_oracle as lo
from dae_rnn_news_recommendation_b200.user_model import ArticleEncoder, UserGRU

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(cell, H=4, N=9, Fdim=12, seed=0):
    rng = np.random.default_rng(seed)
    X = sp.random(N, Fdim, density=0.4, random_state=seed, format='csr', dtype=np.float32)
    W = rng.normal(0, 0.5, (Fdim, H))
    bh = rng.normal(0, 0.2, H)
    if cell == 'attention':
        A = 3
        params = {'self_attn.in_proj_weight': rng.normal(0, .4, (3 * H, H)), 'self_attn.in_proj_bias': rng.normal(0, .1, 3 * H),
                  'self_attn.out_proj.weight': rng.normal(0, .4, (H, H)), 'self_attn.out_proj.bias': rng.normal(0, .1, H),
                  'pool.weight': rng.normal(0, .4, (A, H)), 'pool.bias': rng.normal(0, .1, A), 'pool.query': rng.normal(0, .4, A)}
    else:
        G = 3 if cell == 'gru' else 4
        params = {'weight_ih_l0': rng.normal(0, .4, (G * H, H)), 'weight_hh_l0': rng.normal(0, .4, (G * H, H)),
                  'bias_ih_l0': rng.normal(0, .1, G * H), 'bias_hh_l0': rng.normal(0, .1, G * H)}
    seqs = [np.array([0, 3, 3, 5]), np.array([2, 1, 7]), np.array([8, 0])]
    negs = [np.array([4, 6, 1]), np.array([0, 0]), np.array([3])]
    imps = [(0, 1, np.array([3, 5, 6]), np.array([1, 0, 0])), (1, 0, np.array([1, 2, 4, 8]), np.array([0, 1, 1, 0])),
            (0, 2, np.array([5, 0]), np.array([0, 1]))]
    samples = [(0, 1, 3, np.array([5, 6])), (1, 0, 2, np.array([1, 8])), (1, 0, 4, np.array([1]))]
    return X, W, bh, params, seqs, {'random': negs, 'pairwise': imps, 'softmax': samples}


@pytest.mark.parametrize('cell', ['gru', 'lstm', 'attention'])
@pytest.mark.parametrize('kind', ao.KINDS)
def test_detached_oracle_is_the_frozen_oracle(cell, kind):
    X, W, bh, params, seqs, data = _case(cell)
    r = ao.joint(cell, params, W, bh, X, 'sigmoid', 0.7, seqs, kind, data[kind], heads=2, articles=False)
    E = r['E']
    if kind == 'random':
        ref = {'gru': lambda: go.loss_and_grads(params, seqs, data[kind], E), 'lstm': lambda: lo.loss_and_grads(params, seqs, data[kind], E),
               'attention': lambda: uo.loss_and_grads(params, seqs, data[kind], E, 2)}[cell]()
    elif kind == 'pairwise':
        ref = {'gru': lambda: io_.impression_loss_and_grads(params, seqs, E, data[kind]),
               'lstm': lambda: lo.impression_loss_and_grads(params, seqs, E, data[kind]),
               'attention': lambda: uo.impression_loss_and_grads(params, seqs, E, data[kind], 2)}[cell]()
    else:
        if cell != 'attention':
            pytest.skip('the sampled-softmax oracle of the existing tests is the attention encoder\'s')
        ref = uo.softmax_loss_and_grads(params, seqs, E, data[kind], 2)
    assert abs(r['loss'] - ref[0]) <= 1e-12 * max(1.0, abs(ref[0]))
    for k, g in ref[1].items():
        np.testing.assert_allclose(r['grads'][k], g, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize('cell,kind', [('gru', 'random'), ('lstm', 'pairwise'), ('attention', 'softmax')])
def test_dW_against_central_differences(cell, kind):
    X, W, bh, params, seqs, data = _case(cell, seed=3)
    r = ao.joint(cell, params, W, bh, X, 'tanh', 0.8, seqs, kind, data[kind], heads=2)
    eps = 1e-6
    for (i, j) in [(0, 0), (3, 2), (7, 1), (11, 3)]:
        Wp, Wm = W.copy(), W.copy()
        Wp[i, j] += eps
        Wm[i, j] -= eps
        fp = ao.joint(cell, params, Wp, bh, X, 'tanh', 0.8, seqs, kind, data[kind], heads=2)['loss']
        fm = ao.joint(cell, params, Wm, bh, X, 'tanh', 0.8, seqs, kind, data[kind], heads=2)['loss']
        assert abs((fp - fm) / (2 * eps) - r['dW'][i, j]) <= 1e-6 * max(1.0, abs(r['dW'][i, j]))
    for j in range(W.shape[1]):
        bp, bm = bh.copy(), bh.copy()
        bp[j] += eps
        bm[j] -= eps
        d = (ao.joint(cell, params, W, bp, X, 'tanh', 0.8, seqs, kind, data[kind], heads=2)['loss'] -
             ao.joint(cell, params, W, bm, X, 'tanh', 0.8, seqs, kind, data[kind], heads=2)['loss']) / (2 * eps)
        assert abs(d - r['dbh'][j]) <= 1e-6 * max(1.0, abs(d))


def test_dE_is_the_scatter_of_dX_and_the_loss_gradient():
    """dL/de_a = sum over the positions reading a of dL/dx_p + the loss's own gradient at a: the split the device path uses."""
    X, W, bh, params, seqs, data = _case('gru')
    r = ao.joint('gru', params, W, bh, X, 'sigmoid', 1.0, seqs, 'random', data['random'])
    E = torch.tensor(r['E'], requires_grad=True)
    hs = [torch.tensor(h) for h in r['states']]
    ao.loss('random', hs, E, seqs, data['random']).backward()
    want = E.grad.numpy().copy()
    for s, dx in zip(seqs, r['dX']):
        np.add.at(want, s, dx)
    np.testing.assert_allclose(r['dE'], want, rtol=1e-10, atol=1e-13)


def test_compaction_restatement():
    ids = np.array([5, 2, 5, -1, 7, 2, 0, 7, -1, 9], np.int32)
    rows, slots = ao.compact(ids)
    assert rows.tolist() == [5, 2, 7, 0, 9]
    assert slots.tolist() == [0, 1, 0, -1, 2, 1, 3, 2, -1, 4]
    assert (rows[slots[ids >= 0]] == ids[ids >= 0]).all()
    # impression items join after the reads, the next reads and the negatives, and keep their first-seen slot
    items, nxt, imp = np.array([3, 1]), np.array([1, -1]), np.array([4, 3, 8])
    rows, slots = ao.compact(np.concatenate([items, nxt, imp]))
    assert rows.tolist() == [3, 1, 4, 8] and slots.tolist() == [0, 1, 1, -1, 2, 0, 3]


def _art(**kw):
    X = sp.random(6, 10, density=0.5, random_state=0, format='csr', dtype=np.float32)
    p = {'enc_w': np.zeros((10, 4), np.float32), 'enc_b': np.zeros(4, np.float32)}
    p.update(kw.pop('params', {}))
    return ArticleEncoder(X, p, device='cpu', **kw)


def test_article_encoder_argument_checks():
    with pytest.raises(ValueError, match='F = 10'):
        _art(params={'enc_w': np.zeros((9, 4))})
    with pytest.raises(ValueError, match='hidden bias'):
        _art(params={'enc_b': np.zeros(5)})
    with pytest.raises(ValueError, match='opt'):
        _art(opt='rmsprop')
    with pytest.raises(ValueError, match='learning_rate'):
        _art(learning_rate=-1.0)
    a = _art(params={'enc-w': np.ones((10, 4)), 'hidden-bias': np.ones(4)})
    assert float(a.W.sum()) == 40.0 and a.state_dict()['hidden-bias'].shape == (4,)
    with pytest.raises(ValueError, match='H = 4, the model 5'):
        UserGRU(5, device='cpu').fit((np.array([0, 2]), np.array([0, 1])), a)
    with pytest.raises(ValueError, match='outside'):
        UserGRU(4, device='cpu').fit((np.array([0, 2]), np.array([0, 6])), a)
    imp = {'user': np.array([0]), 'time': np.array([1]), 'indptr': np.array([0, 2]), 'items': np.array([1, 6]),
           'clicked': np.array([1, 0])}
    with pytest.raises(ValueError, match='outside'):
        UserGRU(4, device='cpu').fit((np.array([0, 2]), np.array([0, 1])), a, impressions=imp)


def test_fine_tune_flags(tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    s = tmp_path / 's.npz'
    np.savez(s, indptr=np.array([0, 1]), items=np.array([0]))
    p = cli.build_parser()
    base = ['--top_k', '5', '--user_sequences', str(s)]
    F = cli.check_flags(p.parse_args(base + ['--user_fine_tune_articles', '--user_article_lr', '0.001']))
    assert F.user_fine_tune_articles and F.user_article_lr == 0.001
    assert not cli.check_flags(p.parse_args(base)).user_fine_tune_articles
    with pytest.raises(AssertionError, match='--user_fine_tune_articles needs --user_sequences'):
        cli.check_flags(p.parse_args(['--top_k', '5', '--user_fine_tune_articles']))
    with pytest.raises(AssertionError, match='--user_article_lr needs --user_fine_tune_articles'):
        cli.check_flags(p.parse_args(base + ['--user_article_lr', '0.01']))
    with pytest.raises(AssertionError, match='must be >= 0'):
        cli.check_flags(p.parse_args(base + ['--user_fine_tune_articles', '--user_article_lr', '-1']))


def test_new_exports_refuse_bad_arguments_without_gpu():
    from dae_rnn_news_recommendation_b200 import _cabi
    x = 1 << 20   # a non-null pointer value: every call below fails its checks before reading it
    bad = {
        'dae_encode_csr_fwd_groups': (x, x, x, None, 4, 10, 8, 1.0, x, x, 1, x, 8, None, None, None, 0, 2, None),
        'dae_seq_rank_loss_grad': (x, 8, x, 8, 8, x, x, 4, 1.0, x, 8, x, None, 8, None),
        'dae_impression_rank_loss_grad': (x, 8, x, 8, 8, x, 4, x, x, x, 1.0, x, 8, x, x, 4, None),
        'dae_impression_softmax_loss_grad': (x, 8, x, 8, 8, x, 4, x, x, x, x, 4, 0, 0, 1.0, x, 8, x, x, x, 4, None),
        'dae_touch_compact': (x, 10, 0, x, x, x, x, x, None),
        'dae_rows_scatter_add': (x, 4, x, 3, 8, x, 8, None),
    }
    for name, args in bad.items():
        with pytest.raises(_cabi.DaeError, match=name):
            _cabi.call(name, *args)
    with pytest.raises(_cabi.DaeError, match='dae_touch_compact: null'):
        _cabi.call('dae_touch_compact', None, 10, 1, x, x, x, x, x, None)
    assert _cabi.query('dae_touch_compact_workspace', 1025) == 3
    with pytest.raises(_cabi.DaeError, match='dae_touch_compact_workspace'):
        _cabi.query('dae_touch_compact_workspace', -1)
