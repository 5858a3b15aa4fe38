"""The article encoder fine-tuned through the user encoders' losses (user_model.ArticleEncoder, DESIGN 4.19) on the GPU: the new
exports element by element, one joint batch against the fp64 oracle, the frozen-equivalence at learning rate 0, a few Adam steps,
the row-subset property of vectors(), save / load, the CLI and the cold-start learning check."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import user_article_oracle as ao  # noqa: E402
from helpers import rel_err  # noqa: E402
from impression_softmax_oracle import negative_sets  # noqa: E402
from user_gru_oracle import adam_tf  # noqa: E402

from dae_rnn_news_recommendation_b200 import _cabi, helpers  # noqa: E402
from dae_rnn_news_recommendation_b200._cabi import call  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import (ArticleEncoder, ImpressionBatch, Packed, UserAttention, UserGRU,  # noqa: E402
                                                         UserLSTM, usable_impressions)

D = torch.device('cuda:0')
CELLS = {'gru': UserGRU, 'lstm': UserLSTM, 'attention': UserAttention}


def _st():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(D)


# ---------------------------------------------------------------------------------------------------------------------------
# the new exports
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H', [37, 64])
def test_seq_rank_loss_grad(H):
    rng = np.random.default_rng(H)
    P, N = 300, 40
    h, emb = rng.normal(0, .5, (P, H)).astype(np.float32), rng.normal(0, .5, (N, H)).astype(np.float32)
    pos = rng.integers(0, N, P).astype(np.int32)
    pos[::7] = -1
    neg = ((pos + 1 + rng.integers(0, N - 1, P)) % N).astype(np.int32)   # articles repeat across positions
    neg[pos < 0] = -1
    dh = [torch.empty(P, H, device=D) for _ in range(2)]
    loss = [torch.zeros(1, dtype=torch.float64, device=D) for _ in range(2)]
    demb = torch.zeros(N, H, device=D)
    a = [_dev(x) for x in (h, emb, pos, neg)]
    call('dae_seq_rank_loss', a[0].data_ptr(), H, a[1].data_ptr(), H, H, a[2].data_ptr(), a[3].data_ptr(), P, 0.01, dh[0].data_ptr(), H,
         loss[0].data_ptr(), _st())
    call('dae_seq_rank_loss_grad', a[0].data_ptr(), H, a[1].data_ptr(), H, H, a[2].data_ptr(), a[3].data_ptr(), P, 0.01,
         dh[1].data_ptr(), H, loss[1].data_ptr(), demb.data_ptr(), H, _st())
    assert torch.equal(dh[0], dh[1]) and float(loss[0]) == pytest.approx(float(loss[1]), rel=1e-12)   # fp64 atomics: any order
    E = torch.tensor(emb.astype(np.float64), requires_grad=True)
    hp = torch.tensor(h.astype(np.float64))
    ok = torch.from_numpy(pos >= 0)
    x = (hp * E[torch.from_numpy(np.maximum(neg, 0)).long()]).sum(1) - (hp * E[torch.from_numpy(np.maximum(pos, 0)).long()]).sum(1)
    (0.01 * torch.nn.functional.softplus(x[ok]).sum()).backward()
    assert rel_err(demb.cpu().numpy(), E.grad.numpy()) < 1e-5


def _impressions(rng, P, N, per_pos=2, m=(2, 9)):
    pos_indptr, indptr, items, clicked = [0], [0], [], []
    for p in range(P):
        k = int(rng.integers(0, per_pos + 1))
        for _ in range(k):
            n = int(rng.integers(*m))
            items.append(rng.choice(N, n, replace=False))            # the same article recurs across impressions and positions
            c = np.zeros(n, np.uint8)
            c[rng.choice(n, int(rng.integers(1, n)), replace=False)] = 1
            clicked.append(c)
            indptr.append(indptr[-1] + n)
        pos_indptr.append(pos_indptr[-1] + k)
    return (np.array(pos_indptr, np.int64), np.array(indptr, np.int64), np.concatenate(items).astype(np.int32),
            np.concatenate(clicked))


@pytest.mark.parametrize('loss', ['pairwise', 'softmax0', 'softmax2'])
def test_impression_loss_grads(loss):
    rng = np.random.default_rng(len(loss))
    P, N, H = 120, 30, 37
    h, emb = rng.normal(0, .5, (P, H)).astype(np.float32), rng.normal(0, .5, (N, H)).astype(np.float32)
    pos_indptr, indptr, items, clicked = _impressions(rng, P, N)
    n_imp = indptr.size - 1
    ids = np.arange(n_imp, dtype=np.int64) * 7 + 3
    K = 0 if loss == 'softmax0' else 2
    a = [_dev(x) for x in (h, emb, pos_indptr, indptr, items, clicked, ids)]
    dh = [torch.empty(P, H, device=D) for _ in range(2)]
    ls = [torch.zeros(1, dtype=torch.float64, device=D) for _ in range(2)]
    demb = torch.zeros(N, H, device=D)
    ws = torch.empty(2 * items.size, dtype=torch.int32, device=D)
    head = lambda i: (a[0].data_ptr(), H, a[1].data_ptr(), H, H, a[2].data_ptr(), P, a[3].data_ptr(), a[4].data_ptr(),  # noqa: E731
                      a[5].data_ptr())
    if loss == 'pairwise':
        call('dae_impression_rank_loss', *head(0), 0.5, dh[0].data_ptr(), H, ls[0].data_ptr(), _st())
        call('dae_impression_rank_loss_grad', *head(1), 0.5, dh[1].data_ptr(), H, ls[1].data_ptr(), demb.data_ptr(), H, _st())
    else:
        call('dae_impression_softmax_loss', *head(0), a[6].data_ptr(), K, 5, 1, 0.5, dh[0].data_ptr(), H, ls[0].data_ptr(),
             ws.data_ptr(), _st())
        call('dae_impression_softmax_loss_grad', *head(1), a[6].data_ptr(), K, 5, 1, 0.5, dh[1].data_ptr(), H, ls[1].data_ptr(),
             ws.data_ptr(), demb.data_ptr(), H, _st())
    assert torch.equal(dh[0], dh[1]) and float(ls[0]) == pytest.approx(float(ls[1]), rel=1e-12)
    E = torch.tensor(emb.astype(np.float64), requires_grad=True)
    total = 0.0
    for p in range(P):
        hp = torch.tensor(h[p].astype(np.float64))
        for q in range(pos_indptr[p], pos_indptr[p + 1]):
            it, c = items[indptr[q]:indptr[q + 1]], clicked[indptr[q]:indptr[q + 1]].astype(bool)
            s = E[torch.from_numpy(it).long()] @ hp
            if loss == 'pairwise':
                total = total + torch.nn.functional.softplus(s[torch.from_numpy(~c)][None] - s[torch.from_numpy(c)][:, None]).mean()
            else:
                for cp, S in negative_sets(c, int(ids[q]), K, 5, 1):
                    A = torch.from_numpy(np.concatenate([[cp], S]).astype(np.int64))
                    total = total + torch.logsumexp(s[A], 0) - s[A][0]
    (0.5 * total).backward()
    assert rel_err(demb.cpu().numpy(), E.grad.numpy()) < 1e-5


def test_rows_scatter_add():
    rng = np.random.default_rng(0)
    src = rng.normal(size=(500, 37)).astype(np.float32)
    idx = rng.integers(-1, 20, 500).astype(np.int32)
    dst0 = rng.normal(size=(20, 40)).astype(np.float32)
    dst, s_d, i_d = _dev(dst0), _dev(src), _dev(idx)
    call('dae_rows_scatter_add', s_d.data_ptr(), 37, i_d.data_ptr(), 500, 37, dst.data_ptr(), 40, _st())
    want = dst0.astype(np.float64)
    for p in np.flatnonzero(idx >= 0):
        want[idx[p], :37] += src[p]
    assert rel_err(dst.cpu().numpy(), want) < 1e-6


def test_touch_compact_is_exact_across_calls():
    rng = np.random.default_rng(1)
    N = 5000
    art = ArticleEncoder(sp.random(N, 30, density=0.2, random_state=0, format='csr', dtype=np.float32),
                         {'enc_w': np.zeros((30, 4), np.float32), 'enc_b': np.zeros(4, np.float32)}, device=D)
    for n in (1, 1023, 1024, 1025, 40000):
        ids = rng.integers(-1, N, n).astype(np.int32)
        rows, slots, T = art.touch(_dev(ids))
        r_ref, s_ref = ao.compact(ids)
        assert T == r_ref.size
        assert np.array_equal(rows.cpu().numpy(), r_ref) and np.array_equal(slots.cpu().numpy(), s_ref)


# ---------------------------------------------------------------------------------------------------------------------------
# vectors()
# ---------------------------------------------------------------------------------------------------------------------------
def _art(N=600, F=300, H=37, act='sigmoid', seed=0, **kw):
    rng = np.random.default_rng(seed)
    X = sp.random(N, F, density=0.1, random_state=seed, format='csr', dtype=np.float32)
    p = {'enc_w': rng.normal(0, .3, (F, H)).astype(np.float32), 'enc_b': rng.normal(0, .1, H).astype(np.float32)}
    return ArticleEncoder(X, p, enc_act_func=act, in_scale=0.7, device=D, **kw), X, p


def test_vectors_subset_bit_equal_and_against_transform():
    from dae_rnn_news_recommendation_b200.autoencoder import utils
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR, TrainEngine
    art, X, p = _art(N=9000, H=64)
    full = art.vectors()
    for sel in (np.array([5]), np.arange(100, 140), np.random.default_rng(0).choice(9000, 5000, replace=False)):
        assert np.array_equal(art.vectors(X[sel]), full[sel])
    rows, _, T = art.touch(_dev(np.array([7, 3, 7, 8000], np.int32)))
    E, _ = art.encode_rows(rows, T)
    assert np.array_equal(E.cpu().numpy(), full[[7, 3, 8000]])
    eng = TrainEngine(300, 64, enc_act_func='sigmoid', device=D)
    eng.set_parameters(p['enc_w'], p['enc_b'])
    ref = eng.encode(DeviceCSR(utils.decay_noise(X, 0.3), D)).cpu().numpy()   # the DAE's transform of decayed inputs
    assert rel_err(full, ref) < 1e-5
    with pytest.raises(ValueError, match='features'):
        art.vectors(X[:, :10])


# ---------------------------------------------------------------------------------------------------------------------------
# one joint batch against the oracle
# ---------------------------------------------------------------------------------------------------------------------------
def _workload(N, rng, users=24):
    lens = rng.integers(2, 9, users)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N, int(indptr[-1])).astype(np.int32)
    it, ck, us, tm = [], [], [], []
    for u in range(users):
        for t in range(1, lens[u] + 1):
            n = int(rng.integers(3, 7))
            it.append(rng.choice(N, n, replace=False))
            c = np.zeros(n, np.uint8)
            c[rng.choice(n, int(rng.integers(1, n)), replace=False)] = 1
            ck.append(c)
            us.append(u)
            tm.append(t)
    imp = {'user': np.array(us), 'time': np.array(tm), 'indptr': np.concatenate([[0], np.cumsum([len(a) for a in it])]),
           'items': np.concatenate(it).astype(np.int32), 'clicked': np.concatenate(ck)}
    return indptr, items, imp


def _oracle_batch(m, kind, indptr, items, imp, art, X, p, params):
    """The oracle's (seqs, data) for the model's first batch of epoch 0, in the packed order of the device path."""
    use = usable_impressions(imp, indptr, m.max_len) if kind != 'random' else None
    active = None if kind == 'random' else np.unique(imp['user'][use])
    users = m.batches(indptr, 0, active)[0]
    pk = Packed(indptr, items, users, m.max_len)
    seqs = [items[indptr[u + 1] - L:indptr[u + 1]] for u, L in zip(pk.order, pk.L)]

    def at(pp):
        t = int(np.searchsorted(pk.off, pp, side='right') - 1)
        return int(pp - pk.off[t]), t
    if kind == 'random':
        b = m.article_batch
        P = pk.P
        neg = b['rows'].cpu().numpy()[b['slots'][2 * P:].cpu().numpy()]
        data = [np.array([neg[pk.off[t] + i] for t in range(L - 1)]) for i, L in enumerate(pk.L)]
    else:
        ib = ImpressionBatch(pk, imp, use, indptr)
        data = []
        for k in range(ib.n):
            i, t = at(ib.p[k])
            it, c = ib.items[ib.indptr[k]:ib.indptr[k + 1]], ib.clicked[ib.indptr[k]:ib.indptr[k + 1]]
            if kind == 'pairwise':
                data.append((i, t, it, c))
            else:
                data += [(i, t, it[cp], it[S]) for cp, S in negative_sets(c, int(ib.ids[k]), m.impression_negatives, m.seed, 0)]
    return pk, seqs, data


def _theta_of(cell, grads, H):
    if cell == 'attention':
        g = lambda w, b: np.concatenate([grads[w], grads[b][:, None]], 1).ravel()   # noqa: E731
        return np.concatenate([g('self_attn.in_proj_weight', 'self_attn.in_proj_bias'), g('self_attn.out_proj.weight',
                               'self_attn.out_proj.bias'), g('pool.weight', 'pool.bias'), grads['pool.query']])
    return np.concatenate([np.concatenate([grads['weight_%s_l0' % k], grads['bias_%s_l0' % k][:, None]], 1).ravel() for k in ('hh', 'ih')])


CASES = [(c, k, H) for c in CELLS for k in ao.KINDS for H in (37, 64)] + [('gru', 'softmax', 500), ('lstm', 'random', 'long_term')]


@pytest.mark.parametrize('cell,kind,H', CASES)
def test_joint_batch_against_oracle(cell, kind, H):
    long_term = H == 'long_term'
    H = 40 if long_term else H
    rng = np.random.default_rng(H)
    N = 80
    art, X, p = _art(N=N, F=120, H=H, act='tanh', seed=H, learning_rate=0.0)
    indptr, items, imp = _workload(N, rng)
    kw = dict(long_term_users=len(indptr) - 1, long_term_mask=0.0) if long_term else {}
    if cell == 'attention':
        kw['heads'] = 1 if H == 37 else 4
    m = CELLS[cell](H, max_len=6, batch_users=4096, num_epochs=1, seed=2, learning_rate=0.0,
                    impression_loss='softmax' if kind == 'softmax' else 'pairwise', impression_negatives=2, **kw)
    params = {k: v.numpy().astype(np.float64) for k, v in m.state_dict().items()}
    m.fit((indptr, items), art, impressions=None if kind == 'random' else imp)
    pk, seqs, data = _oracle_batch(m, kind, indptr, items, imp, art, X, p, params)
    r = ao.joint(cell, params, p['enc_w'], p['enc_b'], X, 'tanh', 0.7, seqs, kind, data, heads=kw.get('heads'))
    b = m.article_batch
    rows = b['rows'].cpu().numpy()
    assert np.array_equal(np.sort(rows), np.unique(rows))
    assert rel_err(b['E'].cpu().numpy(), r['E'][rows]) < 1e-5
    dX = np.zeros((pk.P, H))
    for i, L in enumerate(pk.L):
        dX[pk.off[np.arange(L)] + i] = r['dX'][i]
    tol = 2e-4 if H < 500 else 1e-3
    assert rel_err(b['dX'].cpu().numpy(), dX) < tol
    assert rel_err(b['dE'].cpu().numpy(), r['dA'][rows]) < tol          # dE_t after the encoder backward holds dA
    g = art.grad.cpu().numpy()
    assert rel_err(g[:-H].reshape(-1, H), r['dW']) < tol
    assert rel_err(g[-H:], r['dbh']) < tol
    assert rel_err(m.grad.cpu().numpy(), _theta_of(cell, r['grads'], H)) < tol
    assert abs(m.train_loss[0] - r['loss']) < 1e-5 * max(1.0, abs(r['loss']))


# ---------------------------------------------------------------------------------------------------------------------------
# learning rate 0, a few Adam steps, save / load
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cell', list(CELLS))
@pytest.mark.parametrize('kind', ['random', 'softmax'])
def test_learning_rate_zero_is_the_frozen_fit(cell, kind):
    rng = np.random.default_rng(5)
    art, X, p = _art(N=500, F=200, H=64, learning_rate=0.0)
    indptr, items, imp = _workload(500, rng, users=300)
    kw = dict(max_len=6, batch_users=64, num_epochs=2, seed=4, impression_loss='softmax' if kind == 'softmax' else 'pairwise')
    a, b = CELLS[cell](64, **kw), CELLS[cell](64, **kw)
    W0 = art.theta.clone()
    a.fit((indptr, items), art, impressions=None if kind == 'random' else imp)
    b.fit((indptr, items), art.vectors(), impressions=None if kind == 'random' else imp)
    assert torch.equal(art.theta, W0)
    assert torch.equal(a.theta, b.theta)
    assert a.train_loss == pytest.approx(b.train_loss, rel=1e-12)   # the batch loss sums are fp64 atomics in any order


@pytest.mark.parametrize('cell', list(CELLS))
def test_five_adam_steps_against_fp64(cell):
    rng = np.random.default_rng(9)
    H, N = 32, 60
    art, X, p = _art(N=N, F=90, H=H, act='sigmoid', seed=3, learning_rate=1e-2)
    indptr, items, imp = _workload(N, rng, users=12)
    m = CELLS[cell](H, max_len=6, batch_users=4096, num_epochs=5, seed=1, learning_rate=1e-2)
    params = {k: v.numpy().astype(np.float64) for k, v in m.state_dict().items()}
    m.fit((indptr, items), art, impressions=imp)
    W, bh = p['enc_w'].astype(np.float64), p['enc_b'].astype(np.float64)
    state = {k: [np.zeros_like(v), np.zeros_like(v)] for k, v in list(params.items()) + [('W', W), ('bh', bh)]}
    for step in range(1, 6):
        _, seqs, data = _oracle_batch(m, 'pairwise', indptr, items, imp, art, X, p, params)
        r = ao.joint(cell, params, W, bh, X, 'sigmoid', 0.7, seqs, 'pairwise', data, heads=default_heads(H))
        for k in params:
            adam_tf(params[k], r['grads'][k], *state[k], step, 1e-2)
        adam_tf(W, r['dW'], *state['W'], step, 1e-2)
        adam_tf(bh, r['dbh'], *state['bh'], step, 1e-2)
    got = {k: v.numpy() for k, v in m.state_dict().items()}
    for k in params:
        assert rel_err(got[k], params[k]) < 2e-3, k
    assert rel_err(art.W.cpu().numpy(), W) < 2e-3 and rel_err(art.bh.cpu().numpy(), bh) < 2e-3


def default_heads(H):
    from dae_rnn_news_recommendation_b200.user_model import default_heads as d
    return d(H)


def test_save_load_and_entry_points(tmp_path):
    art, X, p = _art(learning_rate=3e-3, opt='momentum')
    art.W.add_(0.01)
    art.save(tmp_path / 'a.npz')
    b = ArticleEncoder.load(tmp_path / 'a.npz', X, device=D)
    assert torch.equal(b.theta, art.theta) and (b.opt, b.learning_rate, b.in_scale, b.enc_act_func) == ('momentum', 3e-3, 0.7, 'sigmoid')
    assert set(art.state_dict()) == {'enc-w', 'hidden-bias'}
    rng = np.random.default_rng(0)
    indptr, items, imp = _workload(600, rng, users=50)
    m = UserGRU(37, max_len=6, num_epochs=1)
    m.fit((indptr, items), art)
    emb = art.vectors()
    assert np.array_equal(m.transform((indptr, items), art), m.transform((indptr, items), emb))
    q = m.impression_states((indptr, items), art, imp)
    assert np.array_equal(q, m.impression_states((indptr, items), emb, imp))
    assert helpers.impression_metrics(q, art, imp) == helpers.impression_metrics(q, emb, imp)
    assert np.array_equal(m.recommend((indptr, items), art, k=3)[0], m.recommend((indptr, items), emb, k=3)[0])


def test_cli_fine_tune_articles(capsys, tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.synth import make_sequences
    argv = ['--model_name', 'synart', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--top_k', '5']
    trX, _, trL, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    indptr, items, targets = make_sequences(300, trL, mean_len=8, seed=4)
    np.savez(tmp_path / 's.npz', indptr=indptr, items=items, targets=targets)
    model = cli.main(argv + ['--user_sequences', str(tmp_path / 's.npz'), '--user_epochs', '2', '--user_fine_tune_articles',
                             '--user_article_lr', '0.001'])
    assert 'users (GRU): hit rate@5' in capsys.readouterr().out
    enc = np.load(model.data_dir + 'article_encoded_fine_tuned.npy')
    z = np.load(model.data_dir + 'user_gru_article_encoder.npz')
    assert enc.shape == (trX.shape[0], z['enc-w'].shape[1]) and float(z['in_scale']) == pytest.approx(0.7)
    assert 0.0 <= model.evaluation['user_gru_hit_rate'] <= 1.0


# test-impression AUC on bench_user_articles.learning_workload's held-out articles, measured on an H100: see DESIGN 4.19; the
# asserted margin is half the measured gap
LEARNING_MARGIN = 0.26


def test_joint_training_helps_cold_start_articles():
    from bench_user_articles import learning_auc, learning_workload
    from dae_rnn_news_recommendation_b200.user_model import ARTICLE_LEARNING_RATE
    data = learning_workload()
    frozen = learning_auc(data)
    joint = learning_auc(data, ARTICLE_LEARNING_RATE)
    print('held-out test-impression AUC: frozen %.4f, joint %.4f' % (frozen, joint))
    assert joint - frozen > LEARNING_MARGIN, (frozen, joint)
