"""The sampled-softmax impression loss on the GPU: dae_impression_softmax_loss through the C ABI against the fp64 reference of
tests/impression_softmax_oracle.py element by element, the drawn sets themselves bit for bit against the host draws, whole
UserGRU / UserLSTM / UserAttention batches against fp64 autograd, the K = 1 reduction to the pairwise fit, the learning check and
the CLI."""
import os
import sys

import numpy as np
import pytest
import torch

import impression_kernel_oracle as ko
import impression_softmax_oracle as so
import user_attention_oracle as ao
from helpers import rel_err
from user_gru_oracle import NAMES, gru_states
from user_lstm_oracle import lstm_states

from dae_rnn_news_recommendation_b200 import _cabi, helpers
from dae_rnn_news_recommendation_b200.user_model import (ATTENTION_NAMES, ImpressionBatch, Packed, UserAttention, UserGRU, UserLSTM,
                                                         check_impressions, usable_impressions)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
f32 = np.float32


def _st():
    return torch.cuda.current_stream().cuda_stream


def _pass_rows():
    """Positions one pass of the kernel's grid covers: 16 CTAs of 4 warps per SM."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 4


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _padded(a, ld, fill=np.nan):
    out = np.full((a.shape[0], ld), fill, f32)
    out[:, :a.shape[1]] = a
    return _dev(out)


def _call(h, emb, pi, ip, items, clicked, ids, K, seed, epoch, scale, H, ld=None, extra=3, loss0=1.25):
    """One dae_impression_softmax_loss call on fresh device copies (operands padded with NaN to their own leading dimensions,
    dh starting as NaN, the workspace as garbage): (dh [n_pos + extra, ld_dh], loss sum)."""
    n_pos = len(pi) - 1
    ld_h, ld_e, ld_dh = ld or (H, H, H)
    d_h, d_e = _padded(h, ld_h), _padded(emb, ld_e)
    d = [_dev(x) for x in (pi, ip, items, clicked, ids)]
    dh = torch.full((n_pos + extra, ld_dh), float('nan'), dtype=torch.float32, device=DEV)
    loss = torch.full((1,), loss0, dtype=torch.float64, device=DEV)
    ws = torch.full((2 * max(int(ip[-1]), 1),), -7, dtype=torch.int32, device=DEV)
    _cabi.call('dae_impression_softmax_loss', d_h.data_ptr(), ld_h, d_e.data_ptr(), ld_e, H, d[0].data_ptr(), n_pos, d[1].data_ptr(),
               d[2].data_ptr(), d[3].data_ptr(), d[4].data_ptr(), K, seed, epoch, scale, dh.data_ptr(), ld_dh, loss.data_ptr(),
               ws.data_ptr(), _st())
    torch.cuda.synchronize()
    return dh.cpu().numpy(), float(loss.cpu().numpy()[0]) - loss0


CASES = [(H, 4) for H in (1, 31, 32, 33, 37, 500)] + [(H, K) for H in (33, 500) for K in (0, 1, 32)]


@pytest.mark.parametrize('H,K', CASES)
def test_kernel_against_fp64(H, K):
    """Impressions of 2 to 5 000 articles (|N| = 1, clicks in the first or last 256-score chunk, 700 clicks), skipped
    impressions, positions without impressions, x at +-100, +-30 and 0, n_pos past three grid passes."""
    rng = np.random.default_rng(3000 + 10 * H + K)
    n_pos = 3 * _pass_rows() + 37
    h, emb, pi, ip, items, clicked, info = ko.loss_case(rng, H, n_pos)
    ids = so.impression_ids(rng, len(ip) - 1)
    ld = (H + 1, H + 3, H + 2)
    scale = 1.0 / 29
    dh, loss = _call(h, emb, pi, ip, items, clicked, ids, K, 12345, 6, scale, H, ld)
    w_dh, s_dh, w_loss, s_loss, sets = so.softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 12345, 6, scale, H)
    tag = 'softmax H=%d K=%d' % (H, K)
    ko.check(tag + ' dh', dh[:n_pos, :H], w_dh, s_dh, ko.C_FP32)
    ko.check(tag + ' sum', loss, w_loss, s_loss, ko.C_FP32, tiny=1e-15)
    used = np.repeat(np.arange(n_pos), np.diff(pi))[ko.usable(ip, clicked)[:pi[-1]]]
    none = np.setdiff1d(np.arange(n_pos), used)
    assert set(info['skipped_only']) <= set(none) and none.size > n_pos // 2
    assert (dh[none, :H] == 0).all()
    assert np.isnan(dh[:, H:]).all() and np.isnan(dh[n_pos:]).all()
    assert np.isin(np.arange(4), used // _pass_rows()).all()
    if K:
        assert any(v is not None and len(v[0][1]) == K for v in sets.values())            # the sampled path ran
    dh2, _ = _call(h, emb, pi, ip, items, clicked, ids, K, 12345, 6, scale, H, ld)
    assert np.array_equal(dh.view(np.uint32), dh2.view(np.uint32))
    print(tag, {k: round(v, 4) for k, v in ko.WORST.items() if k.startswith(tag)})


def _one_hot_case(rng, n_imp, H, K):
    """n_imp impressions of one click and 2 .. H - 1 non-clicks over the one-hot rows e_k = unit vector k (N = H): the non-zero
    columns of dh_p are the articles {c} + S_c."""
    emb = np.eye(H, dtype=f32)
    lists, clicks = [], []
    for i in range(n_imp):
        m = int(rng.integers(K + 2, H)) if i % 3 else int(rng.integers(2, K + 2))      # some with |N| <= K
        it = rng.choice(H, m, replace=False)
        c = np.zeros(m, np.uint8)
        c[rng.integers(0, m)] = 1
        lists.append(it)
        clicks.append(c)
    ip = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return emb, ip, np.concatenate(lists).astype(np.int32), np.concatenate(clicks)


def _support(row):
    return np.flatnonzero(row != 0)


@pytest.mark.parametrize('K', [1, 4, 32])
def test_drawn_sets_bit_for_bit(K):
    H, n_imp, seed, epoch = 64, 300, 77, 3
    rng = np.random.default_rng(K)
    emb, ip, items, clicked = _one_hot_case(rng, n_imp, H, K)
    ids = so.impression_ids(rng, n_imp)
    h = rng.standard_normal((n_imp, H)).astype(f32)
    pi = np.arange(n_imp + 1, dtype=np.int64)                   # impression q at position q
    dh, _ = _call(h, emb, pi, ip, items, clicked, ids, K, seed, epoch, 1.0, H)
    want = {}
    for q in range(n_imp):
        c = clicked[ip[q]:ip[q + 1]]
        (cp, S), = so.negative_sets(c, int(ids[q]), K, seed, epoch)
        it = items[ip[q]:ip[q + 1]]
        want[q] = np.sort(it[np.concatenate([[cp], S])])
        assert np.array_equal(_support(dh[q, :H]), want[q]), (q, _support(dh[q, :H]), want[q])
        assert dh[q, it[cp]] < 0 and (dh[q, it[S]] > 0).all()
    nn = np.diff(ip) - 1
    assert nn.min() <= K < nn.max()                              # both paths: S_c = N and K draws
    # a third of the same impressions in another batch, in reverse order at other positions (every other one empty): the same
    # sets and the same bits
    sel = np.arange(n_imp)[::-3]
    ip2 = np.concatenate([[0], np.cumsum(np.diff(ip)[sel])]).astype(np.int64)
    it2 = np.concatenate([items[ip[q]:ip[q + 1]] for q in sel]).astype(np.int32)
    c2 = np.concatenate([clicked[ip[q]:ip[q + 1]] for q in sel])
    pos2 = 5 + 2 * np.arange(sel.size)
    n_pos2 = int(pos2[-1]) + 4
    pi2 = np.searchsorted(pos2, np.arange(n_pos2 + 1)).astype(np.int64)
    h2 = np.zeros((n_pos2, H), f32)
    h2[pos2] = h[sel]
    dh2, _ = _call(h2, emb, pi2, ip2, it2, c2, ids[sel], K, seed, epoch, 1.0, H)
    for j, q in enumerate(sel):
        assert np.array_equal(dh2[pos2[j], :H].view(np.uint32), dh[q, :H].view(np.uint32)), q
    assert not dh2[np.setdiff1d(np.arange(n_pos2), pos2), :H].any()


# ---------------------------------------------------------------------------------------------------------------------------
# whole batches
# ---------------------------------------------------------------------------------------------------------------------------
def _data(U, H, N, max_len, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 4, U)
    lens[:6] = [1, 2, max_len, max_len + 3, 2 * max_len, 1]
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N, int(indptr[-1])).astype(np.int32)
    emb = (rng.standard_normal((N, H)) * 0.5).astype(f32)
    return indptr, items, emb


def _impressions(rng, indptr, N, per_user=3, shown=(2, 16)):
    user, time_, lists, clicks = [], [], [], []
    lens = np.diff(indptr)
    for u in range(lens.size):
        for _ in range(per_user):
            user.append(u)
            time_.append(rng.integers(0, lens[u] + 1))
            m = int(rng.integers(*shown))
            lists.append(rng.choice(N, m, replace=False))
            c = (rng.random(m) < 0.3).astype(np.uint8)
            c[0] = 1
            clicks.append(c)
    ip = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return {'user': np.array(user, np.int64), 'time': np.array(time_, np.int64), 'indptr': ip,
            'items': np.concatenate(lists).astype(np.int32), 'clicked': np.concatenate(clicks).astype(np.uint8)}


SENTINELS = {UserGRU: (('XP', 'HP', 'Hs', 'gates', 'dH', 'carry'), ('X_hl', 'dXP_hl', 'dHP_hl')),
             UserLSTM: (('XP', 'HP', 'Hs', 'Cs', 'gates', 'dH', 'carry', 'carry_c'), ('X_hl', 'dA_hl')),
             # O_hl keeps the ones column _buffers gave it: no kernel writes column H
             UserAttention: (('QKV', 'O', 'lse', 'M', 'Z', 'score', 'plse', 'Hs', 'dH', 'dM', 'dO', 'ws'),
                             ('X_hl', 'M_hl', 'dM_hl', 'dZ_hl', 'dQKV_hl'))}


@pytest.mark.parametrize('K', [4, 0])
@pytest.mark.parametrize('H,U,max_len', [(37, 200, 10), (500, 100, 8)])
@pytest.mark.parametrize('cell', [UserGRU, UserLSTM, UserAttention])
def test_batch_gradients_against_autograd(cell, H, U, max_len, K):
    N, seed, epoch = 900, 4, 2
    indptr, items, emb = _data(U, H, N, max_len, seed=H + 1)
    rng = np.random.default_rng(H + K)
    imp = check_impressions(_impressions(rng, indptr, N), N, 'test', indptr)
    use = usable_impressions(imp, indptr, max_len)
    m = cell(H, max_len=max_len, batch_users=U, seed=seed, impression_loss='softmax', impression_negatives=K)
    pk = Packed(indptr, items, np.arange(U), max_len)
    ib = ImpressionBatch(pk, imp, use, indptr)
    assert 0 < ib.n < ib.clicks
    b = m._buffers(pk.P, pk.B)
    f_keys, bf_keys = SENTINELS[cell]
    for k in f_keys:
        b[k].fill_(float('nan'))
    for k in bf_keys:
        for t in b[k]:
            t.view(torch.int16).fill_(0x7F7F)
    m.stats.zero_()
    m._forward_backward(pk, torch.from_numpy(emb).cuda(), epoch, 0, ib)
    torch.cuda.synchronize()
    loss = float(m.stats.item()) / ib.clicks
    seqs = [pk.items[[pk.position(i, t) for t in range(int(pk.L[i]))]] for i in range(pk.B)]
    row = {int(u): i for i, u in enumerate(pk.order)}
    samples, sampled = [], 0                                      # sampled: clicks whose impression has more than K non-clicks
    for q, iid in enumerate(ib.ids):
        u = int(imp['user'][iid])
        i = row[u]
        t = int(imp['time'][iid]) - 1 - (int(indptr[u + 1] - indptr[u]) - int(pk.L[i]))
        a, z = ib.indptr[q], ib.indptr[q + 1]
        for c, S in so.negative_sets(ib.clicked[a:z], int(iid), K, seed, epoch):
            sampled += int(0 < K < (ib.clicked[a:z] == 0).sum())
            samples.append((i, t, a + c, a + np.asarray(S, np.int64)))
    assert len(samples) == ib.clicks and (sampled > 20 or K == 0)
    if cell is UserAttention:
        o_loss, o_g = ao.softmax_loss_and_grads({k: v.double().numpy() for k, v in m.state_dict().items()}, seqs, emb,
                                                [(i, t, ib.items[c], ib.items[S]) for i, t, c, S in samples], m.heads)
        assert rel_err(loss, o_loss) < 1e-4, (loss, o_loss)
        A = m.attention_dim
        g = {x: m._theta(x, m.grad).cpu().double().numpy() for x in ('in', 'out', 'pool', 'query')}
        got = {'self_attn.in_proj_weight': g['in'][:, :H], 'self_attn.in_proj_bias': g['in'][:, H],
               'self_attn.out_proj.weight': g['out'][:, :H], 'self_attn.out_proj.bias': g['out'][:, H],
               'pool.weight': g['pool'][:, :H], 'pool.bias': g['pool'][:, H], 'pool.query': g['query'][:A]}
        for k in ATTENTION_NAMES:
            assert rel_err(got[k], o_g[k]) < 1e-4, (k, rel_err(got[k], o_g[k]))
        return
    params = {k: torch.tensor(v.double().numpy(), requires_grad=True) for k, v in m.state_dict().items()}
    hs = (gru_states if cell is UserGRU else lstm_states)(params, seqs, emb)
    E = torch.as_tensor(emb.astype(np.float64))
    terms = []
    for i, t, c, S in samples:
        s = E[torch.from_numpy(ib.items[np.concatenate([[c], S])].astype(np.int64))] @ hs[i][t]
        terms.append(torch.logsumexp(s, 0) - s[0])
    o_loss = torch.stack(terms).mean()
    o_loss.backward()
    o_loss = float(o_loss.detach())
    assert rel_err(loss, o_loss) < 1e-4, (loss, o_loss)
    G, g = m.GATES, m.grad.cpu().double().numpy()
    hh, ih = g[:m.nW].reshape(G * H, H + 1), g[m.nW:].reshape(G * H, H + 1)
    got = {'weight_ih_l0': ih[:, :H], 'weight_hh_l0': hh[:, :H], 'bias_ih_l0': ih[:, H], 'bias_hh_l0': hh[:, H]}
    for k in NAMES:
        assert rel_err(got[k], params[k].grad.numpy()) < 1e-4, (k, rel_err(got[k], params[k].grad.numpy()))


def test_k1_one_pair_fit_equals_pairwise_fit():
    """On one-click / one-non-click impressions the K = 1 softmax term is softplus(s_n - s_c), the pairwise term, and both
    losses average over the same samples: one epoch of each fit agrees."""
    H, U, N, max_len = 37, 500, 800, 12
    indptr, items, emb = _data(U, H, N, max_len, seed=3)
    rng = np.random.default_rng(8)
    lens = np.diff(indptr)
    user = np.repeat(np.arange(U), 2)
    time_ = np.array([rng.integers(1, lens[u] + 1) for u in user])
    lists = np.stack([rng.choice(N, 2, replace=False) for _ in user])
    imp = {'user': user, 'time': time_, 'indptr': np.arange(0, 2 * user.size + 1, 2), 'items': lists.reshape(-1).astype(np.int32),
           'clicked': np.tile(np.array([1, 0], np.uint8), user.size)}
    kw = dict(max_len=max_len, batch_users=128, num_epochs=1, seed=5, learning_rate=3e-3)
    a = UserGRU(H, **kw).fit((indptr, items), emb, impressions=imp)
    b = UserGRU(H, impression_loss='softmax', impression_negatives=1, **kw).fit((indptr, items), emb, impressions=imp)
    assert b.impression_counts == dict(a.impression_counts, clicks=a.impression_counts['used']) and a.impression_counts['used'] > 300
    assert abs(a.train_loss[0] - b.train_loss[0]) <= 1e-6 * abs(a.train_loss[0]), (a.train_loss, b.train_loss)
    sa, sb = a.state_dict(), b.state_dict()
    for k in NAMES:
        assert rel_err(sb[k].numpy(), sa[k].numpy()) < 1e-5, (k, rel_err(sb[k].numpy(), sa[k].numpy()))


# test-impression AUC measured on an H100 80GB HBM3 at 700 W: softmax K = 4 0.9548, pairwise 0.9547, mean profile 0.7813 (DESIGN
# 4.16); the asserted margin is half the gap to the mean profile.  The pairwise number is printed beside it, not compared.
LEARNING_MARGIN = 0.087


def test_learning_beats_mean_profile():
    from dae_rnn_news_recommendation_b200.synth import make_impressions, make_sequences
    from dae_rnn_news_recommendation_b200.user_model import prefix_histories
    from test_gpu_user_gru import _clustered
    N, H = 3000, 64
    labels, emb = _clustered(N, H, 8, 11)
    indptr, items, targets = make_sequences(8000, labels, mean_len=20, session_len=5, seed=12)
    train, test = make_impressions(indptr, items, labels, targets, shown=20, seed=13)
    kw = dict(max_len=50, batch_users=512, num_epochs=8, learning_rate=3e-3, seed=0)
    g_sm = UserGRU(H, impression_loss='softmax', impression_negatives=4, **kw).fit((indptr, items), emb, impressions=train)
    g_pw = UserGRU(H, **kw).fit((indptr, items), emb, impressions=train)
    auc = {}
    for name, g in (('softmax K=4', g_sm), ('pairwise', g_pw)):
        auc[name] = helpers.impression_metrics(g.impression_states((indptr, items), emb, test), emb, test)['auc']
    prof = helpers.user_profiles(prefix_histories((indptr, items), test, N), emb)
    auc['mean profile'] = helpers.impression_metrics(prof, emb, test, metric='cosine')['auc']
    print('test-impression AUC: %s; softmax train loss %s; %s' % (
        ', '.join('%s %.4f' % kv for kv in auc.items()), ['%.4f' % x for x in g_sm.train_loss], g_sm.impression_counts))
    assert g_sm.train_loss[-1] < g_sm.train_loss[0]
    assert auc['softmax K=4'] - auc['mean profile'] > LEARNING_MARGIN, auc


def test_cli_softmax(capsys, tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.synth import make_impressions, make_sequences
    argv = ['--model_name', 'synsm', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--top_k', '5']
    trX, _, trL, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    indptr, items, targets = make_sequences(300, trL, mean_len=8, seed=4)
    train, test = make_impressions(indptr, items, trL, targets, shown=10, seed=5)
    np.savez(tmp_path / 's.npz', indptr=indptr, items=items, targets=targets)
    np.savez(tmp_path / 'tr.npz', **train)
    np.savez(tmp_path / 'te.npz', **test)
    model = cli.main(argv + ['--user_sequences', str(tmp_path / 's.npz'), '--user_epochs', '2', '--user_impressions',
                             str(tmp_path / 'tr.npz'), '--user_test_impressions', str(tmp_path / 'te.npz'),
                             '--user_impression_loss', 'softmax', '--user_negatives', '4'])
    printed = capsys.readouterr().out
    assert 'impression loss: softmax over each click and at most 4 of its non-clicks' in printed
    assert 'test impressions (GRU): AUC' in printed
    assert np.isfinite(model.evaluation['user_gru_train_loss'])
    for who in ('gru', 'mean'):
        for k in ('auc', 'mrr', 'ndcg5', 'ndcg10'):
            assert 0.0 <= model.evaluation['user_%s_imp_%s' % (who, k)] <= 1.0
