"""Every kernel call of the LSTM and attention user encoders' training batches, optimizer steps, transform and impression_states
against the fp64 reference of its own recorded inputs (encoder_stages.Recorder / check_log), and the data flow between the calls:
each stage reads what the stage before it wrote, bit for bit, with the ones columns, leading dimensions, offsets and accumulate
flags of user_model.py.  Kernel-filled buffers start as sentinels (NaN in fp32, 0x7F7F in bf16, -7 in neg) after a smaller batch
has grown them; the columns _buffers initialises and no kernel writes (the ones columns and the padding of O_hl and Hp_hl) are
left as _buffers leaves them, so a ones column lost on regrowth shows in the recorded GEMM operands."""
import numpy as np
import pytest
import torch

import gru_kernel_oracle as go
from encoder_stages import ONE_HI, Recorder, assert_bits, bf16_bits, check_log, worst

from dae_rnn_news_recommendation_b200 import user_model
from dae_rnn_news_recommendation_b200.user_model import (ImpressionBatch, Packed, UserAttention, UserGRU, UserLSTM, check_impressions,
                                                         usable_impressions)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF16_SENT = 0x7F7F
N_ITEMS = 900
f32 = np.float32


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _bits(t):
    torch.cuda.synchronize()
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def _f32_bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _data(U, H, max_len, seed, head):
    """Reading sequences of U users: the first ones have the lengths `head`, the others 1 to 12 reads."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 13, U)
    lens[:len(head)] = head
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N_ITEMS, int(indptr[-1])).astype(np.int32)
    emb = (rng.standard_normal((N_ITEMS, H)) * 0.5).astype(f32)
    return indptr, items, emb


def _impressions(rng, indptr, per_user=2, shown=(2, 14)):
    """per_user impressions per user at random times in [0, len], each with a click first."""
    user, time_, lists, clicks = [], [], [], []
    for u, n in enumerate(np.diff(indptr)):
        for _ in range(per_user):
            user.append(u)
            time_.append(rng.integers(0, n + 1))
            m = int(rng.integers(*shown))
            lists.append(rng.choice(N_ITEMS, m, replace=False))
            c = (rng.random(m) < 0.3).astype(np.uint8)
            c[0] = 1
            clicks.append(c)
    ip = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return {'user': np.array(user, np.int64), 'time': np.array(time_, np.int64), 'indptr': ip,
            'items': np.concatenate(lists).astype(np.int32), 'clicked': np.concatenate(clicks).astype(np.uint8)}


# the kernel-filled buffers of each encoder: fp32, bf16 pairs filled whole, bf16 pairs whose columns [0, H) only a kernel writes
SENTINELS = {UserLSTM: (('XP', 'HP', 'Hs', 'Cs', 'gates', 'dH', 'carry', 'carry_c'), ('X_hl', 'dA_hl'), ('Hp_hl',)),
             UserAttention: (('QKV', 'O', 'lse', 'M', 'Z', 'score', 'plse', 'Hs', 'dH', 'dM', 'dO', 'ws'),
                             ('X_hl', 'M_hl', 'dM_hl', 'dZ_hl', 'dQKV_hl'), ('O_hl',))}


def _prepare(cls, H, U, max_len, loss, K, head, seed, **kw):
    """A model whose buffers held a smaller batch and were then grown for this one and filled with sentinels: (m, pk, ib, emb,
    emb_d)."""
    indptr, items, emb = _data(U, H, max_len, seed, head)
    imp_loss = 'softmax' if loss == 'softmax' else 'pairwise'
    m = cls(H, max_len=max_len, batch_users=U, seed=3, learning_rate=1e-2, impression_loss=imp_loss, impression_negatives=K, **kw)
    emb_d = _dev(emb)
    m._forward_backward(Packed(indptr, items, np.arange(40), max_len), emb_d, 0, 0)
    m._optimizer_step()
    pk = Packed(indptr, items, np.arange(U), max_len)
    ib = None
    if loss != 'random':
        imp = check_impressions(_impressions(np.random.default_rng(seed + 1), indptr), N_ITEMS, 'test', indptr)
        ib = ImpressionBatch(pk, imp, usable_impressions(imp, indptr, max_len), indptr)
        assert ib.n > 20
    b = m._buffers(pk.P, pk.B)
    f_keys, bf_keys, cols_keys = SENTINELS[cls]
    for k in f_keys:
        b[k].fill_(float('nan'))
    b['neg'].fill_(-7)
    for k in bf_keys:
        for t in b[k]:
            t.view(torch.int16).fill_(BF16_SENT)
    for k in cols_keys:
        for t in b[k]:
            t[:, :H].view(torch.int16).fill_(BF16_SENT)
    return m, pk, ib, emb, emb_d


def _ones_operand(tag, hi, lo, H, want_hi=None, want_lo=None):
    """A recorded [v | 1 | 0 ...] GEMM operand: columns [0, H) are want_hi / want_lo (bits; None: 0), column H is 1 (hi 1, lo 0),
    the padding 0."""
    n = hi.shape[0]
    assert_bits('%s: columns [0, H) (hi)' % tag, hi[:, :H], np.zeros((n, H), np.uint16) if want_hi is None else want_hi)
    assert_bits('%s: columns [0, H) (lo)' % tag, lo[:, :H], np.zeros((n, H), np.uint16) if want_lo is None else want_lo)
    assert (hi[:, H] == ONE_HI).all() and (lo[:, H] == 0).all(), '%s: column H is not 1 in %d rows' % (
        tag, int(((hi[:, H] != ONE_HI) | (lo[:, H] != 0)).sum()))
    assert (hi[:, H + 1:] == 0).all() and (lo[:, H + 1:] == 0).all(), '%s: padding not 0' % tag


def _product_check(tag, a, pre, post, add=None):
    """C[:M, :N] of a recorded GEMM against A.B^T alone (add: plus this fp32 array), whatever its accumulate flag."""
    M, N, K = a.M, a.N, a.K
    A = pre['a'].T[:M, :K] if a.a_mn_major else pre['a'][:M, :K]
    B = pre['b'].T[:N, :K] if a.b_mn_major else pre['b'][:N, :K]
    want, s = go.gemm_nt(A, B)
    if add is not None:
        want, s = want + add, s + np.abs(add)
    go.check(tag, post['c'][:, :N], want, s, go.C_BF16X3)


def _bias_check(tag, a, pre, post, H):
    """A weight GEMM [dW | db] = dA^T.[v | 1]: the bias column is the position sum of dA."""
    dA = pre['a'][:a.K, :a.M]
    go.check(tag + ' bias column', post['c'][:, H], dA.sum(0), np.abs(dA).sum(0), go.C_BF16X3)


def _same(tag, got, want):
    assert_bits(tag, _f32_bits(got), _f32_bits(want))


# ---------------------------------------------------------------------------------------------------------------------------
# UserLSTM: a training batch, an Adam step and a momentum step
# ---------------------------------------------------------------------------------------------------------------------------
LOSSES = [('random', 0), ('pairwise', 0), ('softmax', 4), ('softmax', 0)]    # (loss, impression_negatives)
LOSS_CALL = {'random': 'dae_seq_rank_loss', 'pairwise': 'dae_impression_rank_loss', 'softmax': 'dae_impression_softmax_loss'}


@pytest.mark.parametrize('loss,K,H,U,max_len', [(loss, K, 37, 2600, 12) for loss, K in LOSSES] + [('random', 0, 7, 200, 9)])
def test_lstm_training_batch_every_stage(loss, K, H, U, max_len, monkeypatch):
    m, pk, ib, emb, emb_d = _prepare(UserLSTM, H, U, max_len, loss, K, [1, 2, max_len, max_len + 3, 2 * max_len, 1], seed=H + U)
    if U > 2000:
        assert pk.P > 16896                                            # more positions than the loss kernel's grid covers
    assert (pk.L == 1).any()
    b, T, P, G = m._buf, len(pk.n), pk.P, 4 * H
    rec = Recorder(user_model.call)
    monkeypatch.setattr(user_model, 'call', rec)
    m.stats.zero_()
    m._forward_backward(pk, emb_d, 5, 3, ib)
    m._optimizer_step()
    tag = 'lstm %s K=%d H=%d' % (loss, K, H)
    by = check_log(rec.log, emb, H, tag)
    names = [c[0] for c in rec.log]
    want = ((['dae_seq_negatives'] if loss == 'random' else []) + ['dae_gather_split_bf16', 'dae_split_bf16', 'dae_gemm_bf16x3'] +
            ['dae_gemm_bf16x3', 'dae_lstm_cell_fwd'] * T + [LOSS_CALL[loss]] +
            [x for t in range(T - 1, -1, -1) for x in (['dae_lstm_cell_bwd'] + (['dae_gemm_bf16x3'] if t else []))] +
            ['dae_gemm_bf16x3'] * 2 + ['dae_optimizer_step'])
    assert names == want, (tag, names)
    gemms = by['dae_gemm_bf16x3']
    xp_g, hp_g, carry_g, w_g = gemms[0], gemms[1:1 + T], gemms[1 + T:T + T], gemms[-2:]
    fwd, bwd = by['dae_lstm_cell_fwd'], by['dae_lstm_cell_bwd'][::-1]          # bwd by step
    n = [int(x) for x in pk.n]
    off = [int(x) for x in pk.off]
    # forward: the input projection of every position, then per step [h_{t-1} | 1].W~_hh^T and the cell
    ga, gpre, gpost = by['dae_gather_split_bf16'][0]
    assert np.array_equal(gpre['rows'], pk.items) and ga.ones_col == H
    assert xp_g[0].M == P and xp_g[0].K == H + 1 and xp_g[0].N == G
    assert_bits(tag + ' XP GEMM reads [X | 1]', xp_g[1]['a_hi'][:P], gpost['hi'])
    for t in range(T):
        a, pre, post = hp_g[t]
        st = '%s step %d HP GEMM [h_{t-1} | 1].W~_hh^T' % (tag, t)
        assert a.M == n[t] and a.K == H + 1 and a.N == G and a.C == b['HP'].data_ptr(), st
        if t:
            h_prev = fwd[t - 1][2]['h'][:n[t], :H]
            w_hi, w_lo = bf16_bits(h_prev)
            _ones_operand(st, pre['a_hi'], pre['a_lo'], H, w_hi, w_lo)
            assert_bits(st + ' reads the cell\'s own split', pre['a_hi'][:, :H], fwd[t - 1][2]['h_hi'][:n[t], :H])
        else:
            _ones_operand(st, pre['a_hi'], pre['a_lo'], H)
        ca, cpre, cpost = fwd[t]
        ct = '%s step %d lstm cell fwd' % (tag, t)
        assert ca.n == n[t] and ca.n_split == (n[t + 1] if t + 1 < T else 0), ct
        _same(ct + ' reads XP of its positions', cpre['xp'][:, :G], xp_g[2]['c'][off[t]:off[t] + n[t], :G])
        _same(ct + ' reads HP', cpre['hp'][:, :G], post['c'][:n[t], :G])
        if t:
            _same(ct + ' reads c_{t-1}', cpre['c_prev'][:, :H], fwd[t - 1][2]['c'][:n[t], :H])
        else:
            assert cpre['c_prev'] is None, ct
    # the loss reads the states of every position, the backward its dH rows
    _, lpre, lpost = by[LOSS_CALL[loss]][0]
    Hs = np.concatenate([fwd[t][2]['h'][:, :H] for t in range(T)])
    _same(tag + ' loss reads Hs', lpre['h'][:, :H], Hs)
    for t in range(T - 1, -1, -1):
        a, pre, post = bwd[t]
        ct = '%s step %d lstm cell bwd' % (tag, t)
        assert a.n == n[t], ct
        _same(ct + ' reads dH', pre['dh_in'][:, :H], lpost['dh'][off[t]:off[t] + n[t], :H])
        _same(ct + ' reads c_t', pre['c'][:, :H], fwd[t][2]['c'][:, :H])
        _same(ct + ' reads its gates', pre['gates'][:, :G], fwd[t][2]['gates'][:, :G])
        if t + 1 < T:
            # the carry GEMM of step t + 1 STORED dh_t = dA_{t+1}.W_hh in rows [0, n_{t+1}): nothing was added to it
            ga, gpre, gpost = carry_g[T - 2 - t]
            gt = '%s carry GEMM dh_%d = dA_%d.W_hh' % (tag, t, t + 1)
            assert ga.C == b['carry'].data_ptr() and ga.M == n[t + 1] and ga.K == G and ga.N == H and ga.b_mn_major == 1, gt
            assert ga.accumulate == 0, gt + ': accumulates onto the carry the cell has already read'
            assert_bits(gt + ' reads dA_%d' % (t + 1), gpre['a_hi'][:, :G], bwd[t + 1][2]['da_hi'][:, :G])
            _product_check(gt, ga, gpre, gpost)
            _same(ct + ' reads the stored carry', pre['carry_h'][:n[t + 1], :H], gpost['c'][:, :H])
    # the two weight GEMMs: K = P positions, stored into grad[:nW] and grad[nW:]
    for (a, pre, post), (g0, Bk) in zip(w_g, ((0, 'Hp_hl'), (m.nW, 'X_hl'))):
        wt = '%s weight GEMM into grad[%d:]' % (tag, g0)
        assert a.K == P and a.M == G and a.N == H + 1 and a.ldc == H + 1 and a.accumulate == 0, wt
        assert a.C == m.grad.data_ptr() + 4 * g0 and a.b_hi == b[Bk][0].data_ptr(), wt
        _bias_check(wt, a, pre, post, H)
    _ones_operand(tag + ' [h_prev | 1] of every position', w_g[0][1]['b_hi'][:P], w_g[0][1]['b_lo'][:P], H,
                  *bf16_bits(np.concatenate([np.zeros((n[0], H), f32)] + [fwd[t][2]['h'][:n[t + 1], :H] for t in range(T - 1)])))
    # after the Adam step the recurrent GEMM's bf16 copy of W_hh is the split of the new theta_hh
    oa = by['dae_optimizer_step'][0][0]
    assert oa.opt == 3 and oa.n == 2 * m.nW and oa.w_hi == m.W_hl['hh'][0].data_ptr() and oa.F == G and oa.H == H + 1
    hi, lo = m.W_hl['hh']
    w_hi, w_lo = bf16_bits(m._theta('hh').cpu().numpy())
    assert_bits(tag + ' W_hl[hh] after the step', _bits(hi)[:, :H + 1], w_hi)
    assert_bits(tag + ' W_hl[hh] lo after the step', _bits(lo)[:, :H + 1], w_lo)
    # a momentum step on the same gradient, from the Adam step's theta: the rule is checked against its own recorded inputs
    k0 = len(rec.log)
    m.opt = 'momentum'
    m._optimizer_step()
    check_log(rec.log[k0:], emb, H, tag)
    assert rec.log[k0][1].opt == 2
    print(tag, worst(tag))


# ---------------------------------------------------------------------------------------------------------------------------
# UserAttention: a training batch, an Adam step and the next batch's operand refresh
# ---------------------------------------------------------------------------------------------------------------------------
ATTENTION_SHAPES = [(37, 1, 200, 1100), (500, 20, 16, 60), (64, 4, 50, 300)]   # work items (user, head, 32-read tile) past 3 passes


@pytest.mark.parametrize('H,heads,A,U', ATTENTION_SHAPES)
@pytest.mark.parametrize('loss,K', [('random', 0), ('pairwise', 0), ('softmax', 4)])
def test_attention_training_batch_every_stage(loss, K, H, heads, A, U, monkeypatch):
    max_len = 70
    m, pk, ib, emb, emb_d = _prepare(UserAttention, H, U, max_len, loss, K, [1, 31, 32, 33, 70, 2, 73, 140, 1], seed=H + U,
                                     heads=heads, attention_dim=A)
    assert {1, 2, 31, 32, 33, 70} <= set(pk.L) and (pk.L == 70).sum() == 3
    b, P, ldx = m._buf, pk.P, m.ldx
    rec = Recorder(user_model.call)
    monkeypatch.setattr(user_model, 'call', rec)
    m.stats.zero_()
    m._forward_backward(pk, emb_d, 5, 3, ib)
    m._optimizer_step()
    tag = 'attn %s H=%d heads=%d' % (loss, H, heads)
    check_log(rec.log, emb, H, tag)
    names = [c[0] for c in rec.log]
    G = 'dae_gemm_bf16x3'
    want = (['dae_split_bf16'] * 3 + (['dae_seq_negatives'] if loss == 'random' else []) +
            ['dae_gather_split_bf16', G, 'dae_seq_attention_fwd', G, 'dae_split_bf16', G, 'dae_seq_pool_fwd', LOSS_CALL[loss],
             'dae_seq_pool_bwd', G, 'dae_split_bf16', G, 'dae_seq_attention_bwd', G, G, G, 'dae_optimizer_step'])
    assert names == want, (tag, names)
    calls = [c for c in rec.log if c[0] != 'dae_seq_negatives']
    (s_in, s_out, s_pool, gather, g_qkv, att_f, g_out, s_m, g_z, pool_f, loss_c, pool_b, g_dm, s_dm, g_do, att_b, w_in, w_out, w_pool,
     opt) = [(c[1], c[2], c[3]) for c in calls]
    theta0 = opt[1]['theta']
    # the bf16 operands of W~_in, W~_out and W~_a: splits of theta's slices, no ones column
    for (a, pre, post), g in zip((s_in, s_out, s_pool), ('in', 'out', 'pool')):
        assert a.src == m._theta(g).data_ptr() and a.rows == m._rows[g] and a.cols == H + 1 and a.ones_col == -1, (tag, g)
        assert a.hi == m.W_hl[g][0].data_ptr() and a.ld_dst == ldx, (tag, g)
    # gather -> QKV GEMM -> attention forward -> [O | 1].W~_out^T
    a, pre, post = gather
    assert np.array_equal(pre['rows'], pk.items) and a.ones_col == H and a.hi == b['X_hl'][0].data_ptr(), tag
    a, pre, post = g_qkv
    st = tag + ' QKV GEMM [X | 1].W~_in^T'
    assert a.M == P and a.N == 3 * H and a.K == H + 1 and a.C == b['QKV'].data_ptr() and a.ldc == 3 * H, st
    assert_bits(st + ' A', pre['a_hi'], gather[2]['hi'])
    assert_bits(st + ' B', pre['b_hi'][:, :H + 1], s_in[2]['hi'][:, :H + 1])
    a, pre, post = att_f
    ct = tag + ' attention fwd'
    assert a.B == pk.B and a.heads == heads and a.o_hi == b['O_hl'][0].data_ptr() and a.ld_split == ldx, ct
    assert np.array_equal(pre['off'], pk.off) and np.array_equal(pre['lens'], pk.L), ct
    _same(ct + ' reads QKV', pre['qkv'][:, :3 * H], g_qkv[2]['c'][:, :3 * H])
    a, pre, post = g_out
    st = tag + ' out GEMM M = [O | 1].W~_out^T'
    assert a.M == P and a.N == H and a.K == H + 1 and a.C == b['M'].data_ptr(), st
    _ones_operand(st + ' A', pre['a_hi'][:P], pre['a_lo'][:P], H, att_f[2]['o_hi'][:, :H], att_f[2]['o_lo'][:, :H])
    assert_bits(st + ' B', pre['b_hi'][:, :H + 1], s_out[2]['hi'][:, :H + 1])
    M = post['c'][:, :H]
    # M split with its ones column -> [M | 1].W~_a^T -> pooling
    a, pre, post = s_m
    assert a.src == b['M'].data_ptr() and a.ones_col == H and a.cols == H and a.rows == P, tag + ' M split'
    _same(tag + ' M split reads M', pre['src'][:, :H], M)
    a, pre, post = g_z
    st = tag + ' Z GEMM [M | 1].W~_a^T'
    assert a.M == P and a.N == A and a.K == H + 1 and a.C == b['Z'].data_ptr(), st
    _ones_operand(st + ' A', pre['a_hi'][:P], pre['a_lo'][:P], H, s_m[2]['hi'][:, :H], s_m[2]['lo'][:, :H])
    Z = post['c'][:, :A]
    a, pre, post = pool_f
    ct = tag + ' pool fwd'
    _same(ct + ' reads Z', pre['z'][:, :A], Z)
    _same(ct + ' reads M', pre['m'][:, :H], M)
    _same(ct + ' reads q', pre['q'], theta0[m._off['query']:m._off['query'] + A])
    assert a.u == b['Hs'].data_ptr(), ct
    # loss -> pooling backward: dM's value path, dZ, and dq straight into grad's query slice
    _same(tag + ' loss reads Hs', loss_c[1]['h'][:, :H], pool_f[2]['u'][:, :H])
    a, pre, post = pool_b
    ct = tag + ' pool bwd'
    _same(ct + ' reads dH', pre['du'][:, :H], loss_c[2]['dh'][:, :H])
    _same(ct + ' reads u', pre['u'][:, :H], pool_f[2]['u'][:, :H])
    _same(ct + ' reads the scores', pre['score'], pool_f[2]['score'])
    _same(ct + ' reads the prefix lse', pre['plse'], pool_f[2]['plse'])
    assert a.dq == m._theta('query', m.grad).data_ptr() and a.dm == b['dM'].data_ptr() and a.dz_hi == b['dZ_hl'][0].data_ptr(), ct
    # dM += dZ.W_a: the pooling backward's value path plus the scorer path
    a, pre, post = g_dm
    st = tag + ' GEMM dM += dZ.W_a'
    assert a.C == b['dM'].data_ptr() and a.M == P and a.N == H and a.K == A and a.b_mn_major == 1, st
    _same(st + ': C before the call is the value path', pre['c'][:, :H], pool_b[2]['dm'][:, :H])
    assert_bits(st + ' A = dZ', pre['a_hi'][:, :A], pool_b[2]['dz_hi'][:, :A])
    _product_check(st + ' (value path + dZ.W_a)', a, pre, post, add=pre['c'][:, :H].astype(np.float64))
    dM = post['c'][:, :H]
    # dM split without a ones column -> dO = dM.W_out (K = H) -> attention backward
    a, pre, post = s_dm
    assert a.src == b['dM'].data_ptr() and a.ones_col == -1, tag + ' dM split'
    _same(tag + ' dM split reads dM', pre['src'][:, :H], dM)
    a, pre, post = g_do
    st = tag + ' GEMM dO = dM.W_out'
    assert a.K == H and a.M == P and a.N == H and a.b_mn_major == 1 and a.C == b['dO'].data_ptr(), st
    assert_bits(st + ' A = dM', pre['a_hi'], s_dm[2]['hi'])
    a, pre, post = att_b
    ct = tag + ' attention bwd'
    _same(ct + ' reads QKV', pre['qkv'][:, :3 * H], g_qkv[2]['c'][:, :3 * H])
    _same(ct + ' reads O', pre['o'][:, :H], att_f[2]['o'][:, :H])
    _same(ct + ' reads lse', pre['lse'][:, :heads], att_f[2]['lse'][:, :heads])
    _same(ct + ' reads dO', pre['dout'][:, :H], g_do[2]['c'][:, :H])
    # the three weight GEMMs [dW | db] = dA^T.[v | 1] over the P positions, each stored into its slice of grad
    for (a, pre, post), g, dA, v, rows in ((w_in, 'in', att_b[2]['dqkv_hi'][:, :3 * H], gather[2]['hi'], 3 * H),
                                          (w_out, 'out', s_dm[2]['hi'][:, :H], att_f[2]['o_hi'][:, :H], H),
                                          (w_pool, 'pool', pool_b[2]['dz_hi'][:, :A], s_m[2]['hi'][:, :H], A)):
        wt = '%s weight GEMM [dW_%s | db_%s]' % (tag, g, g)
        assert a.K == P and a.M == rows and a.N == H + 1 and a.accumulate == 0 and a.C == m._theta(g, m.grad).data_ptr(), wt
        assert_bits(wt + ' A', pre['a_hi'][:P, :rows], dA)
        assert_bits(wt + ' B', pre['b_hi'][:P, :H], v[:, :H])
        assert (pre['b_hi'][:P, H] == ONE_HI).all() and (pre['b_lo'][:P, H] == 0).all(), wt + ': B column H is not 1'
        _bias_check(wt, a, pre, post, H)
    # after the Adam step the next batch's refresh (the first thing _forward_backward does) splits the new theta, bit for bit
    k0 = len(rec.log)
    m._refresh()
    theta1 = opt[2]['theta']
    _same(tag + ' theta after the step', m.theta.cpu().numpy(), theta1)
    refresh = rec.log[k0:k0 + 3]
    check_log(refresh, emb, H, tag + ' refresh')
    for (name, a, pre, post), g in zip(refresh, ('in', 'out', 'pool')):
        o = m._off[g]
        _same('%s refresh of W~_%s reads the new theta' % (tag, g), pre['src'][:, :H + 1],
              theta1[o:o + m._rows[g] * (H + 1)].reshape(-1, H + 1))
    print(tag, worst(tag))


# ---------------------------------------------------------------------------------------------------------------------------
# inference: UserLSTM.transform step by step; impression_states' captured rows
# ---------------------------------------------------------------------------------------------------------------------------
def test_lstm_transform_every_step(monkeypatch):
    H, U, max_len, B = 37, 333, 12, 150
    indptr, items, emb = _data(U, H, max_len, 9, [1, 2, max_len, max_len + 3, 2 * max_len, 1])
    m = UserLSTM(H, max_len=max_len, batch_users=B, seed=4)
    rec = Recorder(user_model.call)
    monkeypatch.setattr(user_model, 'call', rec)
    out = m.transform((indptr, items), emb)
    tag = 'lstm transform'
    check_log(rec.log, emb, H, tag)
    assert [c[0] for c in rec.log[:2]] == ['dae_split_bf16'] * 2
    steps = rec.log[2:]
    k = 0
    h_ptr = None
    for u0 in range(0, U, B):
        pk = Packed(indptr, items, np.arange(u0, min(U, u0 + B)), max_len)
        prev = None
        for t in range(len(pk.n)):
            n = int(pk.n[t])
            (g_name, ga, gpre, gpost), (x_name, xa, xpre, xpost), (h_name, ha, hpre, hpost), (c_name, ca, cpre, cpost) = steps[k:k + 4]
            k += 4
            st = '%s batch %d step %d' % (tag, u0, t)
            assert (g_name, x_name, h_name, c_name) == ('dae_gather_split_bf16', 'dae_gemm_bf16x3', 'dae_gemm_bf16x3', 'dae_lstm_cell_fwd')
            assert np.array_equal(gpre['rows'], pk.items[int(pk.off[t]):int(pk.off[t]) + n]), st
            assert ga.n_rows == xa.M == ha.M == ca.n == ca.n_split == n, st
            # c and h in place, no gates
            assert ca.c_prev == ca.c_out and ca.ld_cprev == ca.ld_c and ca.gates is None, st
            h_ptr = h_ptr or ca.h_out
            assert ca.h_out == h_ptr and ha.a_hi == ca.h_hi, st
            _same(st + ' cell reads XP', cpre['xp'][:, :4 * H], xpost['c'][:, :4 * H])
            _same(st + ' cell reads HP', cpre['hp'][:, :4 * H], hpost['c'][:, :4 * H])
            if prev is None:
                assert (cpre['c_prev'][:, :H] == 0).all(), st
                _ones_operand(st + ' HP GEMM [h | 1]', hpre['a_hi'][:n], hpre['a_lo'][:n], H)
            else:
                _same(st + ' cell reads c in place', cpre['c_prev'][:, :H], prev['c'][:n, :H])
                _ones_operand(st + ' HP GEMM [h | 1]', hpre['a_hi'][:n], hpre['a_lo'][:n], H, *bf16_bits(prev['h'][:n, :H]))
                assert n <= prev['h'].shape[0], st
            prev = cpost
            if t:
                assert n <= int(pk.n[t - 1]), st
        # each user's vector is its row of h after its last step
        last = {t: steps[k - 4 * (len(pk.n) - t) + 3][3]['h'] for t in range(len(pk.n))}
        for i, u in enumerate(pk.order):
            _same('%s user %d' % (tag, u), out[u], last[int(pk.L[i]) - 1][i, :H])
    assert k == len(steps)
    print(tag, worst(tag))


@pytest.mark.parametrize('cls', [UserGRU, UserLSTM, UserAttention])
def test_impression_states_captured_rows(cls, monkeypatch):
    H, U, max_len = 32, 260, 10
    indptr, items, emb = _data(U, H, max_len, 21, [1, 2, 10, 13, 20, 31, 25, 40, 17, 22, 33, 50])
    kw = dict(heads=4, attention_dim=24) if cls is UserAttention else {}
    m = cls(H, max_len=max_len, batch_users=100, seed=5, **kw)
    imp = _impressions(np.random.default_rng(22), indptr, per_user=3)
    lens = np.diff(indptr)
    imp['time'][:6] = 0
    imp['time'][6:12] = lens[2:4].repeat(3)                     # time = len, at and beyond max_len
    rec = Recorder(user_model.call)
    monkeypatch.setattr(user_model, 'call', rec)
    runs = []
    real = m._run_capture

    def capture(pk, emb_, s, cap_step, cap_row, cap_imp, out_):
        runs.append((len(rec.log), pk, np.array(cap_step), np.array(cap_row), np.array(cap_imp)))
        return real(pk, emb_, s, cap_step, cap_row, cap_imp, out_)
    monkeypatch.setattr(m, '_run_capture', capture)
    out = m.impression_states((indptr, items), emb, imp)
    tag = '%s impression_states' % cls.__name__
    check_log(rec.log, emb, H, tag)
    t_imp = imp['time']
    assert (t_imp == 0).sum() >= 6 and (t_imp > max_len).sum() > 10 and len(runs) > 1
    assert not out[t_imp == 0].any()
    captured = np.concatenate([r[4] for r in runs])
    assert np.array_equal(np.sort(captured), np.flatnonzero(t_imp > 0))
    ends = [r[0] for r in runs[1:]] + [len(rec.log)]
    for (k0, pk, cap_step, cap_row, cap_imp), k1 in zip(runs, ends):
        calls = rec.log[k0:k1]
        gathers = [c for c in calls if c[0] == 'dae_gather_split_bf16']
        if cls is UserAttention:
            read = gathers[0][2]['rows']
            states = [c for c in calls if c[0] == 'dae_seq_pool_fwd'][0][3]['u']
            pos = pk.off[cap_step] + cap_row                        # the state after read cap_step of row cap_row
            got = states[pos, :H]
            seen = [read[pk.off[:s + 1] + r] for s, r in zip(cap_step, cap_row)]
        else:
            cells = [c for c in calls if c[0] in ('dae_gru_cell_fwd', 'dae_lstm_cell_fwd')]
            assert len(cells) == len(gathers) == len(pk.n)
            got = np.stack([cells[s][3]['h'][r, :H] for s, r in zip(cap_step, cap_row)])
            seen = [np.array([gathers[j][2]['rows'][r] for j in range(s + 1)]) for s, r in zip(cap_step, cap_row)]
        _same('%s captured rows' % tag, out[cap_imp], got)
        # the captured state read exactly the impression's window: the last min(time, max_len) reads before it
        for j, q in enumerate(cap_imp):
            u, t = int(imp['user'][q]), int(t_imp[q])
            w = items[indptr[u] + max(0, t - max_len):indptr[u] + t]
            assert np.array_equal(seen[j], w), (tag, int(q), u, t)
    print(tag, worst(tag))
