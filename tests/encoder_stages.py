"""Stage-by-stage checks of the user encoders' host-side chains (user_model.UserGRU, UserLSTM, UserAttention).  Tests only.

Recorder stands in for user_model.call: it decodes each call's positional arguments by the export's C parameter names (ARGS, the
names of include/dae_sm100.h), snapshots the inputs, runs the call, synchronizes and snapshots the outputs.  check_log then checks
every recorded call against the fp64 reference of its own recorded inputs, element by element, with the bounds of the kernels'
oracles (C_FP32 for the CUDA-core kernels, C_BF16X3 for the GEMMs); the splits, gathers and negatives bit for bit.  A call to an
export the recorder does not know fails the test, so a new call in user_model.py cannot pass unchecked.
"""
import numpy as np
import torch

import gru_kernel_oracle as go
import impression_kernel_oracle as ko
import impression_softmax_oracle as smo
import step_kernel_oracle as sko
import user_attention_oracle as ao
import user_lstm_oracle as lo
from helpers import pair_value, snap, snap_vec

from dae_rnn_news_recommendation_b200 import _cabi

ONE_HI = 0x3F80          # bf16 bits of 1.0
OPT_NAME = {v: k for k, v in _cabi.OPT.items()}

# the C parameter names of every export the recorder decodes (include/dae_sm100.h)
ARGS = {
    'dae_split_bf16': ('src', 'rows', 'cols', 'ld_src', 'hi', 'lo', 'ld_dst', 'ones_col', 'scale', 'stream'),
    'dae_gemm_bf16x3': ('M', 'N', 'K', 'alpha', 'a_hi', 'a_lo', 'lda', 'a_mn_major', 'b_hi', 'b_lo', 'ldb', 'b_mn_major', 'C', 'ldc',
                        'n_store', 'special_col', 'special_out', 'k_splits', 'accumulate', 'stream'),
    'dae_optimizer_step': ('theta', 'grad', 'slot1', 'slot2', 'n', 'opt', 'lr', 'momentum', 'grad_scale', 'step', 'ctl', 'w_hi', 'w_lo',
                           'F', 'H', 'ld_split', 'stream'),
    'dae_gather_split_bf16': ('src', 'ld_src', 'rows', 'n_rows', 'cols', 'hi', 'lo', 'ld_dst', 'ones_col', 'stream'),
    'dae_gru_cell_fwd': ('n', 'H', 'xp', 'ld_xp', 'hp', 'ld_hp', 'h_prev', 'ld_hprev', 'h_out', 'ld_h', 'n_split', 'h_hi', 'h_lo',
                         'ld_split', 'gates', 'ld_gates', 'stream'),
    'dae_gru_cell_bwd': ('n', 'H', 'dh_in', 'ld_dh_in', 'carry', 'ld_carry', 'gates', 'ld_gates', 'h_prev', 'ld_hprev', 'dxp_hi',
                         'dxp_lo', 'dhp_hi', 'dhp_lo', 'ld_g', 'stream'),
    'dae_seq_negatives': ('pos', 'n_pos', 'n_items', 'seed', 'epoch', 'batch', 'neg', 'stream'),
    'dae_seq_rank_loss': ('h', 'ld_h', 'emb', 'ld_emb', 'H', 'pos', 'neg', 'n_pos', 'scale', 'dh', 'ld_dh', 'loss_sum', 'stream'),
    'dae_lstm_cell_fwd': ('n', 'H', 'xp', 'ld_xp', 'hp', 'ld_hp', 'c_prev', 'ld_cprev', 'c_out', 'ld_c', 'h_out', 'ld_h', 'n_split',
                          'h_hi', 'h_lo', 'ld_split', 'gates', 'ld_gates', 'stream'),
    'dae_lstm_cell_bwd': ('n', 'H', 'dh_in', 'ld_dh_in', 'carry_h', 'ld_carry_h', 'carry_c', 'ld_carry_c', 'gates', 'ld_gates', 'c',
                          'ld_c', 'c_prev', 'ld_cprev', 'da_hi', 'da_lo', 'ld_da', 'stream'),
    'dae_seq_attention_fwd': ('B', 'T', 'off', 'lens', 'H', 'heads', 'qkv', 'ld_qkv', 'o', 'ld_o', 'o_hi', 'o_lo', 'ld_split', 'lse',
                              'ld_lse', 'stream'),
    'dae_seq_attention_bwd': ('B', 'T', 'off', 'lens', 'H', 'heads', 'qkv', 'ld_qkv', 'o', 'ld_o', 'lse', 'ld_lse', 'dout', 'ld_do',
                              'dqkv_hi', 'dqkv_lo', 'ld_dqkv', 'stream'),
    'dae_seq_pool_fwd': ('B', 'T', 'off', 'lens', 'H', 'A', 'z', 'ld_z', 'q', 'm', 'ld_m', 'u', 'ld_u', 'score', 'plse', 'stream'),
    'dae_seq_pool_bwd': ('B', 'T', 'off', 'lens', 'H', 'A', 'du', 'ld_du', 'u', 'ld_u', 'm', 'ld_m', 'z', 'ld_z', 'q', 'score', 'plse',
                         'dm', 'ld_dm', 'dz_hi', 'dz_lo', 'ld_dz', 'dq', 'workspace', 'stream'),
    'dae_impression_rank_loss': ('h', 'ld_h', 'emb', 'ld_emb', 'H', 'pos_indptr', 'n_pos', 'imp_indptr', 'items', 'clicked', 'scale',
                                 'dh', 'ld_dh', 'loss_sum', 'stream'),
    'dae_impression_softmax_loss': ('h', 'ld_h', 'emb', 'ld_emb', 'H', 'pos_indptr', 'n_pos', 'imp_indptr', 'items', 'clicked',
                                    'imp_ids', 'K', 'seed', 'epoch', 'scale', 'dh', 'ld_dh', 'loss_sum', 'workspace', 'stream'),
}


class Args(tuple):
    """A call's positional arguments, also readable by their C parameter names (a.M, a.ld_h)."""

    def __new__(cls, name, a):
        t = super().__new__(cls, a)
        t._names = ARGS[name]
        return t

    def __getattr__(self, k):
        if k.startswith('_') or k not in self._names:
            raise AttributeError(k)
        return self[self._names.index(k)]


def _u2(ptr, rows, ld):
    """bf16 bits [rows x ld] at ptr (None for a NULL pointer or no rows)."""
    return snap(ptr, rows, ld, 'u2')


def _positions(a):
    """off [T + 1], lens [B] and P of an attention / pooling call."""
    off = snap_vec(a.off, a.T + 1, '<i8')
    return off, snap_vec(a.lens, a.B, '<i4'), int(off[a.T])


def _pre(name, a):
    if name == 'dae_split_bf16':
        return {'src': snap(a.src, a.rows, a.ld_src)}
    if name == 'dae_gemm_bf16x3':
        ra, rb = (a.K if a.a_mn_major else a.M), (a.K if a.b_mn_major else a.N)
        pre = {'a_hi': _u2(a.a_hi, ra, a.lda), 'a_lo': _u2(a.a_lo, ra, a.lda), 'b_hi': _u2(a.b_hi, rb, a.ldb),
               'b_lo': _u2(a.b_lo, rb, a.ldb), 'c': snap(a.C, a.M, a.ldc)}
        pre['a'], pre['b'] = pair_value(pre['a_hi'], pre['a_lo']), pair_value(pre['b_hi'], pre['b_lo'])
        return pre
    if name == 'dae_optimizer_step':
        return {k: snap_vec(getattr(a, k), a.n, '<f4') for k in ('theta', 'grad', 'slot1', 'slot2') if getattr(a, k)}
    if name == 'dae_gather_split_bf16':
        return {'rows': snap_vec(a.rows, a.n_rows, '<i4')}
    if name == 'dae_gru_cell_fwd':
        return {'xp': snap(a.xp, a.n, a.ld_xp), 'hp': snap(a.hp, a.n, a.ld_hp), 'h_prev': snap(a.h_prev, a.n, a.ld_hprev)}
    if name == 'dae_gru_cell_bwd':
        return {'dh_in': snap(a.dh_in, a.n, a.ld_dh_in), 'carry': snap(a.carry, a.n, a.ld_carry), 'gates': snap(a.gates, a.n, a.ld_gates),
                'h_prev': snap(a.h_prev, a.n, a.ld_hprev)}
    if name == 'dae_seq_negatives':
        return {'pos': snap_vec(a.pos, a.n_pos, '<i4')}
    if name == 'dae_seq_rank_loss':
        return {'h': snap(a.h, a.n_pos, a.ld_h), 'pos': snap_vec(a.pos, a.n_pos, '<i4'), 'neg': snap_vec(a.neg, a.n_pos, '<i4'),
                'loss': snap_vec(a.loss_sum, 1, '<f8')}
    if name == 'dae_lstm_cell_fwd':
        return {'xp': snap(a.xp, a.n, a.ld_xp), 'hp': snap(a.hp, a.n, a.ld_hp), 'c_prev': snap(a.c_prev, a.n, a.ld_cprev)}
    if name == 'dae_lstm_cell_bwd':
        return {'dh_in': snap(a.dh_in, a.n, a.ld_dh_in), 'carry_h': snap(a.carry_h, a.n, a.ld_carry_h),
                'carry_c': snap(a.carry_c, a.n, a.ld_carry_c), 'gates': snap(a.gates, a.n, a.ld_gates), 'c': snap(a.c, a.n, a.ld_c),
                'c_prev': snap(a.c_prev, a.n, a.ld_cprev)}
    if name == 'dae_seq_attention_fwd':
        off, lens, P = _positions(a)
        return {'off': off, 'lens': lens, 'P': P, 'qkv': snap(a.qkv, P, a.ld_qkv)}
    if name == 'dae_seq_attention_bwd':
        off, lens, P = _positions(a)
        return {'off': off, 'lens': lens, 'P': P, 'qkv': snap(a.qkv, P, a.ld_qkv), 'o': snap(a.o, P, a.ld_o),
                'lse': snap(a.lse, P, a.ld_lse), 'dout': snap(a.dout, P, a.ld_do)}
    if name == 'dae_seq_pool_fwd':
        off, lens, P = _positions(a)
        return {'off': off, 'lens': lens, 'P': P, 'z': snap(a.z, P, a.ld_z), 'q': snap_vec(a.q, a.A, '<f4'), 'm': snap(a.m, P, a.ld_m)}
    if name == 'dae_seq_pool_bwd':
        off, lens, P = _positions(a)
        return {'off': off, 'lens': lens, 'P': P, 'du': snap(a.du, P, a.ld_du), 'u': snap(a.u, P, a.ld_u), 'm': snap(a.m, P, a.ld_m),
                'z': snap(a.z, P, a.ld_z), 'q': snap_vec(a.q, a.A, '<f4'), 'score': snap_vec(a.score, P, '<f4'),
                'plse': snap_vec(a.plse, P, '<f4')}
    if name in ('dae_impression_rank_loss', 'dae_impression_softmax_loss'):
        pi = snap_vec(a.pos_indptr, a.n_pos + 1, '<i8')
        n_q = int(pi[-1])
        ip = snap_vec(a.imp_indptr, n_q + 1, '<i8')
        pre = {'h': snap(a.h, a.n_pos, a.ld_h), 'pos_indptr': pi, 'indptr': ip, 'items': snap_vec(a.items, int(ip[-1]), '<i4'),
               'clicked': snap_vec(a.clicked, int(ip[-1]), '|u1'), 'loss': snap_vec(a.loss_sum, 1, '<f8')}
        if name == 'dae_impression_softmax_loss':
            pre['ids'] = snap_vec(a.imp_ids, n_q, '<i8')
        return pre
    raise AssertionError(name)


def _post(name, a, pre):
    if name == 'dae_split_bf16':
        return {'hi': _u2(a.hi, a.rows, a.ld_dst), 'lo': _u2(a.lo, a.rows, a.ld_dst)}
    if name == 'dae_gemm_bf16x3':
        return {'c': snap(a.C, a.M, a.ldc)}
    if name == 'dae_optimizer_step':
        post = {k: snap_vec(getattr(a, k), a.n, '<f4') for k in ('theta', 'slot1', 'slot2') if getattr(a, k)}
        if a.w_hi:
            post['w_hi'], post['w_lo'] = _u2(a.w_hi, a.F, a.ld_split), _u2(a.w_lo, a.F, a.ld_split)
        return post
    if name == 'dae_gather_split_bf16':
        return {'hi': _u2(a.hi, a.n_rows, a.ld_dst), 'lo': _u2(a.lo, a.n_rows, a.ld_dst)}
    if name == 'dae_gru_cell_fwd':
        return {'h': snap(a.h_out, a.n, a.ld_h), 'h_hi': _u2(a.h_hi, a.n_split, a.ld_split), 'h_lo': _u2(a.h_lo, a.n_split, a.ld_split),
                'gates': snap(a.gates, a.n, a.ld_gates)}
    if name == 'dae_gru_cell_bwd':
        post = {'carry': snap(a.carry, a.n, a.ld_carry)}
        post.update({k: _u2(getattr(a, k), a.n, a.ld_g) for k in ('dxp_hi', 'dxp_lo', 'dhp_hi', 'dhp_lo')})
        return post
    if name == 'dae_seq_negatives':
        return {'neg': snap_vec(a.neg, a.n_pos, '<i4')}
    if name == 'dae_seq_rank_loss':
        return {'dh': snap(a.dh, a.n_pos, a.ld_dh), 'loss': snap_vec(a.loss_sum, 1, '<f8')}
    if name == 'dae_lstm_cell_fwd':
        return {'c': snap(a.c_out, a.n, a.ld_c), 'h': snap(a.h_out, a.n, a.ld_h), 'h_hi': _u2(a.h_hi, a.n_split, a.ld_split),
                'h_lo': _u2(a.h_lo, a.n_split, a.ld_split), 'gates': snap(a.gates, a.n, a.ld_gates)}
    if name == 'dae_lstm_cell_bwd':
        return {'carry_h': snap(a.carry_h, a.n, a.ld_carry_h), 'carry_c': snap(a.carry_c, a.n, a.ld_carry_c),
                'da_hi': _u2(a.da_hi, a.n, a.ld_da), 'da_lo': _u2(a.da_lo, a.n, a.ld_da)}
    if name == 'dae_seq_attention_fwd':
        P = pre['P']
        return {'o': snap(a.o, P, a.ld_o), 'o_hi': _u2(a.o_hi, P, a.ld_split), 'o_lo': _u2(a.o_lo, P, a.ld_split),
                'lse': snap(a.lse, P, a.ld_lse)}
    if name == 'dae_seq_attention_bwd':
        return {'dqkv_hi': _u2(a.dqkv_hi, pre['P'], a.ld_dqkv), 'dqkv_lo': _u2(a.dqkv_lo, pre['P'], a.ld_dqkv)}
    if name == 'dae_seq_pool_fwd':
        P = pre['P']
        return {'u': snap(a.u, P, a.ld_u), 'score': snap_vec(a.score, P, '<f4'), 'plse': snap_vec(a.plse, P, '<f4')}
    if name == 'dae_seq_pool_bwd':
        P = pre['P']
        return {'dm': snap(a.dm, P, a.ld_dm), 'dz_hi': _u2(a.dz_hi, P, a.ld_dz), 'dz_lo': _u2(a.dz_lo, P, a.ld_dz),
                'dq': snap_vec(a.dq, a.A, '<f4')}
    if name in ('dae_impression_rank_loss', 'dae_impression_softmax_loss'):
        return {'dh': snap(a.dh, a.n_pos, a.ld_dh), 'loss': snap_vec(a.loss_sum, 1, '<f8')}
    raise AssertionError(name)


class Recorder:
    """Stands in for user_model.call: snapshots each kernel's inputs, runs it, synchronizes and snapshots its outputs.  log holds
    (name, Args, pre, post) per call, in call order."""

    def __init__(self, real):
        self.real, self.log = real, []

    def __call__(self, name, *a):
        assert name in ARGS, 'the stage recorder does not know %s: add its arguments, snapshots and check to encoder_stages.py' % name
        assert len(a) == len(ARGS[name]), '%s called with %d arguments, its C signature has %d' % (name, len(a), len(ARGS[name]))
        a = Args(name, a)
        pre = _pre(name, a)
        self.real(name, *a)
        torch.cuda.synchronize()
        self.log.append((name, a, pre, _post(name, a, pre)))


def bf16_bits(x):
    """bf16 hi / lo bit patterns of fp32 x (step_kernel_oracle.bf16_split)."""
    return go.bf16_split(np.asarray(x, np.float32))


def split_bits(v, ld, ones_col=-1):
    """dae_split_bf16's hi / lo of v [rows x cols] into [rows x ld]: zero padding, column ones_col = 1."""
    full = np.zeros((v.shape[0], ld), np.float32)
    full[:, :v.shape[1]] = v
    if ones_col >= 0:
        full[:, ones_col] = 1.0
    return bf16_bits(full)


def assert_bits(tag, got, want):
    got, want = np.asarray(got), np.asarray(want)
    bad = got != want
    assert got.shape == want.shape and not bad.any(), '%s: %d of %d entries differ, first at %s' % (
        tag, int(bad.sum()), bad.size, np.argwhere(bad)[:5].tolist())


def _optimizer_check(tag, a, pre, post):
    opt = OPT_NAME[a.opt]
    g = pre['grad'].astype(np.float64) * float(np.float32(a.grad_scale))
    p, s1, s2, sc = sko.optimizer_steps(opt, pre['theta'], [pre['grad']], a.lr, a.momentum, a.grad_scale, pre.get('slot1'),
                                        pre.get('slot2'), t0=a.step)
    go.check('%s %s theta' % (tag, opt), post['theta'], p, sc, go.C_FP32)
    # the slots: one rounding per operation of a two-term update, within C_FP32 of the sum of its absolute terms
    if opt == 'momentum':
        go.check('%s momentum slot' % tag, post['slot1'], s1, abs(a.momentum) * np.abs(pre['slot1']) + np.abs(g), go.C_FP32)
    elif opt == 'adam':
        b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
        go.check('%s adam m' % tag, post['slot1'], s1, b1 * np.abs(pre['slot1']) + (1 - b1) * np.abs(g), go.C_FP32)
        go.check('%s adam v' % tag, post['slot2'], s2, b2 * np.abs(pre['slot2']) + (1 - b2) * g * g, go.C_FP32)
    elif opt == 'ada_grad':
        go.check('%s adagrad slot' % tag, post['slot1'], s1, np.abs(pre['slot1']) + g * g, go.C_FP32)
    if a.w_hi:
        F, cols = a.F, a.H
        w_hi, w_lo = bf16_bits(post['theta'][:F * cols].reshape(F, cols))
        assert_bits('%s split of the new W' % tag, post['w_hi'][:, :cols], w_hi)
        assert_bits('%s split of the new W (lo)' % tag, post['w_lo'][:, :cols], w_lo)


def check_log(log, emb, H, tag):
    """Every recorded kernel call against the fp64 reference of its own inputs; returns the calls by name.  emb: the article
    embeddings (fp32 [N, H]) the gathers and losses read.  In a training batch the backward cell's carries must be zero in the
    rows of users whose last read is the cell's step: rows [n_{t+1}, n_t) at step t, every row at the last step."""
    by = {}
    prev_bwd_n = None
    for k, (name, a, pre, post) in enumerate(log):
        by.setdefault(name, []).append((a, pre, post))
        ct = '%s call %d %s' % (tag, k, name)
        if name in ('dae_gru_cell_fwd', 'dae_lstm_cell_fwd'):
            prev_bwd_n = None                      # a forward pass starts: the next backward step is a batch's last
        if name == 'dae_gru_cell_fwd':
            want = go.cell_fwd(pre['xp'], pre['hp'], pre['h_prev'], H)
            go.check('%s fwd h' % tag, post['h'][:, :H], *want['h'], go.C_FP32)
            if post['gates'] is not None:
                for j, g in enumerate(('r', 'z', 'n')):
                    go.check('%s fwd %s' % (tag, g), post['gates'][:, j * H:(j + 1) * H], *want[g], go.C_FP32)
                assert np.array_equal(post['gates'][:, 3 * H:4 * H], pre['hp'][:, 2 * H:3 * H])
            if post['h_hi'] is not None:
                w_hi, w_lo = go.bf16_split(post['h'][:a[10], :H])
                assert np.array_equal(post['h_hi'][:, :H], w_hi) and np.array_equal(post['h_lo'][:, :H], w_lo)
        elif name == 'dae_gru_cell_bwd':
            n = a[0]
            c0 = pre['carry'][:, :H]
            lo_row = 0 if prev_bwd_n is None else prev_bwd_n
            assert (c0[lo_row:] == 0).all(), '%s: carry rows [%d, %d) not zero' % (tag, lo_row, n)
            prev_bwd_n = n
            want = go.cell_bwd(pre['dh_in'], c0, pre['gates'], pre['h_prev'], H)
            go.check('%s bwd carry' % tag, post['carry'][:, :H], *want['carry'], go.C_FP32)
            for j, g in enumerate(('dr', 'dz', 'dn')):
                sl = slice(j * H, (j + 1) * H)
                go.check_pair('%s bwd %s' % (tag, g), post['dxp_hi'][:, sl], post['dxp_lo'][:, sl], *want[g], go.C_FP32)
            assert np.array_equal(post['dhp_hi'][:, :2 * H], post['dxp_hi'][:, :2 * H])
            assert np.array_equal(post['dhp_lo'][:, :2 * H], post['dxp_lo'][:, :2 * H])
            go.check_pair('%s bwd r dn' % tag, post['dhp_hi'][:, 2 * H:3 * H], post['dhp_lo'][:, 2 * H:3 * H], *want['rdn'], go.C_FP32)
        elif name == 'dae_lstm_cell_fwd':
            want = lo.cell_fwd(pre['xp'], pre['hp'], pre['c_prev'], H)
            go.check('%s lstm fwd c' % tag, post['c'][:, :H], *want['c'], go.C_FP32)
            go.check('%s lstm fwd h' % tag, post['h'][:, :H], *want['h'], go.C_FP32)
            if post['gates'] is not None:
                for j, g in enumerate('ifgo'):
                    go.check('%s lstm fwd %s' % (tag, g), post['gates'][:, j * H:(j + 1) * H], *want[g], go.C_FP32)
            if post['h_hi'] is not None:
                w_hi, w_lo = bf16_bits(post['h'][:a.n_split, :H])
                assert_bits('%s: h_hi, the split of h' % ct, post['h_hi'][:, :H], w_hi)
                assert_bits('%s: h_lo, the split of h' % ct, post['h_lo'][:, :H], w_lo)
        elif name == 'dae_lstm_cell_bwd':
            n = a.n
            lo_row = 0 if prev_bwd_n is None else prev_bwd_n
            for c in ('carry_h', 'carry_c'):
                assert (pre[c][lo_row:, :H] == 0).all(), '%s: %s rows [%d, %d) not zero' % (ct, c, lo_row, n)
            prev_bwd_n = n
            assert_bits('%s: carry_h is read only' % ct, post['carry_h'][:, :H].view(np.uint32), pre['carry_h'][:, :H].view(np.uint32))
            want = lo.cell_bwd(pre['dh_in'], pre['carry_h'], pre['carry_c'], pre['gates'], pre['c'], pre['c_prev'], H)
            go.check('%s lstm bwd carry_c' % tag, post['carry_c'][:, :H], *want['carry_c'], go.C_FP32)
            for j, g in enumerate(('di', 'df', 'dg', 'do')):
                sl = slice(j * H, (j + 1) * H)
                go.check_pair('%s lstm bwd %s' % (tag, g), post['da_hi'][:, sl], post['da_lo'][:, sl], *want[g], go.C_FP32)
        elif name == 'dae_gemm_bf16x3':
            M, N, K = a[0], a[1], a[2]
            assert a.special_out is None and a.n_store <= 0, ct
            A = pre['a'].T[:M, :K] if a[7] else pre['a'][:M, :K]
            B = pre['b'].T[:N, :K] if a[11] else pre['b'][:N, :K]
            want, s = go.gemm_nt(A, B)
            want, s = a[3] * want, abs(a[3]) * s
            if a[18]:
                want, s = want + pre['c'][:, :N], s + np.abs(pre['c'][:, :N])
            go.check('%s gemm %dx%dx%d' % (tag, M, N, K), post['c'][:, :N], want, s, go.C_BF16X3)
        elif name == 'dae_split_bf16':
            assert a.scale == 1.0, ct
            w_hi, w_lo = split_bits(pre['src'][:, :a.cols], a.ld_dst, a.ones_col)
            assert_bits('%s hi' % ct, post['hi'], w_hi)
            assert_bits('%s lo' % ct, post['lo'], w_lo)
        elif name == 'dae_seq_rank_loss':
            w_dh, s_dh, lt, s_lt = go.seq_rank_loss(pre['h'], emb, pre['pos'], pre['neg'], a[8], H)
            go.check('%s loss dh' % tag, post['dh'][:, :H], w_dh, s_dh, go.C_FP32)
            assert (post['dh'][pre['pos'] < 0, :H] == 0).all()
            go.check('%s loss sum' % tag, post['loss'][0] - pre['loss'][0], lt.sum(), s_lt.sum(), go.C_FP32, tiny=1e-15)
        elif name == 'dae_impression_rank_loss':
            w_dh, s_dh, w_loss, s_loss = ko.rank_loss(pre['h'], emb, pre['pos_indptr'], pre['indptr'], pre['items'], pre['clicked'],
                                                      a.scale, H)
            go.check('%s pairwise dh' % tag, post['dh'][:, :H], w_dh, s_dh, go.C_FP32)
            go.check('%s pairwise sum' % tag, post['loss'][0] - pre['loss'][0], w_loss, s_loss, go.C_FP32, tiny=1e-15)
        elif name == 'dae_impression_softmax_loss':
            w_dh, s_dh, w_loss, s_loss, _ = smo.softmax_loss(pre['h'], emb, pre['pos_indptr'], pre['indptr'], pre['items'], pre['clicked'],
                                                             pre['ids'], a.K, a.seed, a.epoch, a.scale, H)
            go.check('%s softmax dh' % tag, post['dh'][:, :H], w_dh, s_dh, go.C_FP32)
            go.check('%s softmax sum' % tag, post['loss'][0] - pre['loss'][0], w_loss, s_loss, go.C_FP32, tiny=1e-15)
        elif name == 'dae_seq_negatives':
            assert np.array_equal(post['neg'], go.seq_negatives(pre['pos'], a[2], a[3], a[4], a[5]))
        elif name == 'dae_gather_split_bf16':
            w_hi, w_lo = go.gather_split(emb, pre['rows'], a[4], a[7], a[8])
            assert np.array_equal(post['hi'], w_hi) and np.array_equal(post['lo'], w_lo)
        elif name == 'dae_seq_attention_fwd':
            P, hd = pre['P'], a.heads
            want = ao.attention_fwd(pre['qkv'][:, :3 * H], pre['off'], pre['lens'], H, hd)
            go.check('%s attn fwd O' % tag, post['o'][:, :H], *want['O'], go.C_FP32)
            go.check('%s attn fwd lse' % tag, post['lse'][:, :hd], *want['lse'], go.C_FP32)
            w_hi, w_lo = bf16_bits(post['o'][:, :H])
            assert_bits('%s: o_hi, the split of O' % ct, post['o_hi'][:, :H], w_hi)
            assert_bits('%s: o_lo, the split of O' % ct, post['o_lo'][:, :H], w_lo)
        elif name == 'dae_seq_attention_bwd':
            want = ao.attention_bwd(pre['qkv'][:, :3 * H], pre['o'][:, :H], pre['lse'][:, :a.heads], pre['dout'][:, :H], pre['off'],
                                    pre['lens'], H, a.heads)
            for j, g in enumerate(('dQ', 'dK', 'dV')):
                sl = slice(j * H, (j + 1) * H)
                go.check_pair('%s attn bwd %s' % (tag, g), post['dqkv_hi'][:, sl], post['dqkv_lo'][:, sl], want['dQKV'][0][:, sl],
                              want['dQKV'][1][:, sl], go.C_FP32)
        elif name == 'dae_seq_pool_fwd':
            want = ao.pool_fwd(pre['z'], pre['q'], pre['m'], pre['off'], pre['lens'], H, a.A)
            go.check('%s pool fwd a' % tag, post['score'], *want['score'], go.C_FP32)
            go.check('%s pool fwd lse' % tag, post['plse'], *want['plse'], go.C_FP32)
            go.check('%s pool fwd u' % tag, post['u'][:, :H], *want['u'], go.C_FP32)
        elif name == 'dae_seq_pool_bwd':
            want = ao.pool_bwd(pre['du'], pre['u'], pre['m'], pre['z'], pre['q'], pre['score'], pre['plse'], pre['off'], pre['lens'], H,
                               a.A)
            go.check('%s pool bwd dM' % tag, post['dm'][:, :H], *want['dM'], go.C_FP32)
            go.check_pair('%s pool bwd dZ' % tag, post['dz_hi'][:, :a.A], post['dz_lo'][:, :a.A], *want['dZ'], go.C_FP32)
            go.check('%s pool bwd dq' % tag, post['dq'], *want['dq'], go.C_FP32)
        elif name == 'dae_optimizer_step':
            _optimizer_check(tag, a, pre, post)
        else:
            raise AssertionError('%s: no check for %s' % (ct, name))
    return by


def worst(tag):
    """The worst error / bound ratio of every check whose name starts with tag."""
    return {k: round(v, 4) for k, v in go.WORST.items() if k.startswith(tag)}
