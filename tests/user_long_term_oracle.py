"""fp64 reference of the long-term user vectors (user_model._UserRNN with long_term_users, DESIGN 4.18): the row-sparse optimizer
step of dae_rows_optimizer_step, the GRU / LSTM states from a given h_0 with autograd down to h_0, and a stage recorder that also
knows the table's gathers and the row step.  Tests only."""
import numpy as np
import torch

import gru_kernel_oracle as go
import step_kernel_oracle as sko
import user_lstm_oracle as lo
from encoder_stages import OPT_NAME, Recorder, check_log
from helpers import snap, snap_vec

NAMES = ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')
ROWS_ARGS = ('table', 'ld', 'cols', 'rows', 'n', 'grad', 'ld_grad', 'slot1', 'slot2', 'counts', 'opt', 'lr', 'momentum', 'stream')


def rows_step(opt, table, rows, grad, slot1, slot2, counts, lr, momentum):
    """dae_rows_optimizer_step restated: (table, slot1, slot2, counts, scale of table) after the step, fp64 (counts int).  Every
    listed row (rows[i] >= 0) takes one step of dae_optimizer_step's rule with grad row i at Adam step counts[row] + 1."""
    p = np.asarray(table, np.float64).copy()
    s1 = None if slot1 is None else np.asarray(slot1, np.float64).copy()
    s2 = None if slot2 is None else np.asarray(slot2, np.float64).copy()
    c = None if counts is None else np.asarray(counts, np.int64).copy()
    scale = np.abs(p)
    for i, r in enumerate(rows):
        if r < 0:
            continue
        t = 1 if c is None else int(c[r]) + 1
        a, b1, b2, sc = sko.optimizer_steps(opt, p[r], [grad[i]], lr, momentum, 1.0, None if s1 is None else s1[r],
                                            None if s2 is None else s2[r], t0=t)
        p[r], scale[r] = a, sc
        if s1 is not None:
            s1[r] = b1
        if s2 is not None:
            s2[r] = b2
        if c is not None:
            c[r] = t
    return p, s1, s2, c, scale


def states(cell, params, seqs, emb, h0):
    """States h of every user from h_0 = h0[i] (c_0 = 0 for the LSTM): list of [L_u, H] fp64 tensors, differentiable in params
    and in h0 (a [B, H] fp64 tensor)."""
    Wi, Wh, bi, bh = (params[n] for n in NAMES)
    H = Wh.shape[1]
    E = torch.as_tensor(np.asarray(emb, np.float64))
    out = []
    for i, s in enumerate(seqs):
        h, c = h0[i], torch.zeros(H, dtype=torch.float64)
        hs = []
        for a in s:
            xg = Wi @ E[int(a)] + bi
            hg = Wh @ h + bh
            if cell == 'gru':
                r = torch.sigmoid(xg[:H] + hg[:H])
                z = torch.sigmoid(xg[H:2 * H] + hg[H:2 * H])
                n = torch.tanh(xg[2 * H:] + r * hg[2 * H:])
                h = (1 - z) * n + z * h
            else:
                g = xg + hg
                c = torch.sigmoid(g[H:2 * H]) * c + torch.sigmoid(g[:H]) * torch.tanh(g[2 * H:3 * H])
                h = torch.sigmoid(g[3 * H:]) * torch.tanh(c)
            hs.append(h)
        out.append(torch.stack(hs))
    return out


def loss_and_grads(cell, params_np, seqs, negs, emb, h0_np):
    """The random-negative loss of a batch whose users start from h0_np [B, H]: (loss, {name: grad}, states, dL/dh0)."""
    params = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in params_np.items()}
    h0 = torch.tensor(np.asarray(h0_np, np.float64), requires_grad=True)
    hs = states(cell, params, seqs, emb, h0)
    loss = lo.rank_loss(hs, seqs, negs, emb)
    loss.backward()
    return float(loss.detach()), {k: v.grad.numpy() for k, v in params.items()}, [h.detach().numpy() for h in hs], h0.grad.numpy()


class LongTermRecorder(Recorder):
    """encoder_stages.Recorder that also records dae_rows_optimizer_step, and snapshots the long-term table (table: the model's
    full [U + 1, H] table tensor) before each gather that reads it."""

    def __init__(self, real, table):
        super().__init__(real)
        self.table = table

    def __call__(self, name, *a):
        if name == 'dae_gather_split_bf16' and a[0] == self.table.data_ptr():
            torch.cuda.synchronize()
            P = self.table.cpu().numpy()
            rows = snap_vec(a[2], a[3], '<i4')
            self.real(name, *a)
            torch.cuda.synchronize()
            self.log.append(('table_gather', a, {'table': P, 'rows': rows},
                             {'hi': snap(a[5], a[3], a[7], 'u2'), 'lo': snap(a[6], a[3], a[7], 'u2')}))
            return
        if name != 'dae_rows_optimizer_step':
            return super().__call__(name, *a)
        assert len(a) == len(ROWS_ARGS)
        d = dict(zip(ROWS_ARGS, a))
        torch.cuda.synchronize()
        rows_total = self.table.shape[0]
        pre = {k: snap(d[k], rows_total, d['ld']) for k in ('table', 'slot1', 'slot2')}
        pre['counts'] = snap_vec(d['counts'], rows_total, '<i4') if d['counts'] else None
        pre['rows'] = snap_vec(d['rows'], d['n'], '<i4')
        pre['grad'] = snap(d['grad'], d['n'], d['ld_grad'])
        self.real(name, *a)
        torch.cuda.synchronize()
        post = {k: snap(d[k], rows_total, d['ld']) for k in ('table', 'slot1', 'slot2')}
        post['counts'] = snap_vec(d['counts'], rows_total, '<i4') if d['counts'] else None
        self.log.append((name, d, pre, post))


def check_rows_step(tag, d, pre, post):
    """A recorded dae_rows_optimizer_step against rows_step; rows not listed, their slots and counts bit for bit unchanged."""
    H = d['cols']
    opt = OPT_NAME[d['opt']]
    g = pre['grad'][:, :H]
    sl = lambda k: None if pre[k] is None else pre[k][:, :H]   # noqa: E731
    p, s1, s2, c, sc = rows_step(opt, pre['table'][:, :H], pre['rows'], g, sl('slot1'), sl('slot2'), pre['counts'], d['lr'],
                                 d['momentum'])
    go.check('%s rows step table' % tag, post['table'][:, :H], p, sc, go.C_FP32)
    touched = np.zeros(pre['table'].shape[0], bool)
    touched[pre['rows'][pre['rows'] >= 0]] = True
    for k in ('table', 'slot1', 'slot2'):
        if pre[k] is not None:
            assert np.array_equal(post[k][~touched].view(np.uint32), pre[k][~touched].view(np.uint32)), '%s: %s rows not listed changed' % (
                tag, k)
    if pre['counts'] is not None:
        assert np.array_equal(post['counts'], c), tag
    # the slots: one rounding per operation of a two-term update, within C_FP32 of the sum of its absolute terms
    G = np.zeros_like(p)
    ok = pre['rows'] >= 0
    G[pre['rows'][ok]] = np.abs(g[ok])
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    mu = abs(float(np.float32(d['momentum'])))
    scales = [None, None]
    if opt == 'momentum':
        scales[0] = mu * np.abs(sl('slot1')) + G
    elif opt == 'ada_grad':
        scales[0] = np.abs(sl('slot1')) + G * G
    elif opt == 'adam':
        scales = [b1 * np.abs(sl('slot1')) + (1 - b1) * G, b2 * np.abs(sl('slot2')) + (1 - b2) * G * G]
    for k, want, sc_k in (('slot1', s1, scales[0]), ('slot2', s2, scales[1])):
        if sc_k is not None:
            go.check('%s rows step %s' % (tag, k), post[k][touched, :H], want[touched], sc_k[touched], go.C_FP32)


def check_long_term_log(log, emb, H, tag):
    """check_log over the encoder calls, plus the table gathers (bit for bit against the table's split) and the row steps; returns
    check_log's calls by name with 'table_gather' and 'dae_rows_optimizer_step' added."""
    plain = [c for c in log if c[0] not in ('table_gather', 'dae_rows_optimizer_step')]
    by = check_log(plain, emb, H, tag)
    for name, a, pre, post in log:
        if name == 'table_gather':
            assert a[1] == H and a[4] == H and a[8] == H, tag
            w_hi, w_lo = go.gather_split(pre['table'], pre['rows'], H, a[7], H)
            assert np.array_equal(post['hi'], w_hi) and np.array_equal(post['lo'], w_lo), '%s: table gather' % tag
            by.setdefault(name, []).append((a, pre, post))
        elif name == 'dae_rows_optimizer_step':
            check_rows_step(tag, a, pre, post)
            by.setdefault(name, []).append((a, pre, post))
    return by
