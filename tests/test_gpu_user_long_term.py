"""Long-term user vectors on the GPU (user_model.UserGRU / UserLSTM with long_term_users, DESIGN 4.18): dae_rows_optimizer_step
against a NumPy restatement, one training batch with the table against fp64 and stage by stage, the equivalences with the plain
encoder, torch parity from h_0 = P[u], cold-start users, save / load, the CLI and the learning check."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from helpers import rel_err  # noqa: E402
from user_long_term_oracle import LongTermRecorder, check_long_term_log, check_rows_step, loss_and_grads  # noqa: E402

from dae_rnn_news_recommendation_b200 import _cabi, sparse_optim, user_model  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import Packed, UserGRU, UserLSTM  # noqa: E402

DEV = 'cuda:0'
N_ITEMS = 900
CELLS = {'gru': (UserGRU, torch.nn.GRU, 3), 'lstm': (UserLSTM, torch.nn.LSTM, 4)}


def _data(U, H, max_len, seed):
    """Lengths covering 1, 2, max_len and longer than max_len, plus random ones (as tests/test_gpu_user_gru.py)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 4, U)
    lens[:6] = [1, 2, max_len, max_len + 3, 2 * max_len, 1]
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N_ITEMS, int(indptr[-1])).astype(np.int32)
    emb = (rng.standard_normal((N_ITEMS, H)) * 0.5).astype(np.float32)
    return indptr, items, emb


def _impressions(rng, indptr, n_imp):
    user = rng.integers(0, len(indptr) - 1, n_imp)
    time_ = np.array([rng.integers(0, indptr[u + 1] - indptr[u] + 1) for u in user])
    lists = [rng.choice(N_ITEMS, 6, replace=False) for _ in range(n_imp)]
    clicked = np.tile(np.array([1, 0, 0, 1, 0, 0], np.uint8), n_imp)
    return {'user': user.astype(np.int64), 'time': time_.astype(np.int64), 'indptr': np.arange(n_imp + 1, dtype=np.int64) * 6,
            'items': np.concatenate(lists).astype(np.int32), 'clicked': clicked}


def _params(m):
    return {k: v.double().numpy() for k, v in m.state_dict().items()}


def _grads(m):
    H, G, g = m.dim, m.GATES, m.grad.cpu().double().numpy()
    hh, ih = g[:m.nW].reshape(G * H, H + 1), g[m.nW:].reshape(G * H, H + 1)
    return {'weight_ih_l0': ih[:, :H], 'weight_hh_l0': hh[:, :H], 'bias_ih_l0': ih[:, H], 'bias_hh_l0': hh[:, H]}


# ---------------------------------------------------------------------------------------------------------------------------
# dae_rows_optimizer_step
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H', [37, 64])
@pytest.mark.parametrize('opt', sorted(_cabi.OPT))
def test_rows_step_against_numpy(opt, H):
    """Two steps over a table of 300 rows + the zero row: listed rows against rows_step (with their own counts), -1 entries,
    rows not listed, their slots and counts and the zero row bit for bit unchanged."""
    rng = np.random.default_rng(H)
    R, n = 301, 120
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
    table = rng.standard_normal((R, H)).astype(np.float32)
    table[R - 1] = 0
    s1 = (np.abs(rng.standard_normal((R, H))) + (0.1 if opt == 'ada_grad' else 0)).astype(np.float32)
    s2 = np.abs(rng.standard_normal((R, H))).astype(np.float32) * 0.01
    counts = rng.integers(0, 50, R).astype(np.int32)
    t, d1, d2, dc = dev(table), dev(s1), dev(s2), dev(counts)
    st = torch.cuda.current_stream().cuda_stream
    for step in range(2):
        rows = rng.choice(R - 1, n, replace=False).astype(np.int32)
        rows[rng.random(n) < 0.2] = -1
        grad = rng.standard_normal((n, H)).astype(np.float32)
        d_rows, d_grad = dev(rows), dev(grad)
        pre = {'table': t.cpu().numpy(), 'slot1': d1.cpu().numpy() if opt != 'gradient_descent' else None,
               'slot2': d2.cpu().numpy() if opt == 'adam' else None, 'counts': dc.cpu().numpy(), 'rows': rows, 'grad': grad}
        _cabi.call('dae_rows_optimizer_step', t.data_ptr(), H, H, d_rows.data_ptr(), n, d_grad.data_ptr(), H,
                   d1.data_ptr() if opt != 'gradient_descent' else None, d2.data_ptr() if opt == 'adam' else None, dc.data_ptr(),
                   _cabi.OPT[opt], 0.05, 0.7, st)
        torch.cuda.synchronize()
        post = {'table': t.cpu().numpy(), 'slot1': d1.cpu().numpy() if opt != 'gradient_descent' else None,
                'slot2': d2.cpu().numpy() if opt == 'adam' else None, 'counts': dc.cpu().numpy()}
        d = dict(cols=H, opt=_cabi.OPT[opt], lr=np.float32(0.05), momentum=np.float32(0.7))
        check_rows_step('%s H=%d step %d' % (opt, H, step), d, pre, post)
        assert not post['table'][R - 1].any()
        if opt != 'adam':   # counts are optional outside Adam: the same step without them leaves them alone
            c0 = dc.clone()
            _cabi.call('dae_rows_optimizer_step', t.data_ptr(), H, H, d_rows.data_ptr(), n, d_grad.data_ptr(), H,
                       d1.data_ptr() if opt != 'gradient_descent' else None, None, None, _cabi.OPT[opt], 0.0, 0.0, st)
            torch.cuda.synchronize()
            assert torch.equal(dc, c0)


# ---------------------------------------------------------------------------------------------------------------------------
# one training batch with the table
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,U,max_len', [(37, 300, 10), (500, 140, 8)])
@pytest.mark.parametrize('cell', ['gru', 'lstm'])
def test_training_batch_with_table(cell, H, U, max_len, monkeypatch):
    cls = CELLS[cell][0]
    indptr, items, emb = _data(U, H, max_len, seed=H + 1)
    m = cls(H, max_len=max_len, batch_users=U, seed=1, learning_rate=1e-2, long_term_users=U + 5, long_term_mask=0.5)
    rng = np.random.default_rng(3)
    m.long_term.copy_(torch.from_numpy((rng.standard_normal((U + 5, H)) * 0.3).astype(np.float32)))
    emb_d = torch.from_numpy(emb).to(DEV)
    m._forward_backward(Packed(indptr, items, np.arange(40), max_len), emb_d, 0, 0)    # a smaller batch first: buffers regrow
    m._optimizer_step()
    pk = Packed(indptr, items, np.arange(U), max_len)
    epoch = 4
    keep = m.long_term_kept(epoch)[pk.order]
    assert keep.any() and (~keep).any()
    P0, params = m._lt.cpu().numpy(), _params(m)
    rec = LongTermRecorder(user_model.call, m._lt)
    monkeypatch.setattr(user_model, 'call', rec)
    monkeypatch.setattr(sparse_optim, 'call', rec)                         # the row step: user_model -> sparse_optim.rows_step
    m.stats.zero_()
    m._forward_backward(pk, emb_d, epoch, 2)
    m._optimizer_step()
    tag = '%s long-term H=%d' % (cell, H)
    by = check_long_term_log(rec.log, emb, H, tag)
    names = [c[0] for c in rec.log]
    T = len(pk.n)
    cell_f, cell_b = 'dae_%s_cell_fwd' % cell, 'dae_%s_cell_bwd' % cell
    want = (['dae_seq_negatives', 'dae_gather_split_bf16', 'dae_split_bf16', 'dae_gemm_bf16x3', 'table_gather'] +
            ['dae_gemm_bf16x3', cell_f] * T + ['dae_seq_rank_loss'] + [cell_b, 'dae_gemm_bf16x3'] * T +
            ['dae_gemm_bf16x3'] * 2 + ['dae_optimizer_step', 'dae_rows_optimizer_step'])
    assert names == want, (tag, names)
    # data flow: h_0 rows (masked users: the zero row), the step-0 operand, the cell's h_prev, the row step's ids and gradient
    rows = np.where(keep, pk.order, U + 5).astype(np.int32)
    ga, gpre, gpost = by['table_gather'][0]
    assert np.array_equal(gpre['rows'], rows) and ga[3] == pk.B
    gemms = by['dae_gemm_bf16x3']
    hp0 = gemms[1]
    assert hp0[0].M == pk.B and np.array_equal(hp0[1]['a_hi'], gpost['hi']) and np.array_equal(hp0[1]['a_lo'], gpost['lo'])
    h0 = P0[rows].astype(np.float64)
    if cell == 'gru':
        assert np.array_equal(by[cell_f][0][1]['h_prev'][:, :H], P0[rows])
        assert np.array_equal(by[cell_b][-1][1]['h_prev'][:, :H], P0[rows])
    carry0 = gemms[1 + T + T - 1]                                          # the carry GEMM after the backward's step 0
    assert carry0[0].M == pk.B and carry0[0].C == m._buf['carry'].data_ptr()
    ra, rpre, rpost = by['dae_rows_optimizer_step'][0]
    assert np.array_equal(rpre['rows'], np.where(keep, pk.order, -1)) and ra['n'] == pk.B and ra['grad'] == m._buf['carry'].data_ptr()
    assert np.array_equal(rpre['grad'][:, :H], carry0[2]['c'][:, :H])
    assert ra['lr'] == m.long_term_learning_rate and ra['opt'] == _cabi.OPT['adam']
    assert not rpost['table'][U + 5].any()
    # against fp64: states, loss, theta's gradient and dL/dh_0
    neg = m._buf['neg'][:pk.P].cpu().numpy()
    Hs = m._buf['Hs'][:pk.P].cpu().double().numpy()
    seqs, negs, got_states = [], [], []
    for i in range(pk.B):
        pos = [pk.position(i, t) for t in range(int(pk.L[i]))]
        seqs.append(pk.items[pos])
        negs.append(neg[pos[:-1]])
        got_states.append(Hs[pos])
    o_loss, o_grads, o_states, o_dh0 = loss_and_grads(cell, params, seqs, negs, emb, h0)
    assert rel_err(np.concatenate(got_states), np.concatenate(o_states)) < 1e-4
    assert rel_err(float(m.stats.item()) / pk.terms, o_loss) < 1e-4
    g = _grads(m)
    for k in o_grads:
        assert rel_err(g[k], o_grads[k]) < 1e-4, (tag, k, rel_err(g[k], o_grads[k]))
    assert rel_err(rpre['grad'][:, :H], o_dh0) < 1e-4, (tag, rel_err(rpre['grad'][:, :H], o_dh0))


# ---------------------------------------------------------------------------------------------------------------------------
# equivalences with the plain encoder, torch parity, cold-start users, save / load
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cell', ['gru', 'lstm'])
def test_zero_table_equals_plain_encoder(cell):
    cls = CELLS[cell][0]
    H, U, max_len = 37, 250, 9
    indptr, items, emb = _data(U, H, max_len, seed=7)
    imp = _impressions(np.random.default_rng(8), indptr, 300)
    a = cls(H, max_len=max_len, batch_users=90, seed=2)
    b = cls(H, max_len=max_len, batch_users=90, seed=2, long_term_users=U)
    assert np.array_equal(a.transform((indptr, items), emb), b.transform((indptr, items), emb))
    assert np.array_equal(a.impression_states((indptr, items), emb, imp), b.impression_states((indptr, items), emb, imp))


@pytest.mark.parametrize('cell', ['gru', 'lstm'])
def test_full_mask_gives_the_plain_gradient_and_leaves_the_table(cell):
    cls = CELLS[cell][0]
    H, U, max_len = 37, 300, 10
    indptr, items, emb = _data(U, H, max_len, seed=11)
    emb_d = torch.from_numpy(emb).to(DEV)
    a = cls(H, max_len=max_len, batch_users=U, seed=4)
    b = cls(H, max_len=max_len, batch_users=U, seed=4, long_term_users=U, long_term_mask=1.0)
    pk = Packed(indptr, items, np.arange(U), max_len)
    for m in (a, b):
        m._forward_backward(pk, emb_d, 0, 0)
    torch.cuda.synchronize()
    assert rel_err(b.grad.cpu().numpy(), a.grad.cpu().numpy()) < 1e-6
    b.num_epochs = 2
    b.fit((indptr, items), emb)
    assert not b._lt.any() and not b._lt_count.any()


def test_masked_set_does_not_depend_on_batch_users():
    """With SGD a row changes exactly when its user is in a batch, kept by the epoch's draw and has a nonzero dL/dh_0."""
    H, U, max_len = 16, 400, 6
    indptr, items, emb = _data(U, H, max_len, seed=13)
    changed = []
    for B in (37, 400):
        m = UserGRU(H, max_len=max_len, batch_users=B, seed=6, num_epochs=1, opt='gradient_descent', learning_rate=1e-2,
                    long_term_users=U, long_term_mask=0.4)
        m.fit((indptr, items), emb)
        changed.append(m.long_term.abs().sum(1).cpu().numpy() > 0)
        counts = m._lt_count[:U].cpu().numpy()
        assert np.array_equal(counts > 0, changed[-1])
    active = np.diff(indptr) >= 2
    assert np.array_equal(changed[0], changed[1])
    assert np.array_equal(changed[0], m.long_term_kept(0) & active)


@pytest.mark.parametrize('cell', ['gru', 'lstm'])
def test_torch_parity_cold_start_and_save_load(cell, tmp_path):
    cls, torch_cls, _ = CELLS[cell]
    H, U, max_len, cold = 37, 260, 8, 6
    indptr, items, emb = _data(U, H, max_len, seed=17)
    m = cls(H, max_len=max_len, batch_users=64, seed=5, num_epochs=3, learning_rate=1e-2, long_term_users=U - cold,
            long_term_learning_rate=0.05)
    m.fit((indptr[:U - cold + 1], items[:indptr[U - cold]]), emb)
    P = m.long_term.cpu().numpy()
    assert np.abs(P).max() > 1e-3
    out = m.transform((indptr, items), emb)
    imp = _impressions(np.random.default_rng(18), indptr, 400)
    q = m.impression_states((indptr, items), emb, imp)
    g = torch_cls(H, H, batch_first=True)
    g.load_state_dict(m.state_dict())

    def run(seq, u):
        h0 = torch.from_numpy(P[u] if u < U - cold else np.zeros(H, np.float32))[None, None]
        with torch.no_grad():
            x = torch.from_numpy(emb[seq])[None]
            y, _ = g(x, h0) if cell == 'gru' else g(x, (h0, torch.zeros_like(h0)))
        return y[0, -1].numpy()
    for u in (0, 1, 2, 3, 4, 100, U - cold - 1, U - cold, U - 1):
        seq = items[indptr[u]:indptr[u + 1]][-max_len:]
        assert rel_err(out[u], run(seq, u)) < 1e-4, (cell, u)
    for i in range(0, 400, 37):
        u, t = int(imp['user'][i]), int(imp['time'][i])
        if t == 0:
            assert not q[i].any()
            continue
        seq = items[indptr[u] + max(0, t - max_len):indptr[u] + t]
        assert rel_err(q[i], run(seq, u)) < 1e-4, (cell, i)
    # cold-start users: the plain encoder's rows
    plain = cls(H, max_len=max_len, batch_users=64, seed=5)
    plain.load_state_dict(m.state_dict())
    pout = plain.transform((indptr, items), emb)
    assert rel_err(out[U - cold:], pout[U - cold:]) < 1e-6
    assert rel_err(out[:U - cold], pout[:U - cold]) > 1e-3                  # the table changes the others
    # save / load
    m.save(tmp_path / 'm.npz')
    m2 = cls.load(tmp_path / 'm.npz', batch_users=64)
    assert np.array_equal(m2.long_term.cpu().numpy(), P)
    assert np.array_equal(m2.transform((indptr, items), emb), out)


# ---------------------------------------------------------------------------------------------------------------------------
# the CLI and the learning check
# ---------------------------------------------------------------------------------------------------------------------------
def test_cli_user_long_term(capsys, tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.synth import make_sequences
    argv = ['--model_name', 'synlt', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--top_k', '5']
    trX, _, trL, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    indptr, items, targets = make_sequences(300, trL, mean_len=8, seed=4)
    np.savez(tmp_path / 's.npz', indptr=indptr, items=items, targets=targets)
    model = cli.main(argv + ['--user_sequences', str(tmp_path / 's.npz'), '--user_epochs', '2', '--user_cell', 'lstm',
                             '--user_long_term', '--user_long_term_mask', '0.3', '--user_long_term_lr', '0.05'])
    assert 'users (LSTM): hit rate@5' in capsys.readouterr().out
    m = UserLSTM.load(model.data_dir + 'user_lstm.npz')
    assert m.long_term_users == 300 and m.long_term.abs().sum() > 0
    assert np.load(model.data_dir + 'user_lstm_top_k_index.npy').shape == (300, 5)
    assert 0.0 <= model.evaluation['user_lstm_hit_rate'] <= 1.0


# test-impression AUC on synth.make_long_term_impressions measured on an H100: see DESIGN 4.18; the asserted margin is half the
# measured gap
LEARNING_MARGIN = 0.115


def test_learning_beats_the_plain_gru():
    from bench_user_long_term import learning_auc, learning_workload
    data = learning_workload()
    plain = learning_auc(UserGRU, data)
    lt = learning_auc(UserGRU, data, user_model.LONG_TERM_LEARNING_RATE)
    print('test-impression AUC: plain GRU %.4f, with the long-term table %.4f' % (plain, lt))
    assert lt - plain > LEARNING_MARGIN, (plain, lt)
