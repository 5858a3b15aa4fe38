"""Host side of the LSTM user encoder (user_model.UserLSTM): the fp64 oracle of tests/user_lstm_oracle.py against torch.nn.LSTM and
autograd, the per-kernel references composed in UserLSTM's packed layout against the whole-batch oracle, the kernel bounds against
float32 emulations, the C ABI's argument checks, state dicts, save / load and the CLI's --user_cell.  No GPU needed."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import gru_kernel_oracle as go
import impression_oracle as io
import user_lstm_oracle as lo
from user_gru_oracle import NAMES

from dae_rnn_news_recommendation_b200.user_model import Packed, UserGRU, UserLSTM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _params(H, rng, scale=1.0):
    k = scale / np.sqrt(H)
    return {'weight_ih_l0': rng.uniform(-k, k, (4 * H, H)), 'weight_hh_l0': rng.uniform(-k, k, (4 * H, H)),
            'bias_ih_l0': rng.uniform(-k, k, 4 * H), 'bias_hh_l0': rng.uniform(-k, k, 4 * H)}


def _seqs(rng, U, N, max_len):
    lens = rng.integers(1, max_len + 3, U)
    lens[:3] = [1, 2, max_len + 2]
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return indptr, rng.integers(0, N, int(indptr[-1])).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------------------
# the whole-batch oracle against torch.nn.LSTM
# ---------------------------------------------------------------------------------------------------------------------------
def test_oracle_states_match_torch_lstm():
    rng = np.random.default_rng(1)
    H, N = 9, 30
    emb = rng.standard_normal((N, H))
    m = torch.nn.LSTM(H, H, batch_first=True).double()
    params = {k: v.detach().clone() for k, v in m.state_dict().items()}
    seqs = [rng.integers(0, N, L) for L in (6, 1, 3, 6)]
    hs, cs = lo.lstm_states(params, seqs, emb, cells=True)
    for u, s in enumerate(seqs):
        with torch.no_grad():
            y, (hn, cn) = m(torch.as_tensor(emb[s])[None])
        np.testing.assert_allclose(hs[u].numpy(), y[0].numpy(), rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(cs[u][-1].numpy(), cn[0, 0].numpy(), rtol=1e-12, atol=1e-13)


def test_oracle_gradients_match_torch_lstm_autograd():
    """loss_and_grads' four gradients are autograd's through torch.nn.LSTM itself (fp64)."""
    rng = np.random.default_rng(2)
    H, N = 7, 40
    emb = rng.standard_normal((N, H))
    m = torch.nn.LSTM(H, H, batch_first=True).double()
    p = {k: v.detach().numpy().copy() for k, v in m.state_dict().items()}
    seqs = [rng.integers(0, N, L) for L in (5, 1, 2, 7, 4)]
    negs = [(s[1:] + 1 + rng.integers(0, N - 1, len(s) - 1)) % N for s in seqs]
    loss, g, states = lo.loss_and_grads(p, seqs, negs, emb)
    hs = [m(torch.as_tensor(emb[s])[None])[0][0] for s in seqs]
    t_loss = lo.rank_loss(hs, seqs, negs, emb)
    t_loss.backward()
    assert abs(loss - float(t_loss.detach())) <= 1e-12 * abs(loss)
    for k, v in m.named_parameters():
        np.testing.assert_allclose(g[k], v.grad.numpy(), rtol=1e-10, atol=1e-14)
    for u in range(len(seqs)):
        np.testing.assert_allclose(states[u], hs[u].detach().numpy(), rtol=1e-12, atol=1e-13)
    # the impression loss at one-click / one-non-click impressions on the next read is the random-negative loss
    imps = [(u, t, [s[t + 1], ng[t]], [1, 0]) for u, (s, ng) in enumerate(zip(seqs, negs)) for t in range(len(s) - 1)]
    i_loss, i_g = lo.impression_loss_and_grads(p, seqs, emb, imps)
    assert abs(i_loss - loss) <= 1e-12 * abs(loss)
    for k in NAMES:
        np.testing.assert_allclose(i_g[k], g[k], rtol=1e-10, atol=1e-14)
    # and impression_oracle's per-position restatement gives the same loss from the oracle's states
    h = np.concatenate([states[u][[t for (v, t, _, _) in imps if v == u]] for u in range(len(seqs))])
    items = np.array([it for (_, _, it, _) in imps]).reshape(-1)
    total, _ = io.impression_loss(h, emb, np.arange(len(imps) + 1), np.arange(0, 2 * len(imps) + 1, 2), items,
                                  np.tile([1, 0], len(imps)), 1.0)
    assert abs(total / len(imps) - loss) <= 1e-12 * abs(loss)


def test_cell_references_match_lstmcell_and_autograd():
    rng = np.random.default_rng(0)
    H, n = 13, 40
    p = _params(H, rng, 3.0)
    x, h, c = rng.standard_normal((n, H)), rng.standard_normal((n, H)), rng.standard_normal((n, H)) * 2
    cell = torch.nn.LSTMCell(H, H).double()
    cell.load_state_dict({k.replace('_l0', ''): torch.from_numpy(v) for k, v in p.items()})
    want_h, want_c = (t.detach().numpy() for t in cell(torch.from_numpy(x), (torch.from_numpy(h), torch.from_numpy(c))))
    xp = x @ p['weight_ih_l0'].T + p['bias_ih_l0']
    hp = h @ p['weight_hh_l0'].T + p['bias_hh_l0']
    got = lo.cell_fwd(xp, hp, c, H)
    np.testing.assert_allclose(got['h'][0], want_h, rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(got['c'][0], want_c, rtol=1e-12, atol=1e-13)
    z = np.zeros((n, H))
    np.testing.assert_array_equal(lo.cell_fwd(xp, hp, None, H)['h'][0], lo.cell_fwd(xp, hp, z, H)['h'][0])
    # backward: dA and the c carry are the gradients of sum((carry_h + dh_in) h) + sum(carry_c c) w.r.t. the pre-activation and c_prev
    a_t = torch.tensor(xp + hp, requires_grad=True)
    cp_t = torch.tensor(c, requires_grad=True)
    i, f = torch.sigmoid(a_t[:, :H]), torch.sigmoid(a_t[:, H:2 * H])
    g, o = torch.tanh(a_t[:, 2 * H:3 * H]), torch.sigmoid(a_t[:, 3 * H:])
    c_t = f * cp_t + i * g
    h_t = o * torch.tanh(c_t)
    carry_h, carry_c, dh_in = rng.standard_normal((n, H)), rng.standard_normal((n, H)), rng.standard_normal((n, H))
    ((h_t * torch.from_numpy(carry_h + dh_in)).sum() + (c_t * torch.from_numpy(carry_c)).sum()).backward()
    gates = np.concatenate([got[k][0] for k in 'ifgo'], 1)
    b = lo.cell_bwd(dh_in, carry_h, carry_c, gates, got['c'][0], c, H)
    dA = np.concatenate([b[k][0] for k in ('di', 'df', 'dg', 'do')], 1)
    np.testing.assert_allclose(dA, a_t.grad.numpy(), rtol=1e-11, atol=1e-13)
    np.testing.assert_allclose(b['carry_c'][0], cp_t.grad.numpy(), rtol=1e-11, atol=1e-13)
    b0, b1 = lo.cell_bwd(None, carry_h, carry_c, gates, got['c'][0], None, H), lo.cell_bwd(z, carry_h, carry_c, gates, got['c'][0], z, H)
    for k in b0:
        np.testing.assert_array_equal(b0[k][0], b1[k][0])


def _packed_reference(p, pk, emb, neg):
    """The packed training batch composed from the per-kernel references (fp64 GEMMs) the way UserLSTM._forward_backward calls the
    kernels: the h carry is STORED by the carry GEMM, the c carry is the cell's, and both are zeroed once for rows [0, n_0).
    Returns the loss, the four gradients and the states."""
    H, P, T = p['weight_hh_l0'].shape[1], pk.P, len(pk.n)
    Wi, Wh, bi, bh = (p[k] for k in NAMES)
    X = emb[pk.items].astype(np.float64)
    XP = X @ Wi.T + bi
    Hs, Cs, G, Hprev = np.zeros((P, H)), np.zeros((P, H)), np.zeros((P, 4 * H)), np.zeros((P, H))
    for t in range(T):
        o, n = int(pk.off[t]), int(pk.n[t])
        if t:
            Hprev[o:o + n] = Hs[int(pk.off[t - 1]):int(pk.off[t - 1]) + n]
        cprev = Cs[int(pk.off[t - 1]):int(pk.off[t - 1]) + n] if t else None
        f = lo.cell_fwd(XP[o:o + n], Hprev[o:o + n] @ Wh.T + bh, cprev, H)
        Hs[o:o + n], Cs[o:o + n] = f['h'][0], f['c'][0]
        G[o:o + n] = np.concatenate([f[k][0] for k in 'ifgo'], 1)
    dH, _, lt, _ = go.seq_rank_loss(Hs, emb, pk.nxt, neg, 1.0 / pk.terms, H)
    carry_h = np.full((int(pk.n[0]) + 3, H), np.nan)          # rows past n_0 are never read
    carry_c = np.full_like(carry_h, np.nan)
    carry_h[:int(pk.n[0])] = 0
    carry_c[:int(pk.n[0])] = 0
    dA = np.zeros((P, 4 * H))
    for t in range(T - 1, -1, -1):
        o, n = int(pk.off[t]), int(pk.n[t])
        cprev = Cs[int(pk.off[t - 1]):int(pk.off[t - 1]) + n] if t else None
        b = lo.cell_bwd(dH[o:o + n], carry_h[:n], carry_c[:n], G[o:o + n], Cs[o:o + n], cprev, H)
        dA[o:o + n] = np.concatenate([b[k][0] for k in ('di', 'df', 'dg', 'do')], 1)
        carry_c[:n] = b['carry_c'][0]
        if t:
            carry_h[:n] = dA[o:o + n] @ Wh
    g = {'weight_hh_l0': dA.T @ Hprev, 'bias_hh_l0': dA.sum(0), 'weight_ih_l0': dA.T @ X, 'bias_ih_l0': dA.sum(0)}
    return lt.sum() / pk.terms, g, Hs


def test_packed_composition_matches_whole_batch_oracle():
    rng = np.random.default_rng(3)
    H, U, N, max_len = 7, 25, 40, 6
    indptr, items = _seqs(rng, U, N, max_len)
    emb = rng.standard_normal((N, H)).astype(f32)
    p = _params(H, rng, 2.0)
    pk = Packed(indptr, items, np.arange(U), max_len)
    assert (np.diff(pk.n) < 0).any()                           # users end at several steps
    neg = go.seq_negatives(pk.nxt, N, seed=5, epoch=1, batch=2)
    loss, g, Hs = _packed_reference(p, pk, emb, neg)
    assert np.isfinite(loss) and all(np.isfinite(v).all() for v in g.values())
    seqs, negs = [], []
    for i in range(pk.B):
        ps = [pk.position(i, t) for t in range(int(pk.L[i]))]
        seqs.append(pk.items[ps])
        negs.append(neg[ps[:-1]])
    o_loss, o_g, o_states = lo.loss_and_grads(p, seqs, negs, emb)
    sc = float(np.float32(1.0 / pk.terms)) * pk.terms          # the kernel scales dh by fp32(1 / terms)
    np.testing.assert_allclose(loss, o_loss, rtol=1e-12)
    for k in NAMES:
        np.testing.assert_allclose(g[k] / sc, o_g[k], rtol=1e-9, atol=1e-13)
    for i in range(pk.B):
        np.testing.assert_allclose(Hs[[pk.position(i, t) for t in range(int(pk.L[i]))]], o_states[i], rtol=1e-12, atol=1e-14)


# ---------------------------------------------------------------------------------------------------------------------------
# the bounds against float32 emulations of the kernels
# ---------------------------------------------------------------------------------------------------------------------------
MARGIN = 0.5    # the emulation must stay within half the bound


def _sig32(a):
    with np.errstate(over='ignore'):
        return (f32(1) / (f32(1) + np.exp(-a))).astype(f32)


def emu_fwd(xp, hp, cprev, H):
    """float32 emulation of dae_lstm_cell_fwd: (i, f, g, o, c, h)."""
    a = (xp[:, :4 * H] + hp[:, :4 * H]).astype(f32)
    i, f, o = _sig32(a[:, :H]), _sig32(a[:, H:2 * H]), _sig32(a[:, 3 * H:])
    g = np.tanh(a[:, 2 * H:3 * H]).astype(f32)
    cp = np.zeros_like(i) if cprev is None else cprev
    c = (f * cp + i * g).astype(f32)
    return i, f, g, o, c, (o * np.tanh(c)).astype(f32)


def emu_bwd(dh_in, carry_h, carry_c, i, f, g, o, c, cprev):
    """float32 emulation of dae_lstm_cell_bwd: {di, df, dg, do, carry_c}."""
    dh = (carry_h + dh_in).astype(f32)
    tc = np.tanh(c).astype(f32)
    dc = (carry_c + dh * o * (f32(1) - tc * tc)).astype(f32)
    return {'di': (dc * g * i * (f32(1) - i)).astype(f32), 'df': (dc * cprev * f * (f32(1) - f)).astype(f32),
            'dg': (dc * i * (f32(1) - g * g)).astype(f32), 'do': (dh * tc * o * (f32(1) - o)).astype(f32),
            'carry_c': (dc * f).astype(f32)}


def test_cell_bounds_cover_fp32_emulation():
    rng = np.random.default_rng(4)
    H, n = 37, 400
    xp, hp, cprev = lo.lstm_edge_inputs(rng, n, H)
    ref = lo.cell_fwd(xp, hp, cprev, H)
    i, f, g, o, c, h = emu_fwd(xp, hp, cprev, H)
    assert (np.abs(np.tanh(c[2])) == 1).any() and (np.abs(g[1]) == 1).all()     # the edges are reached
    for k, v in zip('ifgoch', (i, f, g, o, c, h)):
        go.check('emu lstm fwd ' + k, v, ref[k][0], ref[k][1], MARGIN * go.C_FP32)
    # backward from the emulated forward
    carry_h = (rng.standard_normal((n, H)) * rng.choice([1e-3, 1.0, 30.0], (n, 1))).astype(f32)
    carry_c = (rng.standard_normal((n, H)) * rng.choice([1e-3, 1.0, 30.0], (n, 1))).astype(f32)
    dh_in = (rng.standard_normal((n, H)) * rng.choice([1e-3, 1.0, 30.0], (n, 1))).astype(f32)
    dh_in[5] = -carry_h[5]                                                     # dh = 0 exactly
    gates = np.concatenate([i, f, g, o], 1)
    ref = lo.cell_bwd(dh_in, carry_h, carry_c, gates, c, cprev, H)
    for k, v in emu_bwd(dh_in, carry_h, carry_c, i, f, g, o, c, cprev).items():
        go.check('emu lstm bwd ' + k, v, ref[k][0], ref[k][1], MARGIN * go.C_FP32)
        hi, lo_ = go.bf16_split(v)
        go.check_pair('emu lstm bwd pair ' + k, hi, lo_, ref[k][0], ref[k][1], go.C_FP32)


# ---------------------------------------------------------------------------------------------------------------------------
# the C ABI without a GPU
# ---------------------------------------------------------------------------------------------------------------------------
def _cabi():
    from dae_rnn_news_recommendation_b200 import _cabi
    return _cabi


P_ = 16   # a non-NULL pointer value: every call below fails its checks before any device work
FWD_OK = dict(n=4, H=4, xp=P_, ld_xp=16, hp=P_, ld_hp=16, c_prev=None, ld_cprev=4, c_out=P_, ld_c=4, h_out=P_, ld_h=4, n_split=4,
              h_hi=None, h_lo=None, ld_split=8, gates=None, ld_gates=16, stream=None)
BWD_OK = dict(n=4, H=4, dh_in=None, ld_dh_in=4, carry_h=P_, ld_carry_h=4, carry_c=P_, ld_carry_c=4, gates=P_, ld_gates=16, c=P_,
              ld_c=4, c_prev=None, ld_cprev=4, da_hi=P_, da_lo=P_, ld_da=16, stream=None)
FWD_BAD = [('n', 0), ('H', 0), ('xp', None), ('hp', None), ('c_out', None), ('h_out', None), ('ld_xp', 15), ('ld_hp', 15),
           ('ld_c', 3), ('ld_h', 3), ({'c_prev': P_, 'ld_cprev': 3}, None), ({'c_prev': P_, 'ld_cprev': 5, 'ld_c': 4}, 'c_out == c_prev'),
           ({'h_hi': P_}, 'split'), ({'h_hi': P_, 'h_lo': P_, 'ld_split': 3}, 'split'), ({'h_hi': P_, 'h_lo': P_, 'n_split': 5}, 'split'),
           ({'h_hi': P_, 'h_lo': P_, 'n_split': -1}, 'split'), ({'gates': P_, 'ld_gates': 15}, 'ld_gates')]
BWD_BAD = [('n', 0), ('H', 0), ('carry_h', None), ('carry_c', None), ('gates', None), ('c', None), ('da_hi', None), ('da_lo', None),
           ('ld_carry_h', 3), ('ld_carry_c', 3), ('ld_gates', 15), ('ld_c', 3), ('ld_da', 15), ({'dh_in': P_, 'ld_dh_in': 3}, None),
           ({'c_prev': P_, 'ld_cprev': 3}, None)]


def _case(ok, change):
    k, v = change
    args = dict(ok)
    if isinstance(k, dict):
        args.update(k)
        return args, v
    args[k] = v
    return args, None


@pytest.mark.parametrize('change', FWD_BAD, ids=[str(c[0]) for c in FWD_BAD])
def test_fwd_bad_arguments(change):
    c = _cabi()
    args, msg = _case(FWD_OK, change)
    with pytest.raises(c.DaeError, match=msg or 'dae_lstm_cell_fwd: bad arguments'):
        c.call('dae_lstm_cell_fwd', *args.values())
    assert c.last_error().startswith('dae_lstm_cell_fwd: ')


@pytest.mark.parametrize('change', BWD_BAD, ids=[str(c[0]) for c in BWD_BAD])
def test_bwd_bad_arguments(change):
    c = _cabi()
    args, _ = _case(BWD_OK, change)
    with pytest.raises(c.DaeError, match='dae_lstm_cell_bwd: bad arguments'):
        c.call('dae_lstm_cell_bwd', *args.values())


def test_last_error_message():
    c = _cabi()
    lib = c.lib()
    rc = getattr(lib, 'dae_lstm_cell_fwd')(*dict(FWD_OK, ld_xp=3).values())
    assert rc != 0
    buf = ctypes.create_string_buffer(512)
    n = lib.dae_last_error(buf, 512)
    assert buf.value.decode() == 'dae_lstm_cell_fwd: bad arguments' and n == len(buf.value)
    rc = getattr(lib, 'dae_lstm_cell_bwd')(*dict(BWD_OK, c=None).values())
    assert rc != 0 and c.last_error() == 'dae_lstm_cell_bwd: bad arguments'


# ---------------------------------------------------------------------------------------------------------------------------
# parameters, save / load, constructor, CLI
# ---------------------------------------------------------------------------------------------------------------------------
def test_state_dict_torch_round_trip_and_init():
    m = UserLSTM(6, seed=3, device='cpu')
    sd = m.state_dict()
    t = torch.nn.LSTM(6, 6)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in t.state_dict().items()}
    t.load_state_dict(sd)
    k = 1.0 / np.sqrt(6)
    assert all(float(v.abs().max()) <= k for v in sd.values())
    assert m.nW == 4 * 6 * 7 and m.theta.numel() == 2 * m.nW
    np.testing.assert_array_equal(m.theta.numpy(), np.random.default_rng(3).uniform(-k, k, 2 * m.nW).astype(f32))
    m2 = UserLSTM(6, seed=5, device='cpu')
    m2.load_state_dict(t.state_dict())
    for name in NAMES:
        assert torch.equal(m2.state_dict()[name], sd[name])
    # theta = [W~_hh | W~_ih], W~ = [W | b] row by row
    hh = m.theta[:m.nW].view(24, 7)
    assert torch.equal(hh[:, :6], sd['weight_hh_l0']) and torch.equal(hh[:, 6], sd['bias_hh_l0'])


def test_load_state_dict_errors():
    m = UserLSTM(4, device='cpu')
    good = m.state_dict()
    with pytest.raises(ValueError, match='UserLSTM.load_state_dict: missing'):
        m.load_state_dict({k: v for k, v in good.items() if k != 'bias_hh_l0'})
    with pytest.raises(ValueError, match='missing'):
        m.load_state_dict(dict({k: v for k, v in good.items() if k != 'weight_ih_l0'}, weight_ih=good['weight_ih_l0']))
    for name in NAMES:
        bad = dict(good)
        bad[name] = torch.zeros(3 * 4, *good[name].shape[1:])                 # GRU-sized
        with pytest.raises(ValueError, match='%s has shape' % name):
            m.load_state_dict(bad)
    with pytest.raises(ValueError, match='shape'):
        m.load_state_dict(UserGRU(4, device='cpu').state_dict())
    with pytest.raises(ValueError, match='shape'):
        UserGRU(4, device='cpu').load_state_dict(good)
    assert torch.equal(m.state_dict()['weight_ih_l0'], good['weight_ih_l0'])   # a refused dict changes nothing


def test_save_load_and_cross_cell_files(tmp_path):
    m = UserLSTM(5, max_len=7, seed=3, device='cpu')
    m.save(tmp_path / 'l.npz')
    m2 = UserLSTM.load(tmp_path / 'l.npz', device='cpu')
    assert m2.dim == 5 and m2.max_len == 7
    for k in NAMES:
        assert torch.equal(m2.state_dict()[k], m.state_dict()[k])
    UserGRU(5, device='cpu').save(tmp_path / 'g.npz')
    with pytest.raises(ValueError, match='UserLSTM.load_state_dict: .*shape'):
        UserLSTM.load(tmp_path / 'g.npz', device='cpu')
    with pytest.raises(ValueError, match='UserGRU.load_state_dict: .*shape'):
        UserGRU.load(tmp_path / 'l.npz', device='cpu')


def test_constructor_checks():
    for kw in (dict(dim=0), dict(dim=4, max_len=0), dict(dim=4, batch_users=0), dict(dim=4, num_epochs=-1)):
        with pytest.raises(ValueError, match='UserLSTM: dim'):
            UserLSTM(device='cpu', **kw)
    with pytest.raises(ValueError, match='UserLSTM: opt'):
        UserLSTM(4, opt='rmsprop', device='cpu')
    m = UserLSTM(4, device='cpu')
    with pytest.raises(ValueError, match='UserLSTM.transform: embeddings are 3 wide'):
        m.transform((np.array([0, 1]), np.array([0])), np.zeros((5, 3), np.float32))
    with pytest.raises(ValueError, match='UserLSTM.fit'):
        m.fit((np.array([0, 2]), np.array([0, 9])), np.zeros((5, 4), np.float32))
    # the same batches as UserGRU for the same seed
    indptr = np.concatenate([[0], np.cumsum(np.arange(50) % 4)]).astype(np.int64)
    a, b = UserLSTM(4, batch_users=7, seed=9, device='cpu'), UserGRU(4, batch_users=7, seed=9, device='cpu')
    for e in (0, 3):
        assert all(np.array_equal(x, y) for x, y in zip(a.batches(indptr, e), b.batches(indptr, e)))


def test_user_cell_flag(tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    p = cli.build_parser()
    assert p.parse_args([]).user_cell == 'gru'
    s = tmp_path / 's.npz'
    np.savez(s, indptr=np.array([0, 1]), items=np.array([0]))
    F = cli.check_flags(p.parse_args(['--top_k', '5', '--user_sequences', str(s), '--user_cell', 'lstm']))
    assert F.user_cell == 'lstm'
    with pytest.raises(SystemExit):
        p.parse_args(['--user_cell', 'rnn'])
