"""CPU checks of tests/gru_kernel_oracle.py: the references against autograd in fp64, torch.nn.GRUCell and the whole-batch oracle
of user_gru_oracle.py; the error bounds against a float32 emulation of each kernel (a bound that a float32 emulation breaks is
wrong); the row arg-max rules; and the C ABI's argument checks and dae_last_error, which need no GPU."""
import ctypes

import numpy as np
import pytest
import torch

import gru_kernel_oracle as go
from user_gru_oracle import NAMES, loss_and_grads

from dae_rnn_news_recommendation_b200.user_model import Packed

f32 = np.float32


def _params(H, rng, scale=1.0):
    k = scale / np.sqrt(H)
    return {'weight_ih_l0': rng.uniform(-k, k, (3 * H, H)), 'weight_hh_l0': rng.uniform(-k, k, (3 * H, H)),
            'bias_ih_l0': rng.uniform(-k, k, 3 * H), 'bias_hh_l0': rng.uniform(-k, k, 3 * H)}


# ---------------------------------------------------------------------------------------------------------------------------
# references against fp64 autograd / torch.nn.GRUCell
# ---------------------------------------------------------------------------------------------------------------------------
def test_cell_fwd_matches_grucell():
    rng = np.random.default_rng(0)
    H, n = 13, 40
    p = _params(H, rng, 3.0)
    x, h = rng.standard_normal((n, H)), rng.standard_normal((n, H))
    cell = torch.nn.GRUCell(H, H).double()
    cell.load_state_dict({k.replace('_l0', ''): torch.from_numpy(v) for k, v in p.items()})
    want = cell(torch.from_numpy(x), torch.from_numpy(h)).detach().numpy()
    xp = x @ p['weight_ih_l0'].T + p['bias_ih_l0']
    hp = h @ p['weight_hh_l0'].T + p['bias_hh_l0']
    got = go.cell_fwd(xp, hp, h, H)
    np.testing.assert_allclose(got['h'][0], want, rtol=1e-12, atol=1e-13)
    np.testing.assert_array_equal(got['hn'][0], hp[:, 2 * H:])
    # h_prev = None is h_prev = 0
    want0 = cell(torch.from_numpy(x), torch.zeros(n, H, dtype=torch.float64)).detach().numpy()
    np.testing.assert_allclose(go.cell_fwd(xp, np.tile(p['bias_hh_l0'], (n, 1)), None, H)['h'][0], want0, rtol=1e-12, atol=1e-13)


def test_cell_bwd_matches_autograd():
    """dXP, dHP and the carry are the gradients of sum(dh * h) with respect to XP, HP and h_prev."""
    rng = np.random.default_rng(1)
    H, n = 11, 30
    xp_t = torch.tensor(rng.standard_normal((n, 3 * H)) * 2, requires_grad=True)
    hp_t = torch.tensor(rng.standard_normal((n, 3 * H)) * 2, requires_grad=True)
    hprev_t = torch.tensor(rng.standard_normal((n, H)), requires_grad=True)
    r = torch.sigmoid(xp_t[:, :H] + hp_t[:, :H])
    z = torch.sigmoid(xp_t[:, H:2 * H] + hp_t[:, H:2 * H])
    nn_ = torch.tanh(xp_t[:, 2 * H:] + r * hp_t[:, 2 * H:])
    h = (1 - z) * nn_ + z * hprev_t
    carry, dh_in = rng.standard_normal((n, H)), rng.standard_normal((n, H))
    (h * torch.from_numpy(carry + dh_in)).sum().backward()
    fwd = go.cell_fwd(xp_t.detach().numpy(), hp_t.detach().numpy(), hprev_t.detach().numpy(), H)
    gates = np.concatenate([fwd[k][0] for k in ('r', 'z', 'n', 'hn')], 1)
    b = go.cell_bwd(dh_in, carry, gates, hprev_t.detach().numpy(), H)
    dxp = np.concatenate([b['dr'][0], b['dz'][0], b['dn'][0]], 1)
    dhp = np.concatenate([b['dr'][0], b['dz'][0], b['rdn'][0]], 1)
    np.testing.assert_allclose(dxp, xp_t.grad.numpy(), rtol=1e-11, atol=1e-13)
    np.testing.assert_allclose(dhp, hp_t.grad.numpy(), rtol=1e-11, atol=1e-13)
    np.testing.assert_allclose(b['carry'][0], hprev_t.grad.numpy(), rtol=1e-11, atol=1e-13)
    # dh_in = None and h_prev = None are zeros
    b0 = go.cell_bwd(None, carry, gates, None, H)
    b1 = go.cell_bwd(np.zeros_like(carry), carry, gates, np.zeros_like(carry), H)
    for k in b0:
        np.testing.assert_array_equal(b0[k][0], b1[k][0])


def test_rank_loss_matches_autograd():
    rng = np.random.default_rng(2)
    H, N, P = 9, 50, 60
    h_t = torch.tensor(rng.standard_normal((P, H)) * 3, requires_grad=True)
    emb = rng.standard_normal((N, H))
    pos = rng.integers(0, N, P)
    pos[::4] = -1
    neg = np.where(pos >= 0, (pos + 1 + rng.integers(0, N - 1, P)) % N, -1)
    has = torch.from_numpy(pos >= 0)
    E = torch.from_numpy(emb)
    x = (h_t * E[torch.from_numpy(np.maximum(neg, 0))]).sum(1) - (h_t * E[torch.from_numpy(np.maximum(pos, 0))]).sum(1)
    terms = (torch.relu(x) + torch.log1p(torch.exp(-x.abs())))[has]   # torch's softplus is linear above x = 20
    scale = 1.0 / float(has.sum())
    (terms.sum() * float(np.float32(scale))).backward()
    dh, s_dh, lt, s_lt = go.seq_rank_loss(h_t.detach().numpy(), emb, pos, neg, scale, H)
    np.testing.assert_allclose(dh, h_t.grad.numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(lt[pos >= 0], terms.detach().numpy(), rtol=1e-12)
    assert (dh[pos < 0] == 0).all() and (lt[pos < 0] == 0).all() and (s_dh[pos < 0] == 0).all()


def _packed_reference(p, pk, emb, neg):
    """The packed training batch composed from the per-kernel references (fp64 GEMMs): loss and the four gradients, in the
    layout user_model.UserGRU uses."""
    H, P, T = p['weight_hh_l0'].shape[1], pk.P, len(pk.n)
    Wi, Wh, bi, bh = (p[k] for k in NAMES)
    X = emb[pk.items].astype(np.float64)
    XP = X @ Wi.T + bi
    Hs, G, Hprev = np.zeros((P, H)), np.zeros((P, 4 * H)), np.zeros((P, H))
    for t in range(T):
        o, n = int(pk.off[t]), int(pk.n[t])
        hprev = Hs[int(pk.off[t - 1]):int(pk.off[t - 1]) + n] if t else None
        if t:
            Hprev[o:o + n] = hprev
        f = go.cell_fwd(XP[o:o + n], (hprev if t else np.zeros((n, H))) @ Wh.T + bh, hprev, H)
        Hs[o:o + n] = f['h'][0]
        G[o:o + n] = np.concatenate([f[k][0] for k in ('r', 'z', 'n', 'hn')], 1)
    dH, _, lt, _ = go.seq_rank_loss(Hs, emb, pk.nxt, neg, 1.0 / pk.terms, H)
    carry = np.zeros((int(pk.n[0]), H))
    dXP, dHP = np.zeros((P, 3 * H)), np.zeros((P, 3 * H))
    for t in range(T - 1, -1, -1):
        o, n = int(pk.off[t]), int(pk.n[t])
        b = go.cell_bwd(dH[o:o + n], carry[:n], G[o:o + n], Hprev[o:o + n] if t else None, H)
        dXP[o:o + n] = np.concatenate([b['dr'][0], b['dz'][0], b['dn'][0]], 1)
        dHP[o:o + n] = np.concatenate([b['dr'][0], b['dz'][0], b['rdn'][0]], 1)
        carry[:n] = b['carry'][0] + (dHP[o:o + n] @ Wh if t else 0.0)
    g = {'weight_hh_l0': dHP.T @ Hprev, 'bias_hh_l0': dHP.sum(0), 'weight_ih_l0': dXP.T @ X, 'bias_ih_l0': dXP.sum(0)}
    return lt.sum() / pk.terms, g, Hs


def test_packed_composition_matches_whole_batch_oracle():
    """The per-kernel references, composed the way UserGRU._forward_backward calls the kernels, give user_gru_oracle's loss,
    gradients and states."""
    rng = np.random.default_rng(3)
    H, U, N, max_len = 7, 25, 40, 6
    lens = rng.integers(1, max_len + 3, U)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N, int(indptr[-1])).astype(np.int32)
    emb = rng.standard_normal((N, H)).astype(np.float32)
    p = _params(H, rng, 2.0)
    pk = Packed(indptr, items, np.arange(U), max_len)
    neg = go.seq_negatives(pk.nxt, N, seed=5, epoch=1, batch=2)
    loss, g, Hs = _packed_reference(p, pk, emb, neg)
    seqs, negs = [], []
    for i in range(pk.B):
        ps = [pk.position(i, t) for t in range(int(pk.L[i]))]
        seqs.append(pk.items[ps])
        negs.append(neg[ps[:-1]])
    o_loss, o_g, o_states = loss_and_grads(p, seqs, negs, emb)
    # the kernel scales dh by fp32(1 / terms); the oracle divides in fp64
    sc = float(np.float32(1.0 / pk.terms)) * pk.terms
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


def _emu_fwd(xp, hp, hprev, H):
    xr, xz, xn = xp[:, :H], xp[:, H:2 * H], xp[:, 2 * H:3 * H]
    hr, hz, hn = hp[:, :H], hp[:, H:2 * H], hp[:, 2 * H:3 * H]
    r, z = _sig32(xr + hr), _sig32(xz + hz)
    n = np.tanh(xn + r * hn).astype(f32)
    hpv = np.zeros_like(n) if hprev is None else hprev
    return r, z, n, hn, ((f32(1) - z) * n + z * hpv).astype(f32)


def test_cell_bounds_cover_fp32_emulation():
    rng = np.random.default_rng(4)
    H, n = 37, 300
    xp, hp, hprev = go.gru_edge_inputs(rng, n, H)
    ref = go.cell_fwd(xp, hp, hprev, H)
    r, z, nn_, hn, h = _emu_fwd(xp, hp, hprev, H)
    for k, v in zip(('r', 'z', 'n', 'h'), (r, z, nn_, h)):
        go.check('emu fwd ' + k, v, ref[k][0], ref[k][1], MARGIN * go.C_FP32)
    # backward from the emulated gates
    gates = np.concatenate([r, z, nn_, hn], 1)
    carry = (rng.standard_normal((n, H)) * rng.choice([1e-3, 1.0, 30.0], (n, 1))).astype(f32)
    dh_in = (rng.standard_normal((n, H)) * rng.choice([1e-3, 1.0, 30.0], (n, 1))).astype(f32)
    dh_in[5] = -carry[5]                                                               # dh = 0 exactly
    ref = go.cell_bwd(dh_in, carry, gates, hprev, H)
    dh = (carry + dh_in).astype(f32)
    dn = (dh * (f32(1) - z) * (f32(1) - nn_ * nn_)).astype(f32)
    dz = (dh * (hprev - nn_) * z * (f32(1) - z)).astype(f32)
    dr = (dn * hn * r * (f32(1) - r)).astype(f32)
    emu = {'dr': dr, 'dz': dz, 'dn': dn, 'rdn': (r * dn).astype(f32), 'carry': (dh * z).astype(f32)}
    for k, v in emu.items():
        go.check('emu bwd ' + k, v, ref[k][0], ref[k][1], MARGIN * go.C_FP32)
        hi, lo = go.bf16_split(v)
        go.check_pair('emu bwd pair ' + k, hi, lo, ref[k][0], ref[k][1], go.C_FP32)


def _warp_dot(a, b):
    """fp32 dot product as the kernels sum it: a sequential fp32 sum per lane (lane j takes j, j + 32, ...), then a tree."""
    H = a.shape[-1]
    pad = (-H) % 32
    a = np.pad(a, [(0, 0), (0, pad)]).reshape(a.shape[0], -1, 32)
    b = np.pad(b, [(0, 0), (0, pad)]).reshape(b.shape[0], -1, 32)
    acc = np.zeros((a.shape[0], 32), f32)
    for k in range(a.shape[1]):
        acc = (acc + a[:, k] * b[:, k]).astype(f32)
    while acc.shape[1] > 1:
        acc = (acc[:, :acc.shape[1] // 2] + acc[:, acc.shape[1] // 2:]).astype(f32)
    return acc[:, 0]


@pytest.mark.parametrize('H', [1, 33, 500])
def test_rank_loss_bounds_cover_fp32_emulation(H):
    rng = np.random.default_rng(5 + H)
    N, P = 300, 400
    emb = rng.standard_normal((N, H)).astype(f32)
    h = (rng.standard_normal((P, H)) * rng.choice([0.1, 1.0, 10.0], (P, 1))).astype(f32)
    pos = rng.integers(0, N, P).astype(np.int32)
    neg = ((pos + 1 + rng.integers(0, N - 1, P)) % N).astype(np.int32)
    pos[::3] = -1
    # x = +-80 and +-90 exactly-ish: h along e(neg) - e(pos)
    for i, x in zip((1, 2, 4, 5, 7, 8, 10, 11), (80.0, -80.0, 90.0, -90.0, 30.0, -30.0, 1e-3, 0.0)):
        d = emb[neg[i]].astype(np.float64) - emb[pos[i]]
        h[i] = (x * d / max(float(d @ d), 1e-30)).astype(f32)
    scale = 1.0 / 777
    dh, s_dh, lt, s_lt = go.seq_rank_loss(h, emb, pos, neg, scale, H)
    has = pos >= 0
    ep, en = emb[np.maximum(pos, 0)], emb[np.maximum(neg, 0)]
    x = (_warp_dot(h, en) - _warp_dot(h, ep)).astype(f32)
    with np.errstate(over='ignore'):
        g = (f32(scale) * _sig32(x)).astype(f32)
        l32 = (np.maximum(x, f32(0)) + np.log1p(np.exp(-np.abs(x)))).astype(f32)
    edh = np.where(has[:, None], g[:, None] * (en - ep), f32(0)).astype(f32)
    go.check('emu loss dh', edh, dh, s_dh, MARGIN * go.C_FP32)
    go.check('emu loss terms', np.where(has, l32, 0.0), lt, s_lt, MARGIN * go.C_FP32)
    go.check('emu loss sum', np.where(has, l32, 0.0).astype(np.float64).sum(), lt.sum(), s_lt.sum(), MARGIN * go.C_FP32)


@pytest.mark.parametrize('kind', [1, 2, 3])
def test_rownorm_bounds_cover_fp32_emulation(kind):
    rng = np.random.default_rng(kind)
    for cols in (1, 33, 4097):
        X = (rng.standard_normal((20, cols)) * rng.choice([1e-6, 1.0, 1e6], (20, 1))).astype(f32)
        X[1] = 0
        X[2] = 0
        X[2, cols // 2] = -3.5
        ref, s = go.rownorm(X, kind)
        Xp = np.pad(X, [(0, 0), (0, (-cols) % 32)]).reshape(20, -1, 32)
        acc = np.zeros((20, 32), f32)
        for k in range(Xp.shape[1]):
            v = Xp[:, k]
            acc = (acc + v * v).astype(f32) if kind == 2 else ((acc + np.abs(v)).astype(f32) if kind == 1 else np.maximum(acc, np.abs(v)))
        while acc.shape[1] > 1:
            m = acc.shape[1] // 2
            acc = np.maximum(acc[:, :m], acc[:, m:]) if kind == 3 else (acc[:, :m] + acc[:, m:]).astype(f32)
        nrm = np.sqrt(acc[:, 0]).astype(f32) if kind == 2 else acc[:, 0]
        with np.errstate(divide='ignore'):
            sc = np.where(acc[:, 0] > 0, f32(1) / nrm, f32(1)).astype(f32)
        go.check('emu rownorm %d' % kind, (X * sc[:, None]).astype(f32), ref, s, MARGIN * go.C_FP32)
        assert (ref[1] == 0).all() and ref[2, cols // 2] == (-1.0 if kind != 0 else -3.5)


def test_gemm_bound_covers_bf16x3_emulation():
    """C_BF16X3 against the three-product bf16 GEMM emulated with fp32 accumulation at K = 3H = 1500."""
    rng = np.random.default_rng(6)
    A = (rng.standard_normal((30, 1500)) * rng.choice([1e-3, 1.0, 1e3], (30, 1))).astype(f32)
    B = rng.standard_normal((20, 1500)).astype(f32)
    want, s = go.gemm_nt(A, B)

    def parts(M):
        hi, lo = go.bf16_split(M)
        return go.bf16_value(hi).astype(f32), go.bf16_value(lo).astype(f32)

    (ah, al), (bh, bl) = parts(A), parts(B)
    acc = np.zeros((30, 20), f32)
    for k in range(0, 1500, 16):   # fp32 accumulation in 16-wide k steps, products exact within a step
        sl = slice(k, k + 16)
        acc = (acc + (ah[:, sl].astype(np.float64) @ bh[:, sl].T.astype(np.float64) + ah[:, sl].astype(np.float64) @
                      bl[:, sl].T.astype(np.float64) + al[:, sl].astype(np.float64) @ bh[:, sl].T.astype(np.float64)).astype(f32)).astype(f32)
    go.check('emu gemm', acc, want, s, MARGIN * go.C_BF16X3)


# ---------------------------------------------------------------------------------------------------------------------------
# bit-exact references
# ---------------------------------------------------------------------------------------------------------------------------
def test_row_argmax_rules():
    inf, nan = np.inf, np.nan
    S = np.array([[1.0, 3.0, 3.0, 2.0],        # tie: the first maximum
                  [nan, 0.5, nan, 0.5],        # NaN skipped, tie
                  [-inf, -inf, -inf, -inf],    # all -inf: the first non-diagonal one
                  [nan, nan, nan, 9.0],        # the diagonal (3, 3) is the only non-NaN: no candidate
                  [-5.0, -1.0, -2.0, -1.0]], np.float32)
    idx, val = go.row_argmax(S, 0)
    assert idx.tolist() == [1, 3, 0, -1, 1]
    assert val[0] == 3.0 and val[1] == 0.5 and val[2] == -inf and val[3] == -inf and val[4] == -1.0
    # np.nanargmax agrees wherever a row has a non-NaN candidate and the diagonal is masked out
    rng = np.random.default_rng(7)
    S = rng.integers(-3, 4, (50, 70)).astype(np.float32)
    S[rng.random(S.shape) < 0.2] = nan
    idx, val = go.row_argmax(S, 10)
    T = S.copy()
    T[np.arange(50), np.arange(50) + 10] = nan
    ok = ~np.isnan(T).all(1)
    assert np.array_equal(idx[ok], np.nanargmax(T[ok], 1)) and np.array_equal(val[ok], np.nanmax(T[ok], 1))
    # diag_offset past the columns: nothing skipped
    assert np.array_equal(go.row_argmax(S, 70)[0][ok], np.nanargmax(S[ok], 1))


def test_gather_split_reference():
    src = np.arange(12, dtype=f32).reshape(3, 4) + f32(1 / 3)
    hi, lo = go.gather_split(src, [2, 0, 2], 3, 8, 5)
    v = go.bf16_value(hi).astype(np.float64) + go.bf16_value(lo)
    np.testing.assert_allclose(v[:, :3], src[[2, 0, 2], :3], rtol=2.0 ** -17)
    assert (v[:, 5] == 1.0).all() and (v[:, [3, 4, 6, 7]] == 0).all()
    assert (go.gather_split(src, [1], 3, 8, -1)[0][:, 3:] == 0).all()


def test_negatives_reference():
    pos = np.array([-1, 0, 1, 998, 999, -5, 3], np.int32)
    neg = go.seq_negatives(pos, 1000, seed=2 ** 40 + 3, epoch=2 ** 33 + 1, batch=7)
    assert neg[0] == -1 and neg[5] == -1
    has = pos >= 0
    assert (neg[has] != pos[has]).all() and (neg[has] >= 0).all() and (neg[has] < 1000).all()
    # two articles: the negative is always the other one
    assert np.array_equal(go.seq_negatives(np.array([0, 1, 1, 0]), 2, 1, 0, 0), [1, 0, 0, 1])


# ---------------------------------------------------------------------------------------------------------------------------
# the C ABI without a GPU: argument checks and dae_last_error
# ---------------------------------------------------------------------------------------------------------------------------
def _lib():
    from dae_rnn_news_recommendation_b200 import _cabi
    return _cabi


BAD_CALLS = [
    ('dae_gather_split_bf16', (None, 4, None, 0, 4, None, None, 8, 4, None)),
    ('dae_gru_cell_fwd', (0, 4, None, 12, None, 12, None, 4, None, 4, 0, None, None, 8, None, 16, None)),
    ('dae_gru_cell_bwd', (4, 0, None, 4, None, 4, None, 16, None, 4, None, None, None, None, 16, None)),
    ('dae_seq_negatives', (None, 10, 1, 0, 0, 0, None, None)),
    ('dae_seq_rank_loss', (None, 4, None, 4, 4, None, None, 0, 1.0, None, 4, None, None)),
    ('dae_rownorm_split_bf16', (None, 1, 1, 1, 2, None, None, 8, None, 0, None)),
    ('dae_row_argmax', (None, 1, 1, 1, 0, 0, None, None, None)),
    ('dae_step_advance', (None, 1, None)),
    ('dae_batch_commit', (0, None, None, None, None, None, None, None, None, None, None, None, None, None)),
    ('dae_batch_prepare_explicit', (None, 0, None, 0, 1, None, None, None)),
    ('dae_col_scan', (None, 0, None, None, None)),
    ('dae_pair_partition', (None, 1, 0, None, None, None, None, None)),
    ('dae_auroc_count', (None, -1, None, 0, 1, None, None)),
    ('dae_allreduce_multimem', (None, None, None, 0, 1, 0, 0, None)),
]


@pytest.mark.parametrize('name,args', BAD_CALLS, ids=[b[0] for b in BAD_CALLS])
def test_bad_arguments_raise_before_any_device_work(name, args):
    c = _lib()
    with pytest.raises(c.DaeError, match=name):
        c.call(name, *args)


def test_last_error_returns_message_and_length():
    c = _lib()
    lib = c.lib()
    assert getattr(lib, 'dae_version')() >= 100
    rc = getattr(lib, 'dae_gru_cell_fwd')(0, 4, None, 12, None, 12, None, 4, None, 4, 0, None, None, 8, None, 16, None)
    assert rc != 0
    buf = ctypes.create_string_buffer(512)
    n = getattr(lib, 'dae_last_error')(buf, 512)
    msg = buf.value.decode()
    assert msg == 'dae_gru_cell_fwd: bad arguments' and n == len(msg)
    # truncated to the buffer, NUL terminated, length of what was copied
    small = ctypes.create_string_buffer(b'\xff' * 8)
    assert lib.dae_last_error(small, 8) == 7 and small.raw[:8] == msg.encode()[:7] + b'\0'
    assert lib.dae_last_error(None, 0) == 0
    # a later failure replaces the message
    with pytest.raises(c.DaeError):
        c.call('dae_seq_negatives', None, 10, 1, 0, 0, 0, None, None)
    assert c.last_error().startswith('dae_seq_negatives: bad arguments (n_pos = 10, n_items = 1')
