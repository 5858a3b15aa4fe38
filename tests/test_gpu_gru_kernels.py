"""The GRU user encoder's kernels (csrc/user_gru.cu) through the C ABI against the fp64 references of tests/gru_kernel_oracle.py,
element by element, and every stage of UserGRU's training batch and transform against its own inputs.  Output buffers start as
sentinels (NaN / -7 in fp32, 0x7F7F in bf16) and every operand has its own leading dimension, so a skipped row or column, a write
past the end and a swapped stride all fail."""
import numpy as np
import pytest
import torch

import gru_kernel_oracle as go

from dae_rnn_news_recommendation_b200 import user_model
from dae_rnn_news_recommendation_b200.user_model import Packed, UserGRU

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF16_SENT = 0x7F7F
f32 = np.float32


def _call(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call(name, *args)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _reach():
    """Elements one pass of a 16-CTA-per-SM grid of 256 threads covers."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _padded(a, ld, fill=0.0):
    """a [rows x cols] fp32 in a [rows x ld] device buffer whose padding holds `fill`."""
    out = np.full((a.shape[0], ld), fill, f32)
    out[:, :a.shape[1]] = a
    return _dev(out)


def _f32_sent(rows, ld, v=float('nan')):
    return torch.full((rows, ld), v, dtype=torch.float32, device=DEV)


def _bf_sent(rows, ld):
    return torch.full((rows, ld), BF16_SENT, dtype=torch.int16, device=DEV)


def _np(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _bits(t):
    torch.cuda.synchronize()
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


# ---------------------------------------------------------------------------------------------------------------------------
# gather + split
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,ones', [(1, True), (7, True), (37, True), (500, True), (1000, True), (37, False)])
def test_gather_split(H, ones):
    rng = np.random.default_rng(H)
    N = 3000
    ld_src = H + 3
    ld_dst = H + 1 if H == 7 else (H + 1 + 7) // 8 * 8 + 8      # H = 7: ldx = H + 1, the ones column last
    ones_col = H if ones else -1
    n_rows = -(-3 * _reach() // ld_dst) + 5                      # three passes of the grid and more
    src = rng.standard_normal((N, H)).astype(f32) * f32(3.0)
    rows = rng.integers(0, N, n_rows).astype(np.int32)
    rows[:4] = [N - 1, N - 1, 0, N - 1]
    rows[-1] = N - 1
    hi, lo = _bf_sent(n_rows + 2, ld_dst), _bf_sent(n_rows + 2, ld_dst)
    src_d, rows_d = _padded(src, ld_src, -7.0), _dev(rows)      # kept alive until the kernel has run
    _call('dae_gather_split_bf16', src_d.data_ptr(), ld_src, rows_d.data_ptr(), n_rows, H, hi.data_ptr(),
          lo.data_ptr(), ld_dst, ones_col, _st())
    w_hi, w_lo = go.gather_split(src, rows, H, ld_dst, ones_col)
    g_hi, g_lo = _bits(hi), _bits(lo)
    assert np.array_equal(g_hi[:n_rows], w_hi) and np.array_equal(g_lo[:n_rows], w_lo)
    assert (g_hi[n_rows:] == BF16_SENT).all() and (g_lo[n_rows:] == BF16_SENT).all()


# ---------------------------------------------------------------------------------------------------------------------------
# cell forward / backward
# ---------------------------------------------------------------------------------------------------------------------------
CELL_N = {1: 4096, 37: 40000, 500: 4096}      # n H spans more than two grid passes at H = 37 and 500


def _fwd_case(H, n, mode, n_split, rng):
    xp, hp, hprev = go.gru_edge_inputs(rng, n, H)
    ld_xp, ld_hp, ld_hprev, ld_h, ld_split, ld_g = 3 * H + 5, 3 * H + 3, H + 2, H + 1, (H + 1 + 7) // 8 * 8 + 8, 4 * H + 7
    xp_d, hp_d = _padded(xp, ld_xp, -7.0), _padded(hp, ld_hp, -7.0)
    if mode == 'alias':                       # h_out is h_prev, as transform() calls it
        ld_h = ld_hprev
        h_out = _padded(np.concatenate([hprev, np.full((2, H), -7.0, f32)]), ld_h, np.nan)
        hprev_d = h_out
    else:
        h_out = _f32_sent(n + 2, ld_h)
        hprev_d = None if mode == 'noprev' else _padded(hprev, ld_hprev, -7.0)
    want = go.cell_fwd(xp, hp, None if mode == 'noprev' else hprev, H)
    split = mode != 'nosplit'
    h_hi, h_lo = _bf_sent(n + 2, ld_split), _bf_sent(n + 2, ld_split)
    gates = None if mode == 'nogates' else _f32_sent(n + 2, ld_g)
    _call('dae_gru_cell_fwd', n, H, xp_d.data_ptr(), ld_xp, hp_d.data_ptr(), ld_hp, None if hprev_d is None else hprev_d.data_ptr(),
          ld_hprev if mode != 'alias' else ld_h, h_out.data_ptr(), ld_h, n_split, h_hi.data_ptr() if split else None,
          h_lo.data_ptr() if split else None, ld_split, None if gates is None else gates.data_ptr(), ld_g, _st())
    h = _np(h_out)
    go.check('fwd h H=%d %s' % (H, mode), h[:n, :H], *want['h'], go.C_FP32)
    assert np.isnan(h[:n, H:]).all() and (np.isnan(h[n:]) | (h[n:] == -7.0)).all()
    hb, lb = _bits(h_hi), _bits(h_lo)
    if split:
        w_hi, w_lo = go.bf16_split(h[:n_split, :H])
        assert np.array_equal(hb[:n_split, :H], w_hi) and np.array_equal(lb[:n_split, :H], w_lo)
        assert (hb[n_split:] == BF16_SENT).all() and (hb[:, H:] == BF16_SENT).all() and (lb[n_split:] == BF16_SENT).all()
    else:
        assert (hb == BF16_SENT).all() and (lb == BF16_SENT).all()
    if gates is not None:
        g = _np(gates)
        for k, name in enumerate(('r', 'z', 'n')):
            go.check('fwd %s H=%d' % (name, H), g[:n, k * H:(k + 1) * H], *want[name], go.C_FP32)
        assert np.array_equal(g[:n, 3 * H:4 * H], hp[:, 2 * H:])
        assert np.isnan(g[:n, 4 * H:]).all() and np.isnan(g[n:]).all()
    return h


@pytest.mark.parametrize('H', [1, 37, 500])
def test_cell_fwd(H):
    rng = np.random.default_rng(10 + H)
    n = CELL_N[H]
    for n_split in (0, 1, n - 1, n):
        _fwd_case(H, n, 'full', n_split, rng)
    for mode in ('noprev', 'alias', 'nogates', 'nosplit'):
        _fwd_case(H, n, mode, n, rng)


def _bwd_case(H, n, rng, dh_in_null=False, hprev_null=False):
    xp, hp, hprev = go.gru_edge_inputs(rng, n, H)
    fw = go.cell_fwd(xp, hp, hprev, H)
    gates = np.concatenate([fw[k][0] for k in ('r', 'z', 'n', 'hn')], 1).astype(f32)
    carry = (rng.standard_normal((n, H)) * rng.choice([1e-3, 1.0, 30.0], (n, 1))).astype(f32)
    dh_in = (rng.standard_normal((n, H)) * rng.choice([1e-3, 1.0, 30.0], (n, 1))).astype(f32)
    ld_dh, ld_c, ld_gt, ld_hp, ld_g = H + 1, H + 3, 4 * H + 5, H + 2, (3 * H + 7) // 8 * 8 + 8
    extra = rng.standard_normal((3, H)).astype(f32)                     # carry rows >= n: untouched
    carry_d = _padded(np.concatenate([carry, extra]), ld_c, -7.0)
    dh_d = None if dh_in_null else _padded(dh_in, ld_dh, -7.0)
    hp_d = None if hprev_null else _padded(hprev, ld_hp, -7.0)
    bufs = [_bf_sent(n + 2, ld_g) for _ in range(4)]
    gates_d = _padded(gates, ld_gt, -7.0)
    _call('dae_gru_cell_bwd', n, H, None if dh_d is None else dh_d.data_ptr(), ld_dh, carry_d.data_ptr(), ld_c,
          gates_d.data_ptr(), ld_gt, None if hp_d is None else hp_d.data_ptr(), ld_hp,
          *[b.data_ptr() for b in bufs], ld_g, _st())
    want = go.cell_bwd(None if dh_in_null else dh_in, carry, gates, None if hprev_null else hprev, H)
    c = _np(carry_d)
    go.check('bwd carry H=%d' % H, c[:n, :H], *want['carry'], go.C_FP32)
    assert np.array_equal(c[n:, :H], extra) and (c[:, H:] == -7.0).all()
    xh, xl, ph, pl = (_bits(b) for b in bufs)
    for k, name in enumerate(('dr', 'dz', 'dn')):
        sl = slice(k * H, (k + 1) * H)
        go.check_pair('bwd dXP %s H=%d' % (name, H), xh[:n, sl], xl[:n, sl], *want[name], go.C_FP32)
    assert np.array_equal(ph[:n, :2 * H], xh[:n, :2 * H]) and np.array_equal(pl[:n, :2 * H], xl[:n, :2 * H])
    go.check_pair('bwd dHP r dn H=%d' % H, ph[:n, 2 * H:3 * H], pl[:n, 2 * H:3 * H], *want['rdn'], go.C_FP32)
    for b in (xh, xl, ph, pl):
        assert (b[n:] == BF16_SENT).all() and (b[:, 3 * H:] == BF16_SENT).all()


@pytest.mark.parametrize('H', [1, 37, 500])
def test_cell_bwd(H):
    rng = np.random.default_rng(20 + H)
    n = CELL_N[H]
    _bwd_case(H, n, rng)
    _bwd_case(H, n, rng, dh_in_null=True)
    _bwd_case(H, n, rng, hprev_null=True)
    _bwd_case(H, 1, rng)


# ---------------------------------------------------------------------------------------------------------------------------
# ranking loss and negatives
# ---------------------------------------------------------------------------------------------------------------------------
def _loss_inputs(rng, H, n_pos, N=1000):
    emb = rng.standard_normal((N, H)).astype(f32)
    h = (rng.standard_normal((n_pos, H)) * rng.choice([0.1, 1.0, 5.0], (n_pos, 1))).astype(f32)
    pos = rng.integers(0, N, n_pos).astype(np.int32)
    neg = ((pos + 1 + rng.integers(0, N - 1, n_pos)) % N).astype(np.int32)
    for i, x in zip(range(1, 9), (90.0, -90.0, 80.0, -80.0, 30.0, -30.0, 1e-3, 0.0)):   # x = s- - s+ up to +-90
        if i < n_pos:
            d = emb[neg[i]].astype(np.float64) - emb[pos[i]]
            h[i] = (x * d / max(float(d @ d), 1e-30)).astype(f32)
    drop = rng.random(n_pos) < 1 / 3
    drop[0] = n_pos > 1
    pos[drop] = np.where(rng.random(int(drop.sum())) < 0.5, -1, -5)
    return emb, h, pos, neg


@pytest.mark.parametrize('H,n_pos', [(1, 1), (1, 100000), (31, 8), (31, 16897), (32, 16897), (32, 100000), (33, 8), (33, 100000),
                                     (500, 1), (500, 16897)])
def test_seq_rank_loss(H, n_pos):
    rng = np.random.default_rng(H * 7 + n_pos)
    emb, h, pos, neg = _loss_inputs(rng, H, n_pos)
    ld_h, ld_e, ld_dh = H + 1, H + 3, H + 2
    scale = 1.0 / 777
    dh = _f32_sent(n_pos + 2, ld_dh)
    loss = torch.full((1,), 1.25, dtype=torch.float64, device=DEV)    # the kernel accumulates onto it
    ins = [_padded(h, ld_h, -7.0), _padded(emb, ld_e, -7.0), _dev(pos), _dev(neg)]
    _call('dae_seq_rank_loss', ins[0].data_ptr(), ld_h, ins[1].data_ptr(), ld_e, H, ins[2].data_ptr(), ins[3].data_ptr(), n_pos, scale, dh.data_ptr(), ld_dh, loss.data_ptr(), _st())
    w_dh, s_dh, lt, s_lt = go.seq_rank_loss(h, emb, pos, neg, scale, H)
    g = _np(dh)
    go.check('loss dh H=%d' % H, g[:n_pos, :H], w_dh, s_dh, go.C_FP32)
    assert (g[:n_pos][pos < 0, :H] == 0).all() and np.isnan(g[:, H:]).all() and np.isnan(g[n_pos:]).all()
    go.check('loss sum H=%d' % H, float(_np(loss)[0]) - 1.25, lt.sum(), s_lt.sum(), go.C_FP32, tiny=1e-15)


@pytest.mark.parametrize('n_items', [2, 3, 1000, 2 ** 31 - 1])
def test_seq_negatives(n_items):
    rng = np.random.default_rng(n_items % 1000)
    n_pos = 2_000_000
    pos = rng.integers(0, n_items, n_pos, dtype=np.int64).astype(np.int32)
    pos[rng.random(n_pos) < 0.2] = -1
    pos[:4] = [-1, n_items - 1, 0, n_items - 1]
    pos[-1] = n_items - 1
    seed, epoch, batch = 2 ** 32 + 12345, 2 ** 33 + 7, 2 ** 20 + 3
    neg = torch.full((n_pos + 2,), -7, dtype=torch.int32, device=DEV)
    pos_d = _dev(pos)
    _call('dae_seq_negatives', pos_d.data_ptr(), n_pos, n_items, seed, epoch, batch, neg.data_ptr(), _st())
    got = _np(neg)
    want = go.seq_negatives(pos, n_items, seed, epoch, batch)
    assert np.array_equal(got[:n_pos], want), np.flatnonzero(got[:n_pos] != want)[:5]
    assert (got[n_pos:] == -7).all()
    has = pos >= 0
    assert (got[:n_pos][has] != pos[has]).all()


# ---------------------------------------------------------------------------------------------------------------------------
# the composed batch: every kernel call of UserGRU._forward_backward / transform against its own inputs
# ---------------------------------------------------------------------------------------------------------------------------
class _CAI:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {'data': (int(ptr), False), 'shape': tuple(shape), 'typestr': typestr, 'version': 3}


def _snap(ptr, rows, ld, kind='f4'):
    """A copy of the device buffer [rows x ld] at ptr (fp32 'f4' or bf16 bits 'u2') as a NumPy array."""
    if ptr is None or rows <= 0:
        return None
    t = torch.as_tensor(_CAI(ptr, (rows, ld), '<f4' if kind == 'f4' else '<i2'), device=DEV).clone()
    torch.cuda.synchronize()
    a = t.cpu().numpy()
    return a if kind == 'f4' else a.view(np.uint16)


def _snap_vec(ptr, n, typestr):
    t = torch.as_tensor(_CAI(ptr, (n,), typestr), device=DEV).clone()
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _pair_value(hi, lo):
    return go.bf16_value(hi).astype(np.float64) + go.bf16_value(lo)


class Recorder:
    """Stands in for user_model.call: snapshots each kernel's inputs, runs it, synchronizes and snapshots its outputs."""

    def __init__(self, real):
        self.real, self.log = real, []

    def __call__(self, name, *a):
        pre, post = {}, {}
        if name == 'dae_gru_cell_fwd':
            n, H = a[0], a[1]
            pre = {'xp': _snap(a[2], n, a[3]), 'hp': _snap(a[4], n, a[5]), 'h_prev': _snap(a[6], n, a[7])}
        elif name == 'dae_gru_cell_bwd':
            n, H = a[0], a[1]
            pre = {'dh_in': _snap(a[2], n, a[3]), 'carry': _snap(a[4], a[0], a[5]), 'gates': _snap(a[6], n, a[7]),
                   'h_prev': _snap(a[8], n, a[9])}
        elif name == 'dae_gemm_bf16x3':
            M, N, K = a[0], a[1], a[2]
            ra, rb = (K if a[7] else M), (K if a[11] else N)
            pre = {'a': _pair_value(_snap(a[4], ra, a[6], 'u2'), _snap(a[5], ra, a[6], 'u2')),
                   'b': _pair_value(_snap(a[8], rb, a[10], 'u2'), _snap(a[9], rb, a[10], 'u2')),
                   'c': _snap(a[12], M, a[13]) if a[18] else None}
        elif name == 'dae_seq_rank_loss':
            pre = {'h': _snap(a[0], a[7], a[1]), 'pos': _snap_vec(a[5], a[7], '<i4'), 'neg': _snap_vec(a[6], a[7], '<i4'),
                   'loss': _snap_vec(a[11], 1, '<f8')}
        elif name == 'dae_seq_negatives':
            pre = {'pos': _snap_vec(a[0], a[1], '<i4')}
        elif name == 'dae_gather_split_bf16':
            pre = {'rows': _snap_vec(a[2], a[3], '<i4')}
        self.real(name, *a)
        torch.cuda.synchronize()
        if name == 'dae_gru_cell_fwd':
            n, H = a[0], a[1]
            post = {'h': _snap(a[8], n, a[9]), 'h_hi': _snap(a[11], a[10], a[13], 'u2') if a[11] else None,
                    'h_lo': _snap(a[12], a[10], a[13], 'u2') if a[11] else None, 'gates': _snap(a[14], n, a[15]) if a[14] else None}
        elif name == 'dae_gru_cell_bwd':
            n = a[0]
            post = {'carry': _snap(a[4], n, a[5])}
            post.update({k: _snap(a[10 + i], n, a[14], 'u2') for i, k in enumerate(('dxp_hi', 'dxp_lo', 'dhp_hi', 'dhp_lo'))})
        elif name == 'dae_gemm_bf16x3':
            post = {'c': _snap(a[12], a[0], a[13])}
        elif name == 'dae_seq_rank_loss':
            post = {'dh': _snap(a[9], a[7], a[10]), 'loss': _snap_vec(a[11], 1, '<f8')}
        elif name == 'dae_seq_negatives':
            post = {'neg': _snap_vec(a[6], a[1], '<i4')}
        elif name == 'dae_gather_split_bf16':
            post = {'hi': _snap(a[5], a[3], a[7], 'u2'), 'lo': _snap(a[6], a[3], a[7], 'u2')}
        self.log.append((name, a, pre, post))


def _check_log(log, emb, H, tag):
    """Every recorded kernel call against the fp64 reference of its own inputs; returns the calls by name."""
    by = {}
    prev_bwd_n = None
    for name, a, pre, post in log:
        by.setdefault(name, []).append((a, pre, post))
        if name == 'dae_gru_cell_fwd':
            n = a[0]
            want = go.cell_fwd(pre['xp'], pre['hp'], pre['h_prev'], H)
            go.check('%s fwd h' % tag, post['h'][:, :H], *want['h'], go.C_FP32)
            if post['gates'] is not None:
                for k, g in enumerate(('r', 'z', 'n')):
                    go.check('%s fwd %s' % (tag, g), post['gates'][:, k * H:(k + 1) * H], *want[g], go.C_FP32)
                assert np.array_equal(post['gates'][:, 3 * H:4 * H], pre['hp'][:, 2 * H:3 * H])
            if post['h_hi'] is not None:
                w_hi, w_lo = go.bf16_split(post['h'][:a[10], :H])
                assert np.array_equal(post['h_hi'][:, :H], w_hi) and np.array_equal(post['h_lo'][:, :H], w_lo)
        elif name == 'dae_gru_cell_bwd':
            n = a[0]
            c0 = pre['carry'][:, :H]
            # rows of users whose last read is at this step carry nothing from later steps
            lo_row = 0 if prev_bwd_n is None else prev_bwd_n
            assert (c0[lo_row:] == 0).all(), '%s: carry rows [%d, %d) not zero' % (tag, lo_row, n)
            prev_bwd_n = n
            want = go.cell_bwd(pre['dh_in'], c0, pre['gates'], pre['h_prev'], H)
            go.check('%s bwd carry' % tag, post['carry'][:, :H], *want['carry'], go.C_FP32)
            for k, g in enumerate(('dr', 'dz', 'dn')):
                sl = slice(k * H, (k + 1) * H)
                go.check_pair('%s bwd %s' % (tag, g), post['dxp_hi'][:, sl], post['dxp_lo'][:, sl], *want[g], go.C_FP32)
            assert np.array_equal(post['dhp_hi'][:, :2 * H], post['dxp_hi'][:, :2 * H])
            assert np.array_equal(post['dhp_lo'][:, :2 * H], post['dxp_lo'][:, :2 * H])
            go.check_pair('%s bwd r dn' % tag, post['dhp_hi'][:, 2 * H:3 * H], post['dhp_lo'][:, 2 * H:3 * H], *want['rdn'], go.C_FP32)
        elif name == 'dae_gemm_bf16x3':
            M, N, K = a[0], a[1], a[2]
            A = pre['a'].T[:M, :K] if a[7] else pre['a'][:M, :K]
            B = pre['b'].T[:N, :K] if a[11] else pre['b'][:N, :K]
            want, s = go.gemm_nt(A, B)
            want, s = a[3] * want, abs(a[3]) * s
            if a[18]:
                want, s = want + pre['c'][:, :N], s + np.abs(pre['c'][:, :N])
            go.check('%s gemm %dx%dx%d' % (tag, M, N, K), post['c'][:, :N], want, s, go.C_BF16X3)
        elif name == 'dae_seq_rank_loss':
            w_dh, s_dh, lt, s_lt = go.seq_rank_loss(pre['h'], emb, pre['pos'], pre['neg'], a[8], H)
            go.check('%s loss dh' % tag, post['dh'][:, :H], w_dh, s_dh, go.C_FP32)
            assert (post['dh'][pre['pos'] < 0, :H] == 0).all()
            go.check('%s loss sum' % tag, post['loss'][0] - pre['loss'][0], lt.sum(), s_lt.sum(), go.C_FP32, tiny=1e-15)
        elif name == 'dae_seq_negatives':
            assert np.array_equal(post['neg'], go.seq_negatives(pre['pos'], a[2], a[3], a[4], a[5]))
        elif name == 'dae_gather_split_bf16':
            w_hi, w_lo = go.gather_split(emb, pre['rows'], a[4], a[7], a[8])
            assert np.array_equal(post['hi'], w_hi) and np.array_equal(post['lo'], w_lo)
    return by


def _data(U, H, N, max_len, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 4, U)
    lens[:6] = [1, 2, max_len, max_len + 3, 2 * max_len, 1]
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N, int(indptr[-1])).astype(np.int32)
    emb = (rng.standard_normal((N, H)) * 0.5).astype(f32)
    return indptr, items, emb


@pytest.mark.parametrize('H,U,max_len', [(37, 300, 10), (37, 2600, 12), (7, 200, 9)])
def test_training_batch_every_stage(H, U, max_len, monkeypatch):
    N = 900
    indptr, items, emb = _data(U, H, N, max_len, seed=H + U)
    m = UserGRU(H, max_len=max_len, batch_users=U, seed=3, learning_rate=1e-2)
    emb_d = _dev(emb)
    small = Packed(indptr, items, np.arange(min(U, 40)), max_len)    # the buffers first hold a smaller batch, then grow
    m._forward_backward(small, emb_d, 0, 0)
    m._optimizer_step()
    pk = Packed(indptr, items, np.arange(U), max_len)
    if U > 2000:
        assert pk.P > 16896                                              # more positions than the loss kernel's grid covers
    b = m._buffers(pk.P, pk.B)
    for k in ('neg', 'XP', 'HP', 'Hs', 'gates', 'dH', 'carry'):                 # sentinels in every buffer a kernel fills
        b[k].fill_(-7 if k == 'neg' else float('nan'))
    for k in ('X_hl', 'dXP_hl', 'dHP_hl'):
        for t in b[k]:
            t.view(torch.int16).fill_(BF16_SENT)
    rec = Recorder(user_model.call)
    monkeypatch.setattr(user_model, 'call', rec)
    m.stats.zero_()
    m._forward_backward(pk, emb_d, 5, 3)
    m._optimizer_step()
    torch.cuda.synchronize()
    tag = 'train H=%d U=%d' % (H, U)
    by = _check_log(rec.log, emb, H, tag)
    T = len(pk.n)
    assert len(by['dae_gru_cell_fwd']) == T and len(by['dae_gru_cell_bwd']) == T
    # the recurrent GEMM of step t reads [h_{t-1} | 1 | 0 ...]: the forward cell's fp32 states of step t-1, bit for bit
    Hs = m._buf['Hs'][:pk.P].cpu().numpy()
    gemms = [g for g in by['dae_gemm_bf16x3'] if g[0][2] == H + 1 and g[0][1] == 3 * H]
    hp_gemms = gemms[1:1 + T]
    for t, (a, pre, post) in enumerate(hp_gemms):
        n = int(pk.n[t])
        assert a[0] == n
        A = pre['a']
        prev = Hs[int(pk.off[t - 1]):int(pk.off[t - 1]) + n] if t else np.zeros((n, H), f32)
        assert np.array_equal(A[:n, :H], _pair_value(*go.bf16_split(prev))), (tag, t)
        assert (A[:n, H] == 1.0).all() and (A[:n, H + 1:] == 0).all(), (tag, t)
    # the weight gradients, K = positions
    Hp_hi, Hp_lo = m._buf['Hp_hl']
    Hp = _pair_value(_bits(Hp_hi[:pk.P]), _bits(Hp_lo[:pk.P]))
    assert (Hp[:, H] == 1.0).all() and (Hp[:, H + 1:] == 0).all()
    wg = [g for g in by['dae_gemm_bf16x3'] if g[0][2] == pk.P]
    assert len(wg) == 2
    # the loss: every term, summed into the stats slot
    assert by['dae_seq_rank_loss'][0][0][7] == pk.P
    # after the optimizer step the recurrent GEMM's bf16 copy of W_hh is the split of the new theta_hh
    hi, lo = m.W_hl['hh']
    w_hi, w_lo = go.bf16_split(m._theta('hh').cpu().numpy())
    assert np.array_equal(_bits(hi)[:, :H + 1], w_hi) and np.array_equal(_bits(lo)[:, :H + 1], w_lo)
    print(tag, {k: round(v, 4) for k, v in go.WORST.items() if k.startswith(tag)})


def test_transform_every_stage(monkeypatch):
    H, U, N, max_len = 37, 333, 700, 12
    indptr, items, emb = _data(U, H, N, max_len, seed=9)
    m = UserGRU(H, max_len=max_len, batch_users=150, seed=4)
    rec = Recorder(user_model.call)
    monkeypatch.setattr(user_model, 'call', rec)
    out = m.transform((indptr, items), emb)
    by = _check_log(rec.log, emb, H, 'transform')
    for a, pre, post in by['dae_gru_cell_fwd']:
        assert a[6] == a[8] and a[10] == a[0] and a[14] is None       # h_out == h_prev, n_split = n, no gates
    assert out.shape == (U, H) and np.isfinite(out).all()
