"""The impression kernels (csrc/impressions.cu) through the C ABI against the fp64 references of tests/impression_kernel_oracle.py,
element by element, and every dae_impression_rank_loss call of real UserGRU / UserLSTM / UserAttention impression batches against its own
inputs.  Outputs start as sentinels, every operand has its own leading dimension with NaN in the padding, and the row counts run
the grid-stride loops past three passes, so a wrong stride, a skipped row or a write past the end fails."""
import numpy as np
import pytest
import torch

import impression_kernel_oracle as ko
import impression_oracle as io
from helpers import snap, snap_vec

from dae_rnn_news_recommendation_b200 import _cabi, helpers, user_model
from dae_rnn_news_recommendation_b200.user_model import (ImpressionBatch, Packed, UserAttention, UserGRU, UserLSTM, check_impressions,
                                                         usable_impressions)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
f32 = np.float32
SCORE_SENT = -12345.0
METRIC_SENT = -3.5


def _st():
    return torch.cuda.current_stream().cuda_stream


def _pass_rows():
    """Rows (positions or impressions) one pass of the impression kernels' grid covers: 16 CTAs of 4 warps per SM."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 4


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _padded(a, ld, fill=np.nan):
    out = np.full((a.shape[0], ld), fill, f32)
    out[:, :a.shape[1]] = a
    return _dev(out)


def _np(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _print_worst(prefix):
    print(prefix, {k: round(v, 4) for k, v in ko.WORST.items() if k.startswith(prefix)})


# ---------------------------------------------------------------------------------------------------------------------------
# (a) dae_impression_rank_loss
# ---------------------------------------------------------------------------------------------------------------------------
def _loss_call(ins, H, n_pos, ld, scale, extra=3, loss0=1.25):
    h_d, e_d, pi_d, ip_d, it_d, c_d = ins
    ld_h, ld_e, ld_dh = ld
    dh = torch.full((n_pos + extra, ld_dh), float('nan'), dtype=torch.float32, device=DEV)
    loss = torch.full((1,), loss0, dtype=torch.float64, device=DEV)
    _cabi.call('dae_impression_rank_loss', h_d.data_ptr(), ld_h, e_d.data_ptr(), ld_e, H, pi_d.data_ptr(), n_pos, ip_d.data_ptr(),
               it_d.data_ptr(), c_d.data_ptr(), scale, dh.data_ptr(), ld_dh, loss.data_ptr(), _st())
    return _np(dh), float(_np(loss)[0]) - loss0


@pytest.mark.parametrize('H', [1, 31, 32, 33, 37, 500])
def test_rank_loss(H):
    rng = np.random.default_rng(1000 + H)
    n_pos = 3 * _pass_rows() + 37
    h, emb, pi, ip, items, clicked, info = ko.loss_case(rng, H, n_pos)
    ld = (H + 1, H + 3, H + 2)
    ins = [_padded(h, ld[0]), _padded(emb, ld[1]), _dev(pi), _dev(ip), _dev(items), _dev(clicked)]
    scale = 1.0 / 29
    dh, loss = _loss_call(ins, H, n_pos, ld, scale)
    w_dh, s_dh, w_loss, s_loss = ko.rank_loss(h, emb, pi, ip, items, clicked, scale, H)
    tag = 'loss H=%d' % H
    ko.check(tag + ' dh', dh[:n_pos, :H], w_dh, s_dh, ko.C_FP32)
    ko.check(tag + ' sum', loss, w_loss, s_loss, ko.C_FP32, tiny=1e-15)
    # rows without a usable impression are exactly 0; padding columns and rows past n_pos stay NaN
    used = np.repeat(np.arange(n_pos), np.diff(pi))[ko.usable(ip, clicked)[:pi[-1]]]
    none = np.setdiff1d(np.arange(n_pos), used)
    assert set(info['skipped_only']) <= set(none) and none.size > n_pos // 2
    assert (dh[none, :H] == 0).all()
    assert np.isnan(dh[:, H:]).all() and np.isnan(dh[n_pos:]).all()
    # impressions reach every pass of the grid, the 5 000-article ones included
    assert np.isin(np.arange(4), used // _pass_rows()).all() and (np.diff(ip) == 5000).sum() == 2
    # deterministic: the same bits again
    dh2, loss2 = _loss_call(ins, H, n_pos, ld, scale)
    assert np.array_equal(dh.view(np.uint32), dh2.view(np.uint32))
    _print_worst(tag)


# ---------------------------------------------------------------------------------------------------------------------------
# (b) dae_impression_metrics
# ---------------------------------------------------------------------------------------------------------------------------
def _metrics_call(q, emb, ip, items, clicked, cosine, H, ld_q, ld_e, extra=5):
    n_imp, nnz = len(ip) - 1, int(ip[-1])
    ins = [_padded(q, ld_q), _padded(emb, ld_e), _dev(ip), _dev(items), _dev(clicked)]
    scores = torch.full((nnz + 40,), SCORE_SENT, dtype=torch.float32, device=DEV)
    metrics = torch.full((n_imp + extra, 4), METRIC_SENT, dtype=torch.float64, device=DEV)
    _cabi.call('dae_impression_metrics', ins[0].data_ptr(), ld_q, ins[1].data_ptr(), ld_e, H, int(cosine), ins[2].data_ptr(),
               ins[3].data_ptr(), ins[4].data_ptr(), n_imp, scores.data_ptr(), metrics.data_ptr(), _st())
    s, m = _np(scores), _np(metrics)
    assert (s[nnz:] == SCORE_SENT).all() and (m[n_imp:] == METRIC_SENT).all()
    return s[:nnz], m[:n_imp]


def _check_metrics(tag, s, m, ip, clicked):
    """The kernel's metrics against impression_oracle.metrics on the kernel's own scores: AUC and its integer numerator exactly,
    MRR and nDCG within 1e-12; NaN rows exactly where there is no click or no non-click."""
    want, ints = io.metrics(s, ip, clicked)
    nan = np.isnan(want[:, 0])
    assert np.array_equal(np.isnan(m), np.repeat(nan[:, None], 4, 1)), tag
    ok = ~nan
    n_c = np.diff(np.concatenate([[0], np.cumsum(clicked, dtype=np.int64)])[ip])
    n_n = np.diff(ip) - n_c
    assert np.array_equal(m[ok, 0], want[ok, 0]), tag
    assert np.array_equal(np.rint(m[ok, 0] * 2 * n_c[ok] * n_n[ok]).astype(np.int64), ints[ok, 0]), tag
    np.testing.assert_allclose(m[ok], want[ok], rtol=1e-12, atol=0, err_msg=tag)
    return want, ints


@pytest.mark.parametrize('cosine', [False, True])
@pytest.mark.parametrize('H', [1, 33, 500])
def test_metrics(H, cosine):
    rng = np.random.default_rng(2000 + H + cosine)
    n_imp = 3 * _pass_rows() + 21
    q, emb, ip, items, clicked, info = ko.metrics_case(rng, H, n_imp)
    s, m = _metrics_call(q, emb, ip, items, clicked, cosine, H, H + 1, H + 3)
    tag = 'metrics H=%d cos=%d' % (H, cosine)
    want_s, scale = ko.scores(q, emb, ip, items, cosine, H)
    ko.check(tag + ' scores', s, want_s, scale, ko.C_FP32)        # skipped impressions' scores included
    zq = info['zero_query']
    assert (s[ip[zq]:ip[zq + 1]] == 0).all()
    if cosine:
        assert (s[np.isin(items, info['zero_items'])] == 0).all()
    want, ints = _check_metrics(tag, s, m, ip, clicked)
    # the edges were reached on the kernel's own scores
    first = s[ip[0]:ip[1]]
    assert first[250] == first[255] == first[256] == first[257] == first[260]
    for i, r in info['rank'].items():
        assert ints[i, 1] == r, (tag, i, r)
    assert np.isnan(want[np.diff(ip) <= 1, 0]).all() and (np.diff(ip) == 0).any()
    _print_worst(tag)


def _range_case(H, v_q, v_e):
    """One impression of two articles: q = v_q (all entries), article 0 = v_e, article 1 = -v_e; click on article 0."""
    q = np.full((1, H), v_q, f32)
    emb = np.stack([np.full(H, v_e, f32), np.full(H, -v_e, f32)])
    ip, items, clicked = np.array([0, 2]), np.array([0, 1], np.int32), np.array([1, 0], np.uint8)
    return q, emb, ip, items, clicked


@pytest.mark.parametrize('H', [37, 64])
def test_cosine_scores_at_the_ends_of_the_fp32_range(H):
    """What DESIGN 4.13 and dae_sm100.h state.  Entries of 2^-80 (squared norms underflow to 0) score 0, as zero vectors do.
    Entries of 2^-68 (subnormal squared norms) score finitely.  At impression_metrics' limit 2^63 / sqrt(H) every score is
    finite and the helper accepts the inputs; at 2^64 the fp32 sums overflow, the kernel gives NaN and the helper refuses them."""
    lim = f32(2.0 ** 63 / np.sqrt(H))
    lim = lim if float(lim) <= 2.0 ** 63 / np.sqrt(H) else np.nextafter(lim, f32(0))
    for v, expect in ((2.0 ** -80, 'zero'), (2.0 ** -68, 'finite'), (float(lim), 'one'), (2.0 ** 64, 'nan')):
        q, emb, ip, items, clicked = _range_case(H, v, v)
        s, m = _metrics_call(q, emb, ip, items, clicked, True, H, H + 1, H + 3)
        if expect == 'zero':
            assert (s == 0).all(), (H, v, s)
        elif expect == 'finite':
            assert np.isfinite(s).all() and s[0] > 0 > s[1], (H, v, s)
        elif expect == 'one':
            assert np.allclose(s, [1.0, -1.0], rtol=1e-5), (H, v, s)
        else:
            assert np.isnan(s).all(), (H, v, s)
        imp = {'indptr': ip, 'items': items, 'clicked': clicked}
        if expect == 'nan':
            with pytest.raises(ValueError, match='2\\^63'):
                helpers.impression_metrics(q, emb, imp, metric='cosine')
            continue
        r = helpers.impression_metrics(q, emb, imp, metric='cosine')
        assert r['impressions'] == 1 and not any(np.isnan(r[k]) for k in ('auc', 'mrr', 'ndcg@5', 'ndcg@10')), (H, v, r)
        r = helpers.impression_metrics(q, emb, imp, metric='linear kernel')
        assert r['impressions'] == 1 and not np.isnan(r['auc']), (H, v, r)


# ---------------------------------------------------------------------------------------------------------------------------
# (c) real training batches: every dae_impression_rank_loss call against its own inputs
# ---------------------------------------------------------------------------------------------------------------------------
class LossRecorder:
    """Stands in for user_model.call: snapshots the inputs of each dae_impression_rank_loss call, runs it, synchronizes and
    snapshots its outputs; every other call passes through."""

    def __init__(self, real):
        self.real, self.log = real, []

    def __call__(self, name, *a):
        if name != 'dae_impression_rank_loss':
            return self.real(name, *a)
        n_pos = a[6]
        pi = snap_vec(a[5], n_pos + 1, '<i8')
        n_q = int(pi[-1])
        ip = snap_vec(a[7], n_q + 1, '<i8')
        pre = {'h': snap(a[0], n_pos, a[1]), 'pos_indptr': pi, 'indptr': ip, 'items': snap_vec(a[8], int(ip[-1]), '<i4'),
               'clicked': snap_vec(a[9], int(ip[-1]), '|u1'), 'loss': snap_vec(a[13], 1, '<f8')}
        self.real(name, *a)
        torch.cuda.synchronize()
        post = {'dh': snap(a[11], n_pos, a[12]), 'loss': snap_vec(a[13], 1, '<f8')}
        self.log.append((a, pre, post))


SENTINEL_BUFFERS = {UserGRU: (('XP', 'HP', 'Hs', 'gates', 'dH', 'carry'), ('X_hl', 'dXP_hl', 'dHP_hl')),
                    UserLSTM: (('XP', 'HP', 'Hs', 'Cs', 'gates', 'dH', 'carry', 'carry_c'), ('X_hl', 'dA_hl')),
                    # O_hl keeps the ones column _buffers gave it: no kernel writes column H
                    UserAttention: (('QKV', 'O', 'lse', 'M', 'Z', 'score', 'plse', 'Hs', 'dH', 'dM', 'dO', 'ws'),
                                    ('X_hl', 'M_hl', 'dM_hl', 'dZ_hl', 'dQKV_hl'))}


def _data(U, H, N, max_len, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 4, U)
    lens[:6] = [1, 2, max_len, max_len + 3, 2 * max_len, 1]
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N, int(indptr[-1])).astype(np.int32)
    emb = (rng.standard_normal((N, H)) * 0.5).astype(f32)
    return indptr, items, emb


def _impressions(rng, indptr, N, per_user=3):
    user, time_, lists, clicks = [], [], [], []
    lens = np.diff(indptr)
    for u in range(lens.size):
        for _ in range(per_user):
            user.append(u)
            time_.append(rng.integers(0, lens[u] + 1))
            m = int(rng.integers(1, 14))
            lists.append(rng.choice(N, m, replace=False))
            clicks.append((rng.random(m) < 0.3).astype(np.uint8))
    ip = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return {'user': np.array(user, np.int64), 'time': np.array(time_, np.int64), 'indptr': ip,
            'items': np.concatenate(lists).astype(np.int32), 'clicked': np.concatenate(clicks).astype(np.uint8)}


@pytest.mark.parametrize('cell', [UserGRU, UserLSTM, UserAttention])
def test_training_batch_loss_calls(cell, monkeypatch):
    H, N, max_len = 37, 900, 10
    U = 4 * _pass_rows() // 6                                        # about 6.5 positions per user: P past three passes
    indptr, items, emb = _data(U, H, N, max_len, seed=77)
    rng = np.random.default_rng(78)
    imp = check_impressions(_impressions(rng, indptr, N), N, 'test', indptr)
    use = usable_impressions(imp, indptr, max_len)
    m = cell(H, max_len=max_len, batch_users=U, seed=2)
    pk = Packed(indptr, items, np.arange(U), max_len)
    assert pk.P > 3 * _pass_rows()
    ib = ImpressionBatch(pk, imp, use, indptr)
    assert 0 < ib.n < use.size
    b = m._buffers(pk.P, pk.B)
    f_keys, bf_keys = SENTINEL_BUFFERS[cell]
    for k in f_keys:
        b[k].fill_(float('nan'))
    b['neg'].fill_(-7)
    for k in bf_keys:
        for t in b[k]:
            t.view(torch.int16).fill_(0x7F7F)
    rec = LossRecorder(user_model.call)
    monkeypatch.setattr(user_model, 'call', rec)
    m.stats.fill_(0.75)
    m._forward_backward(pk, _dev(emb), 0, 0, ib)
    torch.cuda.synchronize()
    assert len(rec.log) == 1
    a, pre, post = rec.log[0]
    # the uploaded batch is ImpressionBatch's host arrays; the scale is 1 / ib.n; dH is written in place, H wide
    assert a[6] == pk.P and a[4] == H and a[1] == H and a[12] == H and a[3] == H
    assert np.array_equal(pre['pos_indptr'], ib.pos_indptr) and np.array_equal(pre['indptr'], ib.indptr)
    assert np.array_equal(pre['items'], ib.items) and np.array_equal(pre['clicked'], ib.clicked)
    assert a[10] == 1.0 / ib.n and a[11] == b['dH'].data_ptr() and a[13] == m.stats.data_ptr()
    assert not np.isnan(pre['h'][:, :H]).any()                      # every state the loss reads was written by the forward
    tag = 'train %s' % cell.__name__
    w_dh, s_dh, w_loss, s_loss = ko.rank_loss(pre['h'], emb, pre['pos_indptr'], pre['indptr'], pre['items'], pre['clicked'],
                                              a[10], H)
    ko.check(tag + ' dh', post['dh'][:, :H], w_dh, s_dh, ko.C_FP32)
    ko.check(tag + ' sum', post['loss'][0] - pre['loss'][0], w_loss, s_loss, ko.C_FP32, tiny=1e-15)
    assert pre['loss'][0] == 0.75
    used = np.repeat(np.arange(pk.P), np.diff(ib.pos_indptr))
    none = np.setdiff1d(np.arange(pk.P), used)
    assert none.size and (post['dh'][none, :H] == 0).all()
    assert (used >= 3 * _pass_rows()).any()
    _print_worst(tag)

