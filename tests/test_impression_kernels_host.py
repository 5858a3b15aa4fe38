"""The impression kernels' references (tests/impression_kernel_oracle.py) on the CPU: float32 emulations of both kernels, in their
operation order, stay within half the per-element bounds on the edge inputs the GPU tests use; the reference dh is the gradient
of the loss by fp64 autograd; the metrics emulation agrees with impression_oracle.metrics; impression_metrics' range check."""
import numpy as np
import pytest
import torch

import impression_kernel_oracle as ko
import impression_oracle as io

from dae_rnn_news_recommendation_b200 import helpers

HALF = ko.C_FP32 / 2


@pytest.mark.parametrize('H', [1, 33, 500])
def test_loss_emulation_within_half_bound(H):
    rng = np.random.default_rng(100 + H)
    h, emb, pi, ip, items, clicked, info = ko.loss_case(rng, H, 96)
    scale = 1.0 / 13
    w_dh, s_dh, w_loss, s_loss = ko.rank_loss(h, emb, pi, ip, items, clicked, scale, H)
    e_dh, e_loss = ko.emu_rank_loss(h, emb, pi, ip, items, clicked, scale, H)
    tag = 'emu H=%d' % H
    ko.check(tag + ' dh', e_dh, w_dh, s_dh, HALF, tiny=ko.TINY / 2)
    ko.check(tag + ' loss', e_loss, w_loss, s_loss, HALF, tiny=ko.TINY / 2)
    # rows without a usable impression are exactly 0, in the reference too
    used = np.repeat(np.arange(h.shape[0]), np.diff(pi))[ko.usable(ip, clicked)[:pi[-1]]]
    none = np.setdiff1d(np.arange(h.shape[0]), used)
    assert set(info['skipped_only']) <= set(none)
    assert (e_dh[none] == 0).all() and (w_dh[none] == 0).all() and (s_dh[none] == 0).all()
    # the edge pairs reach the tails: sigma rounds to 0 and to 1 in fp32
    x = [float(emb[items[ip[q] + 1]].astype(np.float64) @ h[p] - emb[items[ip[q]]].astype(np.float64) @ h[p])
         for p in info['x_pos'] for q in [pi[p]]]
    assert max(x) > 99 and min(x) < -99
    print(tag, {k: round(v, 4) for k, v in ko.WORST.items() if k.startswith(tag)})


@pytest.mark.parametrize('cosine', [False, True])
@pytest.mark.parametrize('H', [1, 33, 500])
def test_scores_emulation_within_half_bound(H, cosine):
    rng = np.random.default_rng(200 + H + cosine)
    q, emb, ip, items, clicked, info = ko.metrics_case(rng, H, 60)
    want, scale = ko.scores(q, emb, ip, items, cosine, H)
    got = ko.emu_scores(q, emb, ip, items, cosine, H)
    tag = 'emu scores H=%d cos=%d' % (H, cosine)
    ko.check(tag, got, want, scale, HALF, tiny=ko.TINY / 2)
    zq = info['zero_query']
    assert (got[ip[zq]:ip[zq + 1]] == 0).all() and (want[ip[zq]:ip[zq + 1]] == 0).all()
    if cosine:
        z = np.isin(items, info['zero_items'])
        assert z.any() and (got[z] == 0).all() and (scale[z] == 0).all()
    print(tag, round(ko.WORST[tag], 4))


def _autograd_loss(h, emb, pi, ip, items, clicked):
    """Sum over the usable impressions of 1 / (|C| |N|) Sum softplus(s_n - s_c) by fp64 autograd: (loss, d loss / d h)."""
    ht = torch.tensor(np.asarray(h, np.float64), requires_grad=True)
    E = torch.as_tensor(np.asarray(emb, np.float64))
    total = torch.zeros((), dtype=torch.float64)
    for p in range(h.shape[0]):
        for q in range(int(pi[p]), int(pi[p + 1])):
            c = torch.from_numpy(clicked[ip[q]:ip[q + 1]].astype(bool))
            if c.all() or not c.any():
                continue
            s = E[torch.from_numpy(items[ip[q]:ip[q + 1]].astype(np.int64))] @ ht[p]
            x = s[~c][None, :] - s[c][:, None]
            total = total + torch.nn.functional.softplus(x).mean()
    total.backward()
    return float(total.detach()), ht.grad.numpy()


def test_reference_dh_is_the_autograd_gradient():
    rng = np.random.default_rng(7)
    H = 9
    h, emb, pi, ip, items, clicked, info = ko.loss_case(rng, H, 40, N=6000)
    h = np.clip(h, -3, 3)                          # softplus' autograd gradient at |x| = 100 is exact anyway; keep x moderate
    assert (np.diff(pi) >= 3).any() and info['skipped_only']
    scale = 0.37
    w_dh, _, w_loss, _ = ko.rank_loss(h, emb, pi, ip, items, clicked, scale, H)
    a_loss, a_g = _autograd_loss(h, emb, pi, ip, items, clicked)
    assert abs(w_loss - a_loss) <= 1e-12 * abs(a_loss)
    want = float(np.float32(scale)) * a_g
    np.testing.assert_allclose(w_dh, want, rtol=1e-10, atol=1e-13 * np.abs(want).max())
    # the old whole-impression restatement agrees too
    o_loss, o_dh = io.impression_loss(h, emb, pi, ip, items, clicked, float(np.float32(scale)))
    np.testing.assert_allclose(w_dh, o_dh, rtol=1e-10, atol=1e-13 * np.abs(want).max())
    assert abs(o_loss - w_loss) <= 1e-12 * abs(w_loss)


@pytest.mark.parametrize('cosine', [False, True])
def test_metrics_emulation_equals_oracle(cosine):
    rng = np.random.default_rng(300 + cosine)
    H = 33
    q, emb, ip, items, clicked, info = ko.metrics_case(rng, H, 150)
    s = ko.emu_scores(q, emb, ip, items, cosine, H)
    got, g_ints = ko.emu_metrics(s, ip, clicked)
    want, w_ints = io.metrics(s, ip, clicked)
    nan = np.isnan(want[:, 0])
    assert np.array_equal(np.isnan(got), np.repeat(nan[:, None], 4, 1))
    assert np.array_equal(g_ints, w_ints)
    assert np.array_equal(got[~nan, 0], want[~nan, 0])
    # MRR and nDCG sum the same terms in another order (per lane and a tree here, pairwise in NumPy)
    np.testing.assert_allclose(got[~nan], want[~nan], rtol=1e-12, atol=0)
    # the edges are reached: ties across the chunk boundary, the nDCG cut-offs, |C| > 32 and > 10, empty and single candidates
    first = s[ip[0]:ip[1]]
    assert first[255] == first[256] == first[250] == first[260]
    for i, r in info['rank'].items():
        assert w_ints[i, 1] == r, (i, r, w_ints[i])
    n_c = np.diff(np.concatenate([[0], np.cumsum(clicked, dtype=np.int64)])[ip])
    assert n_c.max() >= 100 and ((n_c > 10) & (n_c < 32)).any()
    assert (np.diff(ip) == 0).any() and nan[np.flatnonzero(np.diff(ip) == 1)].all()


def test_metrics_helper_range_check():
    """impression_metrics refuses entries beyond 2^63 / sqrt(H), where the kernel's fp32 sums could overflow, before any device
    work (the GPU tests show that the limit itself is accepted and scores finitely)."""
    H = 64
    emb = np.ones((4, H), np.float32)
    imp = {'indptr': np.array([0, 2]), 'items': np.array([0, 1], np.int32), 'clicked': np.array([1, 0], np.uint8)}
    over = np.nextafter(np.float32(2.0 ** 60), np.float32(np.inf))          # 2^63 / sqrt(64) = 2^60, one ulp above
    for metric in ('cosine', 'linear kernel'):
        for bad_q, bad_e in ((over, 1.0), (1.0, over), (-over, 1.0)):
            with pytest.raises(ValueError, match='2\\^63'):
                helpers.impression_metrics(np.full((1, H), bad_q, np.float32), emb * np.float32(bad_e), imp, metric=metric,
                                           device='cpu')
