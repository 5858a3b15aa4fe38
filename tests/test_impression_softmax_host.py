"""The sampled-softmax impression loss on the CPU (tests/impression_softmax_oracle.py): the reference dh is the fp64 autograd
gradient of the loss; the draws are distinct non-clicks of the right count, uniform, and keyed by (seed, epoch, id, r) alone;
K = 1 on one-click / one-non-click impressions is the pairwise loss and K >= |N| is K = 0; a float32 emulation of the kernel
stays within half the bounds (and two wrong variants do not); the argument checks of dae_impression_softmax_loss, the
constructor, fit and the CLI."""
import os
import sys

import numpy as np
import pytest
import torch

import impression_kernel_oracle as ko
import impression_softmax_oracle as so

from dae_rnn_news_recommendation_b200 import _cabi
from dae_rnn_news_recommendation_b200.user_model import UserGRU, UserLSTM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALF = ko.C_FP32 / 2
f32 = np.float32


def _case(rng, H, n_pos=96):
    h, emb, pi, ip, items, clicked, info = ko.loss_case(rng, H, n_pos)
    return h, emb, pi, ip, items, clicked, so.impression_ids(rng, len(ip) - 1), info


def _autograd(h, emb, pi, ip, clicked, items, sets):
    """Sum over the clicks of log(e^{s_c} + Sum_{S_c} e^{s_n}) - s_c by fp64 autograd, on the oracle's sets: (loss, dloss/dh)."""
    ht = torch.tensor(np.asarray(h, np.float64), requires_grad=True)
    E = torch.as_tensor(np.asarray(emb, np.float64))
    total = torch.zeros((), dtype=torch.float64)
    for p in range(h.shape[0]):
        for q in range(int(pi[p]), int(pi[p + 1])):
            if sets[q] is None:
                continue
            s = E[torch.from_numpy(items[ip[q]:ip[q + 1]].astype(np.int64))] @ ht[p]
            for c, S in sets[q]:
                a = torch.cat([s[c:c + 1], s[torch.from_numpy(np.asarray(S, np.int64))]])
                total = total + torch.logsumexp(a, 0) - s[c]
    total.backward()
    return float(total.detach()), ht.grad.numpy()


@pytest.mark.parametrize('K', [0, 1, 4, 32])
def test_reference_dh_is_the_autograd_gradient(K):
    rng = np.random.default_rng(17 + K)
    H = 9
    h, emb, pi, ip, items, clicked, ids, info = _case(rng, H, 40)
    h = np.clip(h, -3, 3)
    scale = 0.37
    w_dh, _, w_loss, _, sets = so.softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 11, 2, scale, H)
    assert info['skipped_only'] and any(v is None for v in sets.values())
    assert max(len(v) for v in sets.values() if v) >= 40                 # multi-click impressions
    a_loss, a_g = _autograd(h, emb, pi, ip, clicked, items, sets)
    assert abs(w_loss - a_loss) <= 1e-12 * abs(a_loss)
    want = float(f32(scale)) * a_g
    np.testing.assert_allclose(w_dh, want, rtol=1e-10, atol=1e-13 * np.abs(want).max())


# ---------------------------------------------------------------------------------------------------------------------------
# the draws
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [0, 1, 4, 7, 32])
def test_sets_are_distinct_non_clicks(K):
    rng = np.random.default_rng(K)
    for m in (2, 3, 5, 6, 9, 33, 40, 300, 1000):
        for _ in range(4):
            c = (rng.random(m) < rng.choice([0.05, 0.3, 0.9])).astype(np.uint8)
            c[0], c[-1] = 1, 0
            nn = int((c == 0).sum())
            for cp, S in so.negative_sets(c, int(rng.integers(0, 2 ** 32)), K, 5, 3):
                assert c[cp] == 1
                assert S.size == (nn if K == 0 else min(K, nn)) and np.unique(S).size == S.size
                assert (c[S] == 0).all()


def test_floyd_without_the_collision_rule_repeats():
    """The distinctness check above catches Floyd's algorithm without its collision rule: it repeats an ordinal here."""
    u = so.draws(5, 3, np.arange(2000), 0, 4)
    assert any(len(set(so.floyd(x, 6, 4, collision_rule=False))) < 4 for x in u)
    assert all(len(set(so.floyd(x, 6, 4))) == 4 for x in u)


@pytest.mark.parametrize('nn,K', [(10, 4), (5, 4), (33, 32), (7, 1)])
def test_inclusion_frequency_is_uniform(nn, K):
    """Over n = 40 000 (id, r) pairs each non-click is in S_c with probability K / |N|: the count is Binomial(n, K / |N|), and every
    frequency lies within 5 standard deviations (about 3e-7 per ordinal to fail by chance)."""
    n = 40000
    ids = np.arange(n) * 7919 % (2 ** 32)
    u = so.draws(123, 4, ids, np.arange(n) % 13, K)
    hits = np.zeros(nn)
    for x in u:
        hits[so.floyd(x, nn, K)] += 1
    pr = K / nn
    tol = 5 * np.sqrt(pr * (1 - pr) / n)
    assert np.abs(hits / n - pr).max() <= tol, (hits / n, pr, tol)


def test_draws_depend_on_seed_epoch_id_and_r_only():
    K = 8
    base = so.draws(9, 3, [77], [2], K)[0]
    # the same key gives the same words, alone or among other keys, in any order
    many = so.draws(9, 3, [5, 77, 77, 123456], [2, 2, 0, 2], K)
    assert np.array_equal(many[1], base) and not np.array_equal(many[2], base)
    assert np.array_equal(so.draws(9, 3 + 2 ** 32, [77], [2], K)[0], base)             # the epoch's low 32 bits
    for other in (so.draws(10, 3, [77], [2], K), so.draws(9, 4, [77], [2], K), so.draws(9, 3, [78], [2], K),
                  so.draws(9, 3, [77], [3], K), so.draws(2 ** 32 + 9, 3, [77], [2], K)):
        assert not np.array_equal(other[0], base)
    # word d & 3 of counter d >> 2: draws 0..3 and 4..7 come from two Philox calls
    c0 = so.philox4x32_10((77, 2, 3, 0), (9, 0))
    c1 = so.philox4x32_10((77, 2, 3, 1), (9, 0))
    assert [int(x) for x in base] == [int(v) for v in c0] + [int(v) for v in c1]
    # the sets of one impression: the same whatever else is in the batch
    c = np.array([1, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.uint8)
    a = so.negative_sets(c, 77, 3, 9, 3)
    b = so.negative_sets(c, 77, 3, 9, 3)
    assert all(np.array_equal(x[1], y[1]) for x, y in zip(a, b))
    assert any(not np.array_equal(x[1], y[1]) for x, y in zip(a, so.negative_sets(c, 76, 3, 9, 3)))


# ---------------------------------------------------------------------------------------------------------------------------
# identities and the emulation
# ---------------------------------------------------------------------------------------------------------------------------
def test_one_pair_k1_is_the_pairwise_loss():
    rng = np.random.default_rng(3)
    H, P, N = 17, 30, 500
    emb = rng.standard_normal((N, H)).astype(f32)
    h = (rng.standard_normal((P, H)) * 3).astype(f32)
    pi = np.concatenate([[0], np.cumsum(rng.integers(0, 3, P))]).astype(np.int64)
    n_imp = int(pi[-1])
    ip = np.arange(0, 2 * n_imp + 1, 2, dtype=np.int64)
    items = np.concatenate([rng.choice(N, 2, replace=False) for _ in range(n_imp)]).astype(np.int32)
    clicked = np.tile(np.array([1, 0], np.uint8), n_imp)
    ids = so.impression_ids(rng, n_imp)
    for K in (0, 1, 4):
        s_dh, _, s_loss, _, _ = so.softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 1, 0, 0.25, H)
        p_dh, _, p_loss, _ = ko.rank_loss(h, emb, pi, ip, items, clicked, 0.25, H)
        np.testing.assert_allclose(s_dh, p_dh, rtol=1e-12, atol=1e-14)
        assert abs(s_loss - p_loss) <= 1e-12 * abs(p_loss)


def test_k_at_least_n_is_k0():
    """On the positions whose impressions all have |N| <= K, K gives K = 0's dh bit for bit (reference and emulation)."""
    rng = np.random.default_rng(4)
    H = 33
    h, emb, pi, ip, items, clicked, ids, info = _case(rng, H, 64)
    cs = np.concatenate([[0], np.cumsum(clicked, dtype=np.int64)])
    nn = np.diff(ip) - (cs[ip[1:]] - cs[ip[:-1]])
    pos_of = np.repeat(np.arange(h.shape[0]), np.diff(pi))
    ref = so.softmax_loss(h, emb, pi, ip, items, clicked, ids, 0, 3, 1, 0.5, H)
    emu = so.emu_softmax_loss(h, emb, pi, ip, items, clicked, ids, 0, 3, 1, 0.5, H)
    for K in (4, 32):
        rows = np.setdiff1d(np.arange(h.shape[0]), pos_of[nn[:pos_of.size] > K])
        used = np.setdiff1d(rows, np.flatnonzero(np.diff(pi) == 0))
        assert used.size > 10
        r = so.softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 3, 1, 0.5, H)
        e = so.emu_softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 3, 1, 0.5, H)
        assert np.array_equal(r[0][rows], ref[0][rows]) and np.array_equal(e[0][rows], emu[0][rows])


@pytest.mark.parametrize('K', [0, 1, 4, 32])
@pytest.mark.parametrize('H', [1, 33, 500])
def test_emulation_within_half_bound(H, K):
    rng = np.random.default_rng(100 * K + H)
    h, emb, pi, ip, items, clicked, ids, info = _case(rng, H)
    scale = 1.0 / 13
    w_dh, s_dh, w_loss, s_loss, sets = so.softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 7, 5, scale, H)
    e_dh, e_loss = so.emu_softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 7, 5, scale, H)
    tag = 'emu softmax H=%d K=%d' % (H, K)
    ko.check(tag + ' dh', e_dh, w_dh, s_dh, HALF, tiny=ko.TINY / 2)
    ko.check(tag + ' loss', e_loss, w_loss, s_loss, HALF, tiny=ko.TINY / 2)
    used = np.repeat(np.arange(h.shape[0]), np.diff(pi))[ko.usable(ip, clicked)[:pi[-1]]]
    none = np.setdiff1d(np.arange(h.shape[0]), used)
    assert (e_dh[none] == 0).all() and (w_dh[none] == 0).all()
    print(tag, {k: round(v, 4) for k, v in ko.WORST.items() if k.startswith(tag)})


@pytest.mark.parametrize('mutate', ['no_max', 'no_minus_one'])
def test_bounds_reject_wrong_variants(mutate):
    """The bounds are tight enough to fail a kernel that does not subtract the max (scores of +-100 overflow expf) or that
    writes the click's weight as p_cc instead of p_cc - 1."""
    rng = np.random.default_rng(9)
    H = 33
    h, emb, pi, ip, items, clicked, ids, info = _case(rng, H)
    for K in (0, 4):
        w_dh, s_dh, w_loss, s_loss, _ = so.softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 7, 5, 0.1, H)
        e_dh, e_loss = so.emu_softmax_loss(h, emb, pi, ip, items, clicked, ids, K, 7, 5, 0.1, H, mutate=mutate)
        with pytest.raises(AssertionError):
            ko.check('mutant', e_dh, w_dh, s_dh, ko.C_FP32)
            ko.check('mutant', e_loss, w_loss, s_loss, ko.C_FP32)


# ---------------------------------------------------------------------------------------------------------------------------
# argument checks: the export, the constructor, fit, the CLI
# ---------------------------------------------------------------------------------------------------------------------------
P_ = 16   # a non-NULL pointer value: every call below fails its checks before any device work
OK = dict(h=P_, ld_h=8, emb=P_, ld_emb=8, H=8, pos_indptr=P_, n_pos=4, imp_indptr=P_, items=P_, clicked=P_, imp_ids=P_, K=4,
          seed=1, epoch=0, scale=1.0, dh=P_, ld_dh=8, loss_sum=P_, workspace=P_, stream=None)
BAD = [('h', None), ('emb', None), ('pos_indptr', None), ('imp_indptr', None), ('items', None), ('clicked', None),
       ('imp_ids', None), ('dh', None), ('loss_sum', None), ('workspace', None), ('H', 0), ('H', -1), ('n_pos', 0), ('K', -1),
       ('K', 33), ('ld_h', 7), ('ld_emb', 7), ('ld_dh', 7)]


@pytest.mark.parametrize('key,value', BAD, ids=['%s=%s' % b for b in BAD])
def test_export_bad_arguments(key, value):
    args = dict(OK, **{key: value})
    with pytest.raises(_cabi.DaeError, match='dae_impression_softmax_loss: bad arguments'):
        _cabi.call('dae_impression_softmax_loss', *args.values())
    assert 'dae_impression_softmax_loss' in _cabi.exported_symbols()


@pytest.mark.parametrize('cell', [UserGRU, UserLSTM])
def test_constructor_checks(cell):
    m = cell(4, device='cpu')
    assert m.impression_loss == 'pairwise' and m.impression_negatives == 4
    m = cell(4, device='cpu', impression_loss='softmax', impression_negatives=np.int64(0))
    assert m.impression_loss == 'softmax' and m.impression_negatives == 0
    assert cell(4, device='cpu', impression_negatives=32).impression_negatives == 32
    for kw, msg in ((dict(impression_loss='listwise'), 'impression_loss'), (dict(impression_loss=None), 'impression_loss'),
                    (dict(impression_negatives=-1), 'impression_negatives'), (dict(impression_negatives=33), 'impression_negatives'),
                    (dict(impression_negatives=2.0), 'impression_negatives'), (dict(impression_negatives=True), 'impression_negatives')):
        with pytest.raises(ValueError, match='%s: %s' % (cell.__name__, msg)):
            cell(4, device='cpu', **kw)


def test_fit_rejects_2_32_impressions():
    """The draws are keyed by a 32-bit impression id: fit refuses a larger log before reading it (a zero-stride indptr stands in
    for 2^32 impressions)."""
    seqs = (np.array([0, 2]), np.array([0, 1]))
    emb = np.zeros((3, 4), np.float32)
    huge = {'user': np.zeros(1), 'time': np.zeros(1), 'indptr': np.broadcast_to(np.int64(0), (2 ** 32 + 1,)),
            'items': np.zeros(0, np.int32), 'clicked': np.zeros(0, np.uint8)}
    m = UserGRU(4, device='cpu', impression_loss='softmax')
    with pytest.raises(ValueError, match='UserGRU.fit: .*2\\^32'):
        m.fit(seqs, emb, impressions=huge)


def test_cli_flags(tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    p = cli.build_parser()
    s, i = tmp_path / 's.npz', tmp_path / 'i.npz'
    np.savez(s, indptr=np.array([0, 1]), items=np.array([0]))
    np.savez(i, user=np.array([0]), time=np.array([1]), indptr=np.array([0, 2]), items=np.array([0, 1]), clicked=np.array([1, 0]))
    base = ['--top_k', '5', '--user_sequences', str(s)]
    F = cli.check_flags(p.parse_args(base))
    assert F.user_impression_loss == 'pairwise' and F.user_negatives == 4
    F = cli.check_flags(p.parse_args(base + ['--user_impressions', str(i), '--user_impression_loss', 'softmax', '--user_negatives',
                                             '0']))
    assert F.user_impression_loss == 'softmax' and F.user_negatives == 0
    for extra in (['--user_impression_loss', 'softmax'], ['--user_negatives', '4']):
        with pytest.raises(AssertionError, match='needs --user_impressions'):
            cli.check_flags(p.parse_args(base + extra))
    for k in ('-1', '33'):
        with pytest.raises(AssertionError, match='--user_negatives'):
            cli.check_flags(p.parse_args(base + ['--user_impressions', str(i), '--user_negatives', k]))
    with pytest.raises(SystemExit):
        p.parse_args(base + ['--user_impression_loss', 'listwise'])
