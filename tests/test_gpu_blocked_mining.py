"""Block mining (TrainEngine(mining_block_rows=R)): the Gram blocks, the rows kernels and the block-mined step against the
materialising path at B <= 32 768, and against the fp64 block oracle (tests/block_oracle.py) above that cap."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import REL_TOL, rel_err, elem_err, xavier

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
KW = dict(enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy', opt='gradient_descent', learning_rate=0.1,
          alpha=1.0)


@pytest.fixture(autouse=True)
def _restore_global_rng():
    """Some of these tests draw from torch's global generators, and `fit(seed=...)` reseeds them.  Restore them afterwards, so that
    the tests that run later draw the same random inputs whether this module ran first or not."""
    with torch.random.fork_rng(devices=[torch.cuda.current_device()] if torch.cuda.is_available() else []):
        yield


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _free_gb():
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0] / 1e9


def _split(E):
    """E [B x H] fp32 -> the bf16 hi / lo pair [B x Hp] the engine's GEMMs read."""
    from dae_rnn_news_recommendation_b200._cabi import call, ptr
    B, H = E.shape
    Hp = (H + 1 + 63) // 64 * 64
    hi = torch.zeros(B, Hp, dtype=torch.bfloat16, device=DEV)
    lo = torch.zeros(B, Hp, dtype=torch.bfloat16, device=DEV)
    call('dae_split_bf16', ptr(E), B, H, H, ptr(hi), ptr(lo), Hp, -1, 1.0, _st())
    return hi, lo


def _gemm(M, N, K, A, a_mn, Bm, b_mn, C, ldc):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr
    call('dae_gemm_bf16x3', M, N, K, 1.0, ptr(A[0]), ptr(A[1]), A[0].stride(0), a_mn, ptr(Bm[0]), ptr(Bm[1]), Bm[0].stride(0), b_mn,
         ptr(C), ldc, 0, -1, None, 1, 0, _st())


def _problem(B, n_classes, H=64, scale=0.3, seed=0):
    """label-sorted batch: labels, E, segments, N_valid (what dae_batch_prepare leaves)."""
    rng = np.random.default_rng(seed)
    lab = np.sort(rng.integers(0, n_classes, B).astype(np.float32))
    E = rng.normal(0.0, scale, (B, H)).astype(np.float32)
    lo = np.searchsorted(lab, lab, side='left').astype(np.int32)
    hi = np.searchsorted(lab, lab, side='right').astype(np.int32)
    n = (hi - lo).astype(np.float64)
    return lab, E, lo, hi, float(np.sum((n - 1.0) * (B - n)))


def _blocks(B, R):
    return [(r0, min(R, B - r0)) for r0 in range(0, B, R)]


BR = [(800, 128), (800, 1024), (5000, 128), (5000, 1024), (5000, 640), (9800, 1024), (9800, 3072)]


@pytest.mark.parametrize('B,R', BR)
def test_gram_blocks_equal_the_full_gram_bit_for_bit(B, R):
    """Every entry of S runs the same k16 sequence in whichever tile holds it, so a block of rows equals those rows of the full
    Gram GEMM exactly."""
    _, E, _, _, _ = _problem(B, 4, H=500 if B == 800 else 128, seed=B + R)
    Ehl = _split(_t(E))
    S = torch.empty(B, B, device=DEV)
    _gemm(B, B, E.shape[1], Ehl, 0, Ehl, 0, S, B)
    S_blk = torch.full((R, B), 7.0, device=DEV)
    for r0, n in _blocks(B, R):
        _gemm(n, B, E.shape[1], (Ehl[0][r0:], Ehl[1][r0:]), 0, Ehl, 0, S_blk, B)
        assert torch.equal(S_blk[:n], S[r0:r0 + n]), (r0, n)


@pytest.mark.parametrize('B,R', BR)
@pytest.mark.parametrize('n_classes', [4, 300])
def test_batch_all_rows_equal_the_tiled_sweep(B, R, n_classes):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr, STAT
    lab, E, lo, hi, NV = _problem(B, n_classes, scale=0.15 if n_classes == 4 else 0.8, seed=B + 1)
    Ed = _t(E).double()
    S = (Ed @ Ed.t()).float()
    lo_d, hi_d = _t(lo), _t(hi)
    Bp = (B + 7) // 8 * 8

    def stats0():
        s = torch.zeros(16, dtype=torch.float64, device=DEV)
        s[STAT['n_valid']] = NV
        return s
    G = torch.empty(B, B, device=DEV)
    gh, gl = (torch.empty(B, Bp, dtype=torch.bfloat16, device=DEV) for _ in range(2))
    st = stats0()
    try:
        call('dae_triplet_config', 1)
        call('dae_triplet_batch_all', ptr(S), B, B, ptr(lo_d), ptr(hi_d), ptr(G), B, ptr(st), 0, ptr(gh), ptr(gl), Bp, _st())
    finally:
        call('dae_triplet_config', 0)
    Gb = torch.full((R, B + 3), 9.0, device=DEV)         # ldg > B
    bh, bl = (torch.full((R, Bp), 5.0, dtype=torch.bfloat16, device=DEV) for _ in range(2))
    Sb = torch.empty(R, B + 5, device=DEV)             # lds > B
    sb = stats0()
    for r0, n in _blocks(B, R):
        Sb[:n, :B] = S[r0:r0 + n]
        call('dae_triplet_batch_all_rows', ptr(Sb), B + 5, r0, n, B, ptr(lo_d), ptr(hi_d), ptr(Gb), B + 3, ptr(sb), 0, ptr(bh), ptr(bl), Bp,
             _st())
        assert torch.equal(Gb[:n, :B], G[r0:r0 + n])
        assert torch.equal(bh[:n, :B], gh[r0:r0 + n, :B]) and torch.equal(bl[:n, :B], gl[r0:r0 + n, :B])
    a, b = st.cpu().numpy(), sb.cpu().numpy()
    assert a[STAT['num']] == b[STAT['num']]
    assert abs(a[STAT['triplet_sum']] - b[STAT['triplet_sum']]) <= 1e-12 * abs(a[STAT['triplet_sum']])


@pytest.mark.parametrize('B,R', BR)
@pytest.mark.parametrize('n_classes', [4, 300])
def test_batch_hard_rows_equal_the_materialising_kernel(B, R, n_classes):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr, STAT
    lab, E, _, _, _ = _problem(B, n_classes, scale=0.5, seed=B + 2)
    if n_classes == 4:
        E = np.round(E * 4.0).astype(np.float32)      # small integers: exact ties in S
    Ed = _t(E).double()
    S = (Ed @ Ed.t()).float()
    lab_d = _t(lab)
    G = torch.empty(B, B, device=DEV)
    w = torch.full((B,), 3.0, device=DEV)
    st = torch.zeros(16, dtype=torch.float64, device=DEV)
    call('dae_triplet_batch_hard', ptr(S), B, B, ptr(lab_d), ptr(G), B, ptr(w), ptr(st), _st())
    Sb = torch.empty(R, B + 5, device=DEV)
    Gb = torch.empty(R, B + 3, device=DEV)
    Graw = torch.empty(B, B, device=DEV)
    wb = torch.zeros(B, device=DEV)
    sb = torch.zeros(16, dtype=torch.float64, device=DEV)
    for r0, n in _blocks(B, R):
        Sb[:n, :B] = S[r0:r0 + n]
        call('dae_triplet_batch_hard_rows', ptr(Sb), B + 5, r0, n, B, ptr(lab_d), ptr(Gb), B + 3, ptr(wb), ptr(sb), _st())
        Graw[r0:r0 + n] = Gb[:n, :B]
    call('dae_triplet_batch_hard_finish', ptr(wb), B, ptr(sb), None, 0, 0, _st())
    torch.cuda.synchronize()
    a, b = st.cpu().numpy(), sb.cpu().numpy()
    assert torch.equal(wb, w)
    assert a[STAT['num']] == b[STAT['num']] and a[STAT['n_active']] == b[STAT['n_active']] and b[STAT['n_active']] > 0
    assert a[STAT['sum_w']] == b[STAT['sum_w']]
    assert abs(a[STAT['triplet_sum']] - b[STAT['triplet_sum']]) <= 1e-12 * abs(a[STAT['triplet_sum']])
    inv = np.float32(1.0 / (b[STAT['n_active']] + 1e-16))
    assert torch.equal(Graw * float(inv), G)
    # finish with dE2: every entry times the same factor
    dE2 = torch.randn(B, 40, device=DEV, generator=torch.Generator(device=DEV).manual_seed(B + R))
    want = dE2 * float(inv)
    call('dae_triplet_batch_hard_finish', ptr(wb), B, ptr(sb), ptr(dE2), 40, 40, _st())
    assert torch.equal(dE2, want)


@pytest.mark.parametrize('B', [800, 9800])
def test_blocked_prepare_equals_the_capped_prepare(B):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr
    n_all = B + 777
    labels = _t(np.random.default_rng(B).integers(0, 30, n_all).astype(np.float32))
    perm = _t(np.random.default_rng(B + 1).permutation(n_all).astype(np.int32))
    i32, f32 = dict(dtype=torch.int32, device=DEV), dict(dtype=torch.float32, device=DEV)

    def bufs():
        return [torch.full((B,), -7, **i32), torch.full((B,), 9.0, **f32), torch.full((B,), -7, **i32), torch.full((B,), -7, **i32),
                torch.full((B,), 9.0, **f32), torch.full((16,), 5.0, dtype=torch.float64, device=DEV)]
    ctl = torch.tensor([300, 0, 1, 0], dtype=torch.int64, device=DEV)
    for strategy in (1, 2):
        a, b = bufs(), bufs()
        call('dae_batch_prepare', ptr(perm), 500, None, B, ptr(labels), strategy, *[ptr(t) for t in a], _st())
        call('dae_batch_prepare_blocked', ptr(perm), 500, None, B, ptr(labels), strategy, *[ptr(t) for t in b], _st())
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        a, b = bufs(), bufs()
        call('dae_batch_prepare_next', ptr(perm), n_all, 200, ptr(ctl), B, ptr(labels), strategy, *[ptr(t) for t in a], _st())
        call('dae_batch_prepare_next_blocked', ptr(perm), n_all, 200, ptr(ctl), B, ptr(labels), strategy, *[ptr(t) for t in b], _st())
        assert all(torch.equal(x, y) for x, y in zip(a, b))


def _masked(x, seed):
    keep = np.random.default_rng(seed).random(x.nnz) >= 0.3
    xc = x.copy()
    xc.data = (xc.data * keep).astype(np.float32)
    return xc


def _engine_step(x, xc, labels, W0, strategy, R, **kw):
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    F, H = W0.shape
    args = dict(KW)
    args.update(kw)
    eng = TrainEngine(F, H, device=DEV, triplet_strategy=strategy, mining_block_rows=R, **args)
    eng.set_parameters(W0)
    eng.set_data(DeviceCSR(x, eng.device), _t(xc.data.astype(np.float32)), _t(labels))
    eng.step(None, 0, x.shape[0])
    torch.cuda.synchronize()
    return eng


@pytest.mark.parametrize('B,F,H,R,strategy,w_scale', [
    (800, 10000, 500, 128, 'batch_all', 1.0),        # the C2 shape
    (800, 10000, 500, 384, 'batch_hard', 1.0),
    (6001, 2000, 128, 1024, 'batch_all', 1.0),
    (6001, 2000, 128, 1024, 'batch_hard', 10.0),     # W0 x 10: see test_gpu_large_batch.test_step_against_chunked_oracle
])
def test_blocked_step_matches_the_materialising_step(B, F, H, R, strategy, w_scale):
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    x = make_sparse(B, F, 100 if F >= 10000 else 40, 'tfidf' if strategy == 'batch_all' else 'binary', seed=B + 1)
    labels = make_labels(B, 4, seed=B + 1)
    xc = _masked(x, B + 2)
    W0 = xavier(F, H, B + 3) * np.float32(w_scale)
    e0 = _engine_step(x, xc, labels, W0, strategy, None)
    e1 = _engine_step(x, xc, labels, W0, strategy, R)
    assert not hasattr(e1, 'Z') and e1.S.shape == (R, B)
    s0, s1 = e0.read_stats(), e1.read_stats()
    for k in ('cost', 'ae_loss', 'triplet_loss', 'sum_w'):
        assert rel_err(s1[k], s0[k]) < 1e-5, k
    assert s1['num'] == pytest.approx(s0['num'], rel=1e-6, abs=0.5)
    assert rel_err(e1.grad.cpu().numpy(), e0.grad.cpu().numpy()) < 1e-5
    assert rel_err(e1.theta.cpu().numpy(), e0.theta.cpu().numpy()) < 1e-5
    if B == 800:
        from oracle.chunked_oracle import ChunkedOracleDAE
        o = ChunkedOracleDAE(W0, device=DEV, triplet_strategy=strategy, **KW).step(x, xc, labels)
        assert rel_err(s1['cost'], o['cost']) < REL_TOL
        assert rel_err(s1['triplet_loss'], o['triplet_loss']) < REL_TOL
        g = e1.grad.cpu().numpy()
        assert rel_err(g[:F * H].reshape(F, H), o['grads'][0]) < REL_TOL
        assert rel_err(g[F * H + H:], o['grads'][2]) < REL_TOL


def _hard_margin_over_gram_error(eng, E64, labels, B, block=4096):
    """The precondition of comparing a block-mined batch_hard step with the fp64 oracle: no active anchor's hardest negative /
    positive may swap with the runner-up under the Gram's rounding.  For every active anchor (fp64), the lead of its hardest negative
    and of its hardest positive over the runner-up (the next DISTINCT value: exact ties are ties in both), divided by the largest
    |S_kernel - S_fp64| of its row, where S_kernel is the bf16x3 Gram of the engine's own E hi / lo (what its mining saw).  Returns
    the smallest ratio."""
    rows = eng.rows[:B].long()
    E, lab = E64[rows], labels[rows]
    H = E.shape[1]
    Ehl = (eng.E_hi[:B], eng.E_lo[:B])
    S32 = torch.empty(block, B, device=DEV)
    cols = torch.arange(B, device=DEV)
    worst = np.inf
    for r0, n in _blocks(B, block):
        A = cols[r0:r0 + n]
        s = E[A] @ E.t()
        _gemm(n, B, H, (eng.E_hi[r0:], eng.E_lo[r0:]), 0, Ehl, 0, S32, B)
        err = (S32[:n].double() - s).abs().max(1).values
        same = lab[A][:, None] == lab[None, :]
        pos = same & (A[:, None] != cols[None, :])
        m = s.max(1, keepdim=True).values
        ans = torch.where(~same, s, torch.zeros_like(s))                          # an * S
        hn = ans.max(1, keepdim=True).values
        hn_2 = torch.where(ans < hn, ans, torch.full_like(s, -np.inf)).max(1, keepdim=True).values
        hpi = torch.where(pos, s, s + m)                                          # S + m (1 - ap)
        hp = hpi.min(1, keepdim=True).values
        hp_2 = torch.where(hpi > hp, hpi, torch.full_like(s, np.inf)).min(1, keepdim=True).values
        active = ((hn - hp) > 0).squeeze(1)
        gap = torch.minimum(hn - hn_2, hp_2 - hp).squeeze(1)
        if bool(active.any()):
            worst = min(worst, float((gap / err)[active].min()))
        del s, same, pos, ans, hpi
    return worst


# batch_hard at B = 40 000: with 30 000 candidates per anchor, continuous scores put some runner-up within the Gram's rounding of the
# hardest one (measured: the closest at 0.1x the row's error).  The rows are therefore drawn from 400 distinct articles: copies of
# one article are exact ties in fp32 and in fp64 alike, and distinct ones lie far apart.  No corruption, so copies stay copies.
# W0 x 3: at W0 x 10 the embeddings after the step differ element-wise by 1.4e-4 (norm-wise they agree).
HARD_40K = dict(seed=40001, w_scale=3.0, articles=400)


@pytest.mark.parametrize('strategy,kind,n_classes', [('batch_hard', 'binary', 4), ('batch_all', 'tfidf', 1000)])
def test_step_above_the_cap_against_the_block_oracle(strategy, kind, n_classes):
    """One B = 40 000 training step with R = 4096 against BlockOracleDAE (fp64 on the GPU): losses, every gradient, the updated
    parameters and the embeddings within 1e-4, as test_gpu_large_batch.test_step_against_chunked_oracle at B <= 32 768."""
    from block_oracle import BlockOracleDAE
    from oracle.dae_oracle import encode
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    B, F, H, R = 40000, 2000, 128, 4096
    if _free_gb() < 30:
        pytest.skip('needs 30 GB of free device memory (%.1f GB free on this shared GPU)' % _free_gb())
    seed = HARD_40K['seed'] if strategy == 'batch_hard' else 40011
    if strategy == 'batch_hard':
        x = make_sparse(HARD_40K['articles'], F, 40, kind, seed=seed)[np.random.default_rng(seed).integers(0, HARD_40K['articles'], B)]
        xc = x
    else:
        x = make_sparse(B, F, 40, kind, seed=seed)
        xc = _masked(x, seed + 1)
    labels = make_labels(B, n_classes, seed=seed)
    W0 = xavier(F, H, seed + 2) * np.float32(HARD_40K['w_scale'] if strategy == 'batch_hard' else 1.0)
    orc = BlockOracleDAE(W0, device=DEV, triplet_strategy=strategy, block_rows=R, **KW)
    eng = _engine_step(x, xc, labels, W0, strategy, R)
    if strategy == 'batch_hard':   # precondition: no anchor's hardest positive / negative is within the Gram's rounding of another
        with torch.no_grad():
            E = encode(orc._sparse_or_dense(xc), orc.W, orc.bh, orc.enc_act_func)
        ratio = _hard_margin_over_gram_error(eng, E, _t(labels), B)
        del E
        assert ratio > 2.0, ratio
    st = eng.read_stats()
    o = orc.step(x, xc, labels)
    assert st['num'] == pytest.approx(float(o['num']), rel=1e-3, abs=2.0)
    assert st['fraction'] == pytest.approx(float(o['fraction']), rel=1e-3, abs=1e-5)
    assert rel_err(st['cost'], o['cost']) < REL_TOL
    assert rel_err(st['ae_loss'], o['autoencoder_loss']) < REL_TOL
    assert rel_err(st['triplet_loss'], o['triplet_loss']) < REL_TOL
    gW, gbh, gbv = o['grads']
    g = eng.grad.cpu().numpy()
    assert rel_err(g[:F * H].reshape(F, H), gW) < REL_TOL
    assert rel_err(g[F * H + H:], gbv) < REL_TOL
    assert np.abs(g[F * H:F * H + H] - gbh).max() < REL_TOL * max(float(np.abs(gW).max()), float(np.abs(gbh).max()))
    p, q = eng.get_parameters(), orc.get_parameters()
    assert rel_err(p['enc_w'], q['enc_w']) < REL_TOL
    assert rel_err(p['dec_b'], q['dec_b']) < REL_TOL
    emb = eng.encode(DeviceCSR(x, eng.device)).cpu().numpy()
    want = orc.transform(x)
    assert rel_err(emb, want) < REL_TOL
    assert elem_err(emb, want, floor=0.1) < REL_TOL


def test_graph_replay_matches_eager_steps_above_the_cap():
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    from dae_rnn_news_recommendation_b200._cabi import STAT
    F, H, B, steps, R = 400, 32, 40000, 3, 4096
    x = make_sparse(B * steps, F, 12, 'binary', seed=51)
    xc = _masked(x, 52)
    W0 = xavier(F, H, 54) * 3
    for strategy, n_classes in (('batch_hard', 4), ('batch_all', 1000)):
        labels = make_labels(B * steps, n_classes, seed=53)
        res = []
        for mode in ('eager', 'graph'):
            eng = TrainEngine(F, H, device=DEV, opt='adam', learning_rate=0.01, triplet_strategy=strategy, mining_block_rows=R)
            eng.set_parameters(W0)
            eng.set_data(DeviceCSR(x, eng.device), _t(xc.data.astype(np.float32)), _t(labels))
            perm = _t(np.random.default_rng(55).permutation(B * steps).astype(np.int32))
            log = torch.zeros(steps, 16, dtype=torch.float64, device=eng.device)
            if mode == 'eager':
                for s in range(steps):
                    eng.step(perm, s * B, B, log[s])
            else:
                eng.capture_step_graph(perm, B, log)
                eng.set_step_cursor(0, 0)
                for s in range(steps):
                    eng.replay_step()
            torch.cuda.synchronize()
            res.append((log.cpu().numpy().copy(), eng.get_parameters()))
            del eng
        for k in ('cost', 'triplet_loss', 'ae_loss'):
            assert rel_err(res[1][0][:, STAT[k]], res[0][0][:, STAT[k]]) < 1e-5, (strategy, k)
        assert rel_err(res[1][1]['enc_w'], res[0][1]['enc_w']) < 5e-3


def test_fit_with_default_batch_fraction_above_the_cap(monkeypatch):
    """batch_size = 0.1 of 400 000 rows with mining_block_rows = 4096: 40 000-row batch_hard batches replayed from the captured
    graph, and a 40 000-row validation batch whose cost equals an eager evaluate."""
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    X = make_sparse(440000, 1000, 20, 'binary', seed=61)
    lab = make_labels(440000, 4, seed=61)
    monkeypatch.setenv('DAE_CUDA_GRAPH', '1')
    m = DenoisingAutoencoder(model_name='fb', main_dir='fb', compress_factor=20, enc_act_func='sigmoid', dec_act_func='sigmoid',
                             loss_func='cross_entropy', num_epochs=1, batch_size=0.1, opt='adam', learning_rate=0.001,
                             corr_type='masking', corr_frac=0.3, verbose=False, verbose_step=1, seed=7, triplet_strategy='batch_hard',
                             mining_block_rows=4096)
    m.fit(X[:400000], X[400000:], lab[:400000], lab[400000:])
    eng = m.engine
    assert eng._ws_B == 40000 and eng._graph is not None and m.history[0].shape[0] == 10
    assert np.isfinite(m.history[0]).all()
    v = m.validation_cost
    assert np.isfinite(v['cost']) and v['triplet_loss'] > 0
    again = eng.evaluate(DeviceCSR(X[400000:], eng.device), _t(lab[400000:]))
    for k in ('cost', 'ae_loss', 'triplet_loss'):
        assert rel_err(again[k], v[k]) < 1e-6, k   # fp32 atomics of the decode row losses: last-bit differences


def test_fit_refuses_batches_above_the_blocked_cap():
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    X = make_sparse(262145, 64, 3, 'binary', seed=1)
    lab = make_labels(262145, 4, seed=1)
    m = DenoisingAutoencoder(model_name='bcap', main_dir='bcap', compress_factor=8, num_epochs=1, batch_size=262145.0, verbose=False,
                             triplet_strategy='batch_hard', mining_block_rows=4096)
    with pytest.raises(AssertionError) as e:
        m.fit(X, None, lab, None)
    assert '262144' in str(e.value) and 'GB' in str(e.value)
    assert m.engine._ws_B == 0


def test_cli_above_the_cap(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'main_autoencoder.py'), '--model_name', 'syn', '--synthetic', '400000',
                        '--triplet_strategy', 'batch_hard', '--mining_block_rows', '4096', '--num_epochs', '1'], cwd=str(tmp_path),
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def test_peak_memory_at_100000_rows():
    """A B = 100 000, F = 10 000, H = 500 batch_hard step with R = 4096 stays inside the workspace its shapes need: no B x B buffer
    and no B x F fp32 Z."""
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    B, F, H, R = 100000, 10000, 500, 4096
    if _free_gb() < 20:
        pytest.skip('needs 20 GB of free device memory (%.1f GB free on this shared GPU)' % _free_gb())
    x = make_sparse(B, F, 100, 'binary', seed=71)
    labels = make_labels(B, 4, seed=71)
    eng = TrainEngine(F, H, device=DEV, triplet_strategy='batch_hard', mining_block_rows=R, **KW)
    eng.set_parameters(xavier(F, H, 72))
    eng.set_data(DeviceCSR(x, eng.device), None, _t(labels))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    eng.step(None, 0, B)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    Hp, Fp, Bp = eng.Hp, eng.Fp, (B + 7) // 8 * 8
    need = (8 * R * B + 4 * R * Bp                # S, G fp32 [R x B], their bf16 hi / lo [R x Bp]
            + 4 * B * Fp                             # dZ hi / lo
            + 4 * B * Hp + 3 * 4 * B * H             # E hi / lo; E, dE, dE2
            + 4 * B * (4 * ((F + 255) // 256) + 1)   # decode tile table
            + 12 * x.nnz + 64 * B)                   # encode-backward buckets, per-row vectors
    assert not hasattr(eng, 'Z')
    assert peak < 1.1 * need + (256 << 20), (peak / 1e9, need / 1e9)   # Z would add 4 B F = 4 GB
    st = eng.read_stats()
    assert all(np.isfinite(v) for v in st.values()) and st['num'] > 0
