"""Triplet batches above 4096 rows (up to DAE_MAX_TRIPLET_BATCH = 32768): the global-memory batch preparation, the tiled batch_all
sweep, and the step / fit / CLI paths that use them, against NumPy and the fp64 chunked oracle (oracle/chunked_oracle.py), which
runs with torch ops on the GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import batch_prepare_oracle as bo
from helpers import REL_TOL, rel_err, elem_err, xavier

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'


def _labels(B, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == 'one':
        return np.full(B, 3.0, np.float32)
    if kind == 'c4':
        return rng.integers(0, 4, B).astype(np.float32)
    if kind == 'c300':
        return rng.integers(0, 300, B).astype(np.float32)
    if kind == 'negf':        # negative / fractional labels, one singleton class
        lab = (-rng.integers(0, 7, B) * 0.37).astype(np.float32)
        lab[B // 2] = 1.5
        return lab
    raise AssertionError(kind)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _expected_prepare(perm, offset, B, labels_all, strategy):
    rows, lab, lo, hi, w, stats = bo.prepare(perm, offset, B, labels_all, strategy)
    return rows, lab, lo, hi, w, stats[bo.STAT_N_VALID]


@pytest.mark.parametrize('B', [4097, 9800, 32768])
@pytest.mark.parametrize('kind', ['c4', 'c300', 'one', 'negf'])
def test_prepare_above_4096(B, kind):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr, STAT
    n_all = B + 1234
    labels_all = _labels(n_all, kind, seed=B)
    perm = np.random.default_rng(B + 1).permutation(n_all).astype(np.int32)
    offset = 1000
    lab_d, perm_d = _t(labels_all), _t(perm)
    i32 = dict(dtype=torch.int32, device=DEV)
    f32 = dict(dtype=torch.float32, device=DEV)
    for strategy in (1, 2):
        rows, labs, lo, hi, w = (torch.full((B,), -7, **i32), torch.full((B,), 9.0, **f32), torch.full((B,), -7, **i32),
                                 torch.full((B,), -7, **i32), torch.full((B,), 9.0, **f32))
        stats = torch.full((16,), 5.0, dtype=torch.float64, device=DEV)
        call('dae_batch_prepare', ptr(perm_d), offset, None, B, ptr(lab_d), strategy, ptr(rows), ptr(labs), ptr(lo), ptr(hi), ptr(w),
             ptr(stats), torch.cuda.current_stream().cuda_stream)
        er, el, elo, ehi, ew, NV = _expected_prepare(perm, offset, B, labels_all, strategy)
        np.testing.assert_array_equal(rows.cpu().numpy(), er)
        np.testing.assert_array_equal(labs.cpu().numpy(), el)
        np.testing.assert_array_equal(lo.cpu().numpy(), elo)
        np.testing.assert_array_equal(hi.cpu().numpy(), ehi)
        np.testing.assert_array_equal(w.cpu().numpy(), ew)
        st = stats.cpu().numpy()
        assert st[STAT['n_valid']] == (NV if strategy == 1 else 0.0)
        assert st[STAT['sum_w']] == (3.0 * NV if strategy == 1 else 0.0)
        assert st[STAT['triplet_sum']] == 0.0 and st[STAT['num']] == 0.0

    # staged variant: batch at ctl[0] + stride; nothing is written when it would run past n_perm
    ctl = torch.tensor([offset - 300, 0, 1, 0], dtype=torch.int64, device=DEV)
    out = [torch.full((B,), -7, **i32), torch.full((B,), 9.0, **f32), torch.full((B,), -7, **i32), torch.full((B,), -7, **i32),
           torch.full((B,), 9.0, **f32), torch.full((16,), 5.0, dtype=torch.float64, device=DEV)]
    st_ = torch.cuda.current_stream().cuda_stream
    call('dae_batch_prepare_next', ptr(perm_d), n_all, 300, ptr(ctl), B, ptr(lab_d), 1, *[ptr(t) for t in out], st_)
    er, el, elo, ehi, ew, NV = _expected_prepare(perm, offset, B, labels_all, 1)
    for t, e in zip(out[:5], (er, el, elo, ehi, ew)):
        np.testing.assert_array_equal(t.cpu().numpy(), e)
    assert out[5][STAT['n_valid']].item() == NV
    before = [t.clone() for t in out]
    ctl[0] = n_all - B - 299           # ctl[0] + stride + B = n_all + 1: past the end
    call('dae_batch_prepare_next', ptr(perm_d), n_all, 300, ptr(ctl), B, ptr(lab_d), 1, *[ptr(t) for t in out], st_)
    torch.cuda.synchronize()
    for a, b in zip(out, before):
        assert torch.equal(a, b)


def _sorted_problem(B, kind, scale, H=16, seed=0):
    """label-sorted batch (as dae_batch_prepare leaves it): labels, E, segments, N_valid."""
    lab = np.sort(_labels(B, kind, seed=seed))
    E = (np.random.default_rng(seed + 5).normal(0.0, scale, (B, H))).astype(np.float32)
    lo = np.searchsorted(lab, lab, side='left').astype(np.int32)
    hi = np.searchsorted(lab, lab, side='right').astype(np.int32)
    n = (hi - lo).astype(np.float64)
    return lab, E, lo, hi, float(np.sum((n - 1.0) * (B - n)))


def _sweep(S, lo, hi, NV, pos_only=0, split=True):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr, STAT
    B = S.shape[0]
    G = torch.full((B, B), 7.0, device=DEV)
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    stats[STAT['n_valid']] = NV
    Bp = (B + 7) // 8 * 8
    gh = torch.full((B, Bp), 3.0, dtype=torch.bfloat16, device=DEV) if split else None
    gl = torch.full((B, Bp), 3.0, dtype=torch.bfloat16, device=DEV) if split else None
    call('dae_triplet_batch_all', ptr(S), B, B, ptr(lo), ptr(hi), ptr(G), B, ptr(stats), pos_only, ptr(gh), ptr(gl), Bp if split else 0,
         torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return G, stats, gh, gl


def _gram(E):
    Ed = E.double()
    return (Ed @ Ed.t()).float()     # S rounded once from fp64: both the kernel and the oracle see the same S


@pytest.mark.parametrize('B,kind,scale,pos_only,tier', [
    (4097, 'c4', 0.15, 0, 0),
    (4097, 'c4', 0.15, 1, 3),        # pos_triplets_only
    (6001, 'c300', 0.8, 0, 1),
    (6001, 'one', 0.8, 0, None),     # no valid triplet
    (6001, 'negf', 2.6, 0, 2),
    (9800, 'c4', 0.6, 0, None),      # rows in tiers 0 and 1
])
def test_tiled_sweep_against_chunked_oracle(B, kind, scale, pos_only, tier):
    from dae_rnn_news_recommendation_b200._cabi import STAT
    lab, E, lo, hi, NV = _sorted_problem(B, kind, scale, seed=B)
    Ed = _t(E)
    S = _gram(Ed)
    row_range = float((S.max(1).values - S.min(1).values).max())    # the widest row's tier (0: < 10, 1: < 80, 2: above)
    if tier in (0, 1, 2):
        assert (0.0, 10.0, 80.0)[tier] <= row_range < (10.0, 80.0, 1e30)[tier]
    lo_d, hi_d = _t(lo), _t(hi)
    G, stats, gh, gl = _sweep(S, lo_d, hi_d, NV, pos_only)
    G2, stats2, gh2, gl2 = _sweep(S, lo_d, hi_d, NV, pos_only)
    assert torch.equal(G, G2) and torch.equal(gh, gh2) and torch.equal(gl, gl2)      # deterministic
    assert stats2[STAT['num']].item() == stats[STAT['num']].item()
    # bf16 hi / lo: the split of G, zero in the padding columns is not required (the GEMM reads columns < B)
    h = G.to(torch.bfloat16)
    assert torch.equal(gh[:, :B], h)
    assert torch.equal(gl[:, :B], (G - h.float()).to(torch.bfloat16))
    from oracle.chunked_oracle import batch_all_triplet_loss_chunked as oracle
    loss, w, frac, num, Go = oracle(_t(lab), None, pos_triplets_only=bool(pos_only), device=DEV, S=S.double())
    st = stats.cpu().numpy()
    n_den = num if pos_only else NV
    if n_den == 0:
        assert float(G.abs().max()) == 0.0 and st[STAT['triplet_sum']] == 0.0
        return
    assert st[STAT['num']] == pytest.approx(float(num), rel=1e-3, abs=2.0)
    got_loss = st[STAT['triplet_sum']] / (n_den + 1e-16)
    assert rel_err(got_loss, float(loss)) < REL_TOL
    if not pos_only:
        assert rel_err(G.double().cpu().numpy(), Go.cpu().numpy()) < REL_TOL
        assert float(G.double().sum(1).abs().max()) < 1e-5 * float(G.abs().max()) * np.sqrt(B)     # every row sums to ~0
    else:   # G holds the positive-triplet counts: -#k at positives, +#j at negatives; each row sums to 0 exactly
        assert float(G.double().sum(1).abs().max()) == 0.0



@pytest.mark.parametrize('B', [64, 800, 4096])
@pytest.mark.parametrize('scale', [0.15, 0.8])
def test_tiled_sweep_matches_shared_memory_sweep(B, scale):
    """dae_triplet_config(1) runs the tiled sweep where the in-shared-memory one would serve: same results up to the fp32 rounding of
    the per-chunk row sums and of the loss partials."""
    from dae_rnn_news_recommendation_b200._cabi import call, STAT
    lab, E, lo, hi, NV = _sorted_problem(B, 'c4', scale, seed=B + 3)
    S = _gram(_t(E))
    lo_d, hi_d = _t(lo), _t(hi)
    G0, st0, gh0, gl0 = _sweep(S, lo_d, hi_d, NV)
    try:
        call('dae_triplet_config', 1)
        G1, st1, gh1, gl1 = _sweep(S, lo_d, hi_d, NV)
    finally:
        call('dae_triplet_config', 0)
    assert st1[STAT['num']].item() == st0[STAT['num']].item()
    # the shared-memory kernel adds up to n_pos * n_neg / 256 log terms per thread in fp32 (~5e4 at B = 4096), the tiled one flushes
    # them into fp64 per chunk: their loss sums differ by ~1e-6 of the sum (1.05e-6 measured at B = 4096, tier 1)
    assert rel_err(st1[STAT['triplet_sum']].item(), st0[STAT['triplet_sum']].item()) < 3e-6
    assert rel_err(G1.cpu().numpy(), G0.cpu().numpy()) < 1e-6


def test_eager_losses_above_4096():
    from dae_rnn_news_recommendation_b200.autoencoder import triplet_loss_utils as tlu
    from oracle.chunked_oracle import batch_all_triplet_loss_chunked, _batch_hard_on
    B, H = 5000, 24
    rng = np.random.default_rng(17)
    labels = rng.integers(0, 5, B).astype(np.float32)
    E = rng.normal(0.0, 0.3, (B, H)).astype(np.float32)
    loss, w, frac, num = tlu.batch_all_triplet_loss(False, labels, E)
    o = batch_all_triplet_loss_chunked(_t(labels), _t(E).double(), device=DEV)
    assert rel_err(loss, float(o[0])) < REL_TOL
    np.testing.assert_allclose(w, o[1].cpu().numpy(), rtol=1e-6)
    assert float(num) == pytest.approx(o[3], rel=1e-3, abs=2.0)
    assert float(frac) == pytest.approx(o[2], rel=1e-3, abs=1e-5)
    loss, w, frac, num = tlu.batch_hard_triplet_loss(False, labels, E)
    oh = _batch_hard_on(_t(labels), _t(E).double())
    assert rel_err(loss, float(oh[0])) < REL_TOL
    assert float(num) == pytest.approx(float(oh[3]), abs=2.0)


def _masked(x, seed):
    keep = np.random.default_rng(seed).random(x.nnz) >= 0.3
    xc = x.copy()
    xc.data = (xc.data * keep).astype(np.float32)
    return xc


KW = dict(enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy', opt='gradient_descent', learning_rate=0.1,
          alpha=1.0)


@pytest.mark.parametrize('B,F,H,strategy,kind,w_scale', [
    (6001, 2000, 128, 'batch_all', 'tfidf', 1.0),
    # batch_hard picks each anchor's hardest positive / negative by comparing entries of S: two candidates closer than the fp32
    # rounding of S can swap, which moves 1/sum_w of the weight (~6e-5 of the gradients at B = 6001).  At W0 x 1 this batch has a pair
    # 1.2e-7 x max|S| apart; at W0 x 10 the closest one is 2.4e-6 apart, clear of the bf16x3 Gram's rounding.
    (6001, 2000, 128, 'batch_hard', 'binary', 10.0),
    (9800, 10000, 500, 'batch_all', 'tfidf', 1.0),    # the C2 shape at batch_size = 0.1 of 98 000 rows
])
def test_step_against_chunked_oracle(B, F, H, strategy, kind, w_scale):
    """One training step through the wgmma path against ChunkedOracleDAE (fp64 on the GPU), with the assertions of the B = 800
    full-size oracle test: losses, every gradient, the updated parameters and the embeddings within 1e-4."""
    from oracle.chunked_oracle import ChunkedOracleDAE
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    x = make_sparse(B, F, 100 if F >= 10000 else 40, kind, seed=B + 1)
    labels = make_labels(B, 4, seed=B + 1)
    xc = _masked(x, B + 2)
    W0 = xavier(F, H, B + 3) * np.float32(w_scale)
    eng = TrainEngine(F, H, device=DEV, triplet_strategy=strategy, **KW)
    eng.set_parameters(W0)
    eng.set_data(DeviceCSR(x, eng.device), torch.from_numpy(xc.data).to(eng.device), torch.from_numpy(labels).to(eng.device))
    eng.step(None, 0, B)
    torch.cuda.synchronize()
    st = eng.read_stats()
    orc = ChunkedOracleDAE(W0, device=DEV, triplet_strategy=strategy, **KW)
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


def test_graph_replay_matches_eager_steps_above_4096():
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    from dae_rnn_news_recommendation_b200._cabi import STAT
    F, H, B, steps = 400, 32, 5000, 3
    x = make_sparse(B * steps, F, 12, 'binary', seed=41)
    xc = _masked(x, 42)
    labels = make_labels(B * steps, 4, seed=43)
    W0 = xavier(F, H, 44) * 3
    for strategy in ('batch_all', 'batch_hard'):
        res = []
        for mode in ('eager', 'graph'):
            eng = TrainEngine(F, H, device=DEV, opt='adam', learning_rate=0.01, triplet_strategy=strategy)
            eng.set_parameters(W0)
            eng.set_data(DeviceCSR(x, eng.device), torch.from_numpy(xc.data.astype(np.float32)).to(eng.device), _t(labels))
            perm = _t(np.random.default_rng(45).permutation(B * steps).astype(np.int32))
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
        assert rel_err(res[1][0][:, STAT['cost']], res[0][0][:, STAT['cost']]) < 1e-5
        assert rel_err(res[1][0][:, STAT['triplet_loss']], res[0][0][:, STAT['triplet_loss']]) < 1e-5
        assert rel_err(res[1][1]['enc_w'], res[0][1]['enc_w']) < 5e-3
        assert rel_err(res[1][1]['dec_b'], res[0][1]['dec_b']) < 5e-3


def _fit(monkeypatch, graph, X, lab, Xv, labv, strategy='batch_all', batch_size=0.1, num_epochs=2):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder
    monkeypatch.setenv('DAE_CUDA_GRAPH', '1' if graph else '0')
    m = DenoisingAutoencoder(model_name='lb', main_dir='lb', compress_factor=20, enc_act_func='sigmoid', dec_act_func='sigmoid',
                             loss_func='cross_entropy', num_epochs=num_epochs, batch_size=batch_size, opt='adam',
                             learning_rate=0.001, corr_type='masking', corr_frac=0.3, verbose=False, verbose_step=1, seed=7,
                             triplet_strategy=strategy)
    m.fit(X, Xv, lab, labv)
    return m


def test_fit_with_default_batch_fraction(monkeypatch):
    """batch_size = 0.1 of 60 000 rows: 6000-row batches replayed from the captured graph, a 6000-row validation batch, and the same
    per-step costs as eager steps."""
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    from dae_rnn_news_recommendation_b200._cabi import STAT
    X = make_sparse(66000, 2000, 40, 'tfidf', seed=3)
    lab = make_labels(66000, 4, seed=3)
    runs = [_fit(monkeypatch, g, X[:60000], lab[:60000], X[60000:], lab[60000:]) for g in (True, False)]
    for m in runs:
        assert m.engine._ws_B == 6000 and len(m.history) == 2 and m.history[0].shape[0] == 10
        assert np.isfinite(m.validation_cost['cost']) and m.validation_cost['triplet_loss'] > 0
    assert runs[0].engine._graph is not None and runs[1].engine._graph is None
    for e in range(2):
        a, b = runs[0].history[e], runs[1].history[e]
        assert rel_err(a[:, STAT['cost']], b[:, STAT['cost']]) < 1e-5
        assert rel_err(a[:, STAT['triplet_loss']], b[:, STAT['triplet_loss']]) < 1e-5
    assert rel_err(runs[0].validation_cost['cost'], runs[1].validation_cost['cost']) < 1e-5


def test_cli_default_batch_fraction(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'main_autoencoder.py'), '--model_name', 'syn', '--synthetic', '60000',
                        '--num_epochs', '1'], cwd=str(tmp_path), capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def test_fit_refuses_batches_above_the_cap(monkeypatch):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    X = make_sparse(33000, 100, 5, 'binary', seed=1)
    lab = make_labels(33000, 4, seed=1)
    m = DenoisingAutoencoder(model_name='cap', main_dir='cap', compress_factor=10, num_epochs=1, batch_size=32769.0, verbose=False,
                             triplet_strategy='batch_hard')
    with pytest.raises(AssertionError) as e:
        m.fit(X, None, lab, None)
    assert '32768' in str(e.value) and 'GB' in str(e.value)
    assert m.engine._ws_B == 0          # no workspace was allocated
    m = DenoisingAutoencoder(model_name='cap2', main_dir='cap2', compress_factor=10, num_epochs=1, batch_size=100.0, verbose=False)
    with pytest.raises(AssertionError) as e:
        m.fit(X[:1000], X, lab[:1000], lab)        # a 33 000-row validation batch
    assert '32768' in str(e.value)
    assert m.engine._ws_B == 0


def _free_gb():
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0] / 1e9


def test_at_the_cap():
    """B = 32 768: a batch_hard training step is finite; one batch_all sweep is deterministic, its rows sum to zero and its bf16
    hi / lo copy is the split of G."""
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    B, F, H = 32768, 300, 16
    if _free_gb() < 20:
        pytest.skip('needs 20 GB of free device memory (%.1f GB free on this shared GPU)' % _free_gb())
    x = make_sparse(B, F, 10, 'binary', seed=5)
    labels = make_labels(B, 300, seed=5)
    eng = TrainEngine(F, H, device=DEV, triplet_strategy='batch_hard', **KW)
    eng.set_parameters(xavier(F, H, 6) * 3)
    eng.set_data(DeviceCSR(x, eng.device), None, _t(labels))
    eng.step(None, 0, B)
    torch.cuda.synchronize()
    st = eng.read_stats()
    assert all(np.isfinite(v) for v in st.values()) and st['num'] > 0
    assert np.isfinite(eng.grad.cpu().numpy()).all()
    del eng
    if _free_gb() < 20:
        pytest.skip('needs 20 GB of free device memory (%.1f GB free on this shared GPU)' % _free_gb())
    lab, E, lo, hi, NV = _sorted_problem(B, 'c300', 0.15, seed=8)
    S = _gram(_t(E))
    lo_d, hi_d = _t(lo), _t(hi)
    G, stats, gh, gl = _sweep(S, lo_d, hi_d, NV)
    for r0 in range(0, B, 4096):
        h = G[r0:r0 + 4096].to(torch.bfloat16)
        assert torch.equal(gh[r0:r0 + 4096, :B], h)
        assert torch.equal(gl[r0:r0 + 4096, :B], (G[r0:r0 + 4096] - h.float()).to(torch.bfloat16))
    del gh, gl
    torch.cuda.empty_cache()
    G2, stats2, _, _ = _sweep(S, lo_d, hi_d, NV, split=False)
    from dae_rnn_news_recommendation_b200._cabi import STAT
    assert torch.equal(G, G2)
    assert stats2[STAT['num']].item() == stats[STAT['num']].item() > 0
    del G2
    gmax = G.abs().max().item()
    rs = max(G[r0:r0 + 4096].double().sum(1).abs().max().item() for r0 in range(0, B, 4096))
    assert gmax > 0 and rs < 1e-5 * gmax * np.sqrt(B)
