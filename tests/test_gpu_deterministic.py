"""Deterministic training mode (TrainEngine(deterministic=True), DESIGN 4.7): the fixed-order kernels against NumPy restatements and
fp64, their run-to-run bit equality while other work shares the GPU, and whole seeded runs that reproduce themselves bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from helpers import REL_TOL, rel_err, xavier

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
KW = dict(enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy', opt='gradient_descent', learning_rate=0.1,
          alpha=1.0)


@pytest.fixture(autouse=True)
def _restore_global_rng():
    """`fit(seed=...)` reseeds torch's global generators: restore them, so later test modules draw the same inputs either way."""
    with torch.random.fork_rng(devices=[torch.cuda.current_device()] if torch.cuda.is_available() else []):
        yield


def _st():
    return torch.cuda.current_stream().cuda_stream


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _split(X, ld, ones_col=-1):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr
    rows, cols = X.shape
    hi = torch.zeros(rows, ld, dtype=torch.bfloat16, device=DEV)
    lo = torch.zeros(rows, ld, dtype=torch.bfloat16, device=DEV)
    call('dae_split_bf16', ptr(X), rows, cols, X.stride(0), ptr(hi), ptr(lo), ld, ones_col, 1.0, _st())
    return hi, lo


def _gemm_ws():
    from dae_rnn_news_recommendation_b200 import _cabi
    return torch.empty(_cabi.query('dae_gemm_det_workspace'), dtype=torch.uint8, device=DEV)


class _Noise:
    """A 4096^3 GEMM on a second stream, issued before every measured launch: the kernels under test share the SMs with it."""

    def __init__(self):
        g = torch.Generator(device=DEV).manual_seed(5)
        self.a = torch.randn(4096, 4096, device=DEV, generator=g)
        self.s = torch.cuda.Stream(device=DEV)

    def kick(self):
        self.s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.s):
            self.b = self.a @ self.a

    def join(self):
        torch.cuda.current_stream().wait_stream(self.s)


# ---- the GEMMs: [dW | dbv] = dZ^T.[E | 1], dE = dZ.W, and batch_all's alpha (G + G^T).E --------------------------------------------
@pytest.mark.parametrize('B,F,H', [(800, 10000, 500), (333, 1234, 77)])
def test_stream_k_gemms_are_bitwise_repeatable_and_accurate(B, F, H):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr
    g = torch.Generator(device=DEV).manual_seed(B + F + H)
    dZ = torch.randn(B, F, device=DEV, generator=g) * 1e-3
    E = torch.rand(B, H, device=DEV, generator=g)
    W = torch.randn(F, H, device=DEV, generator=g) * 0.05
    Hp, Fp = (H + 1 + 63) // 64 * 64, (F + 31) // 32 * 32
    dZhl, Ehl, Whl = _split(dZ, Fp), _split(E, Hp, ones_col=H), _split(W, Hp)
    ws = _gemm_ws()
    noise = _Noise()
    want_dW = (dZ.double().t() @ E.double()).cpu().numpy()
    want_dbv = dZ.double().sum(0).cpu().numpy()
    want_dE = (dZ.double() @ W.double()).cpu().numpy()
    outs = []
    for _ in range(10):
        dW = torch.full((F, H), 7.0, device=DEV)       # stored, not accumulated: the fill must disappear
        dbv = torch.full((F,), 7.0, device=DEV)
        dE = torch.full((B, H), 7.0, device=DEV)
        noise.kick()
        call('dae_gemm_bf16x3_det', F, H + 1, B, 1.0, ptr(dZhl[0]), ptr(dZhl[1]), Fp, 1, ptr(Ehl[0]), ptr(Ehl[1]), Hp, 1, ptr(dW), H, H,
             H, ptr(dbv), -1, 0, ptr(ws), ws.numel(), _st())
        call('dae_gemm_bf16x3_det', B, H, F, 1.0, ptr(dZhl[0]), ptr(dZhl[1]), Fp, 0, ptr(Whl[0]), ptr(Whl[1]), Hp, 1, ptr(dE), H, 0,
             -1, None, -1, 0, ptr(ws), ws.numel(), _st())
        noise.join()
        torch.cuda.synchronize()
        outs.append((dW.cpu().numpy(), dbv.cpu().numpy(), dE.cpu().numpy()))
    for o in outs[1:]:
        for a, b in zip(o, outs[0]):
            assert np.array_equal(a, b)
    dW, dbv, dE = outs[0]
    assert rel_err(dW, want_dW) < 2e-5 and rel_err(dbv, want_dbv) < 2e-5 and rel_err(dE, want_dE) < 2e-5
    # accumulate = 1 adds onto C exactly once
    acc = torch.full((B, H), 0.5, device=DEV)
    call('dae_gemm_bf16x3_det', B, H, F, 1.0, ptr(dZhl[0]), ptr(dZhl[1]), Fp, 0, ptr(Whl[0]), ptr(Whl[1]), Hp, 1, ptr(acc), H, 0, -1,
         None, -1, 1, ptr(ws), ws.numel(), _st())
    assert rel_err(acc.cpu().numpy(), want_dE + 0.5) < 2e-5


@pytest.mark.parametrize('B,H', [(800, 500), (333, 77), (4100, 64)])
def test_sym_gemm_is_bitwise_repeatable_and_accurate(B, H):
    from dae_rnn_news_recommendation_b200._cabi import call, ptr
    g = torch.Generator(device=DEV).manual_seed(B * 7 + H)
    G = torch.randn(B, B, device=DEV, generator=g) * 1e-3
    E = torch.rand(B, H, device=DEV, generator=g)
    Bp, Hp = (B + 7) // 8 * 8, (H + 1 + 63) // 64 * 64
    Ghl, Ehl = _split(G, Bp), _split(E, Hp)
    ws = _gemm_ws()
    noise = _Noise()
    want = (0.7 * (G.double() + G.double().t()) @ E.double()).cpu().numpy()
    outs = []
    for _ in range(10):
        C = torch.full((B, H), 3.0, device=DEV)
        noise.kick()
        call('dae_gemm_sym_bf16x3_det', B, H, 0.7, ptr(Ghl[0]), ptr(Ghl[1]), Bp, ptr(Ehl[0]), ptr(Ehl[1]), Hp, ptr(C), H, 0, ptr(ws),
             ws.numel(), _st())
        noise.join()
        torch.cuda.synchronize()
        outs.append(C.cpu().numpy())
    for o in outs[1:]:
        assert np.array_equal(o, outs[0])
    assert rel_err(outs[0], want) < 2e-5


# ---- encode backward -------------------------------------------------------------------------------------------------------------------
def _stable_buckets(x, rows, vals_c):
    """(batch row, column, value) of the batch's kept entries, bucketed by column in batch-row order: np.argsort(kind='stable')."""
    r_of, c_of, v_of = [], [], []
    for r, row in enumerate(rows):
        a, b = x.indptr[row], x.indptr[row + 1]
        v = vals_c[a:b]
        keep = v != 0
        r_of.append(np.full(int(keep.sum()), r))
        c_of.append(x.indices[a:b][keep])
        v_of.append(v[keep])
    r_of, c_of, v_of = np.concatenate(r_of), np.concatenate(c_of), np.concatenate(v_of).astype(np.float32)
    order = np.argsort(c_of, kind='stable')
    return r_of[order], c_of[order], v_of[order]


def _sparse_dw_restated(x, rows, vals_c, dA, dW0, CH=64):
    """The order DESIGN 4.7 states, in float32 NumPy (every multiply and add rounded on its own): the batch's kept entries bucketed by
    column in batch-row order; chunks of CH consecutive bucketed entries; inside a chunk each column run summed in entry order; a
    column inside one chunk is its run, a column cut by chunk boundaries is the sum of its runs in chunk order; then dW0 + that."""
    r_of, c_of, v_of = _stable_buckets(x, rows, vals_c)
    n = len(c_of)
    out = dW0.copy()
    pieces = {}
    for base in range(0, n, CH):
        end = min(base + CH, n)
        q = base
        while q < end:
            c = c_of[q]
            acc = np.zeros(dA.shape[1], np.float32)
            while q < end and c_of[q] == c:
                acc = acc + v_of[q] * dA[r_of[q]]
                q += 1
            pieces.setdefault(c, []).append(acc)
    for c, ps in pieces.items():
        s = ps[0]
        for p in ps[1:]:
            s = s + p
        out[c] = out[c] + s
    return out


def _bwd_det(x, rows, vals_c, E, bh, dE, F, H, act=1):
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200._cabi import call, ptr
    B = len(rows)
    kept = np.concatenate([x.indices[x.indptr[r]:x.indptr[r + 1]][vals_c[x.indptr[r]:x.indptr[r + 1]] != 0] for r in rows])
    cap = int(len(kept))
    ws = torch.empty(_cabi.query('dae_encode_csr_bwd_det_workspace', B, F, H, cap), dtype=torch.uint8, device=DEV)
    col_count = _t(np.bincount(kept, minlength=F).astype(np.int32))
    ip, ix, vc = _t(x.indptr.astype(np.int64)), _t(x.indices.astype(np.int32)), _t(vals_c.astype(np.float32))
    dE_d, dbh = _t(dE.copy()), torch.full((H,), 9.0, device=DEV)
    rows_d, E_d, bh_d = _t(rows.astype(np.int32)), _t(E), _t(bh)     # (named: they must outlive the asynchronous kernels)
    call('dae_encode_csr_bwd_det', ptr(ip), ptr(ix), ptr(vc), ptr(rows_d), B, F, H, 1.0, ptr(E_d), ptr(bh_d), act,
         ptr(dE_d), None, H, ptr(dbh), ptr(col_count), cap, ptr(ws), ws.numel(), _st())
    dW0 = (np.random.default_rng(H).standard_normal((F, H)) * 1e-2).astype(np.float32)
    dW = _t(dW0)
    call('dae_encode_sparse_dw_add', B, F, H, cap, ptr(ws), ws.numel(), ptr(dW), _st())
    torch.cuda.synchronize()
    # the bucketed entries, read from the workspace (layout: col_start int32[F + 1] | cursors int32[F] | ent_col | ent_row | ent_val,
    # int32 / int32 / float32 [cap], every region 256-byte aligned)
    al = lambda b: (b + 255) // 256 * 256
    o = al(4 * (F + 1)) + al(4 * F)
    wb = ws.cpu().numpy()
    ent = tuple(wb[o + k * al(4 * cap):o + k * al(4 * cap) + 4 * cap].view(dt) for k, dt in enumerate((np.int32, np.int32, np.float32)))
    return dE_d.cpu().numpy(), dbh.cpu().numpy(), dW.cpu().numpy(), dW0, ent


@pytest.mark.parametrize('B,F,H', [(800, 10000, 500), (800, 3000, 37), (800, 3000, 1000), (600, 2000, 1100), (5000, 2000, 64)])
def test_encode_backward_is_bit_exact_against_the_stated_order(B, F, H):
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    N = B + 300
    x = make_sparse(N, F, 100 if F >= 10000 else 40, 'tfidf', seed=B + H)   # Zipf columns: head buckets hold hundreds of entries
    rng = np.random.default_rng(B * 3 + H)
    vals_c = (x.data * (rng.random(x.nnz) >= 0.3)).astype(np.float32)       # masking noise: zeros are dropped from the buckets
    rows = rng.permutation(N)[:B].astype(np.int64)
    E = rng.random((B, H)).astype(np.float32) * 0.5
    bh = (rng.standard_normal(H) * 0.1).astype(np.float32)
    dE = (rng.standard_normal((B, H)) * 1e-2).astype(np.float32)
    noise = _Noise()
    runs = []
    for _ in range(3):
        noise.kick()
        runs.append(_bwd_det(x, rows, vals_c, E, bh, dE, F, H))
        noise.join()
    for r in runs[1:]:
        for a, b in zip(r[:4], runs[0][:4]):
            assert np.array_equal(a, b)
    dA, dbh, dW, dW0, (ent_col, ent_row, ent_val) = runs[0]
    # the stable buckets: exactly np.argsort(batch columns, kind='stable') of the batch's kept (row, column, value) entries
    r_of, c_of, v_of = _stable_buckets(x, rows, vals_c)
    assert np.array_equal(ent_col, c_of) and np.array_equal(ent_row, r_of) and np.array_equal(ent_val, v_of)
    counts = np.bincount(np.concatenate([x.indices[x.indptr[r]:x.indptr[r + 1]] for r in rows]), minlength=F)
    assert counts.max() >= 100                                              # the head column's bucket spans several chunks
    assert np.array_equal(dW, _sparse_dw_restated(x, rows, vals_c, dA, dW0))
    # against fp64: sparse dW = X_c^T . dA (dA as computed), dbh = sum_r (dA - f'(bh) dE)
    Xc = sp.csr_matrix((vals_c, x.indices, x.indptr), shape=x.shape)[rows].astype(np.float64)
    want = dW0.astype(np.float64) + Xc.T @ dA.astype(np.float64)
    assert rel_err(dW - dW0, want - dW0) < 1e-5
    fb = 1.0 / (1.0 + np.exp(-bh.astype(np.float64)))
    fa = E.astype(np.float64) + fb
    assert rel_err(dA, dE * fa * (1.0 - fa)) < 1e-5
    want_dbh = (dA.astype(np.float64) - fb * (1.0 - fb) * dE.astype(np.float64)).sum(0)
    assert np.abs(dbh - want_dbh).max() < 1e-5 * max(1.0, float(np.abs(dA).sum(0).max()))


# ---- whole runs ----------------------------------------------------------------------------------------------------------------------
def _fit(kind, N, F, ncomp, batch, **kw):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder, DenoisingAutoencoderTriplet
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels, perturb_rows
    V = 300                                     # validation rows: their costs are part of what must reproduce
    x = make_sparse(N + V, F, 30, kind, seed=N)
    xv, x = x[N:], x[:N]
    common = dict(model_name='d', main_dir='d', compress_factor=F // ncomp, enc_act_func='sigmoid', dec_act_func='sigmoid',
                  num_epochs=2, batch_size=float(batch), verbose=False, verbose_step=1, seed=3, corr_type='masking', corr_frac=0.3,
                  learning_rate=0.05, deterministic=True)
    common.update(kw)
    if common.get('triplet_strategy') == 'explicit':
        del common['triplet_strategy']
        data = {'org': x, 'pos': perturb_rows(x, 0.3, seed=4), 'neg': make_sparse(N, F, 30, 'binary', seed=N + 1)}
        val = {'org': xv, 'pos': perturb_rows(xv, 0.3, seed=5), 'neg': make_sparse(V, F, 30, 'binary', seed=N + 2)}
        m = DenoisingAutoencoderTriplet(**common)
        m.fit(data, val)
        emb = m.transform(x)
    else:
        lab = make_labels(N + V, 4, seed=N)
        m = DenoisingAutoencoder(**common)
        m.fit(x, xv, lab[:N], lab[N:])
        emb = m.transform(x)
    e = m.engine
    assert e.deterministic and e.enc_bwd_mode == 'det'
    slots = [t.cpu().numpy() for t in (e.theta, e.slot1, e.slot2) if t is not None]
    scal = [np.asarray(v, dtype=np.float64) for v in (*m.train_cost_batch, m.fraction_triplet_batch, m.num_triplet_batch)]
    scal.append(np.array([m.validation_cost[k] for k in sorted(m.validation_cost)]))
    scal.extend(getattr(m, 'history', []))
    return slots, scal, emb


CASES = [
    dict(kind='binary', N=1100, F=2000, ncomp=50, batch=256, triplet_strategy='none', loss_func='cross_entropy', opt='adam'),
    dict(kind='tfidf', N=1100, F=2000, ncomp=50, batch=256, triplet_strategy='batch_all', loss_func='mean_squared',
         opt='gradient_descent', rng_mode='numpy'),
    dict(kind='binary', N=1100, F=2000, ncomp=63, batch=256, triplet_strategy='batch_hard', loss_func='cosine_proximity', opt='adam'),
    dict(kind='binary', N=2100, F=1500, ncomp=30, batch=1000, triplet_strategy='batch_hard', loss_func='cross_entropy',
         opt='gradient_descent', mining_block_rows=128),
    dict(kind='binary', N=700, F=1500, ncomp=30, batch=200, triplet_strategy='explicit', loss_func='cross_entropy', opt='adam'),
]


@pytest.mark.parametrize('case', CASES, ids=lambda c: '%s-%s-%s' % (c['triplet_strategy'], c['loss_func'], c['opt']))
def test_two_seeded_fits_are_bit_identical(case):
    a = _fit(**case)
    b = _fit(**case)
    for x, y in zip(a[0], b[0]):
        assert np.array_equal(x, y)
    assert len(a[1][0]) > 0
    for x, y in zip(a[1], b[1]):
        assert np.array_equal(x, y)
    assert np.array_equal(a[2], b[2])


def test_replayed_graph_with_branches_equals_eager_single_stream_steps():
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    F, H, B, steps = 3000, 100, 400, 20
    x = make_sparse(B * steps, F, 40, 'tfidf', seed=71)
    keep = np.random.default_rng(72).random(x.nnz) >= 0.3
    labels = make_labels(B * steps, 4, seed=73)
    W0 = xavier(F, H, 74)
    for strategy in ('batch_all', 'batch_hard', 'none'):
        res = []
        for mode in ('eager', 'graph'):
            eng = TrainEngine(F, H, device=DEV, opt='adam', learning_rate=0.01, triplet_strategy=strategy, deterministic=True)
            eng.set_parameters(W0)
            eng.set_data(DeviceCSR(x, eng.device), _t((x.data * keep).astype(np.float32)), _t(labels))
            perm = _t(np.random.default_rng(75).permutation(B * steps).astype(np.int32))
            log = torch.zeros(steps, 16, dtype=torch.float64, device=eng.device)
            if mode == 'eager':
                eng.fork_branches = False
                for s in range(steps):
                    eng.step(perm, s * B, B, log[s])
            else:
                eng.capture_step_graph(perm, B, log)
                eng.set_step_cursor(0, 0)
                for s in range(steps):
                    eng.replay_step()
            torch.cuda.synchronize()
            res.append((log.cpu().numpy().copy(), eng.theta.cpu().numpy(), eng.slot1.cpu().numpy(), eng.slot2.cpu().numpy()))
            del eng
        for u, v in zip(res[0], res[1]):
            assert np.array_equal(u, v), strategy


@pytest.mark.parametrize('strategy,kind', [('batch_all', 'tfidf'), ('batch_hard', 'binary')])
def test_c2_step_against_oracle_and_default_mode(strategy, kind):
    """One C2-size step (B = 800, F = 10 000, H = 500): within 1e-4 of the fp64 oracle, as the default mode is, and within 1e-5 of it."""
    from oracle.dae_oracle import OracleDAE
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    B, F, H = 800, 10000, 500
    x = make_sparse(B, F, 100, kind, seed=21)
    labels = make_labels(B, 4, seed=21)
    keep = np.random.default_rng(22).random(x.nnz) >= 0.3
    xc = x.copy()
    xc.data = (xc.data * keep).astype(np.float32)
    W0 = xavier(F, H, 23)
    out = {}
    for det in (False, True):
        eng = TrainEngine(F, H, device=DEV, triplet_strategy=strategy, deterministic=det, **KW)
        eng.set_parameters(W0)
        eng.set_data(DeviceCSR(x, eng.device), _t(xc.data), _t(labels))
        eng.step(None, 0, B)
        torch.cuda.synchronize()
        out[det] = (eng.read_stats(), eng.grad.cpu().numpy(), eng.theta.cpu().numpy())
        del eng
    orc = OracleDAE(W0, triplet_strategy=strategy, **KW)
    o = orc.step(x, xc, labels)
    st, g, th = out[True]
    assert rel_err(st['cost'], o['cost']) < REL_TOL and rel_err(st['triplet_loss'], o['triplet_loss']) < REL_TOL
    gW, gbh, gbv = o['grads']
    assert rel_err(g[:F * H].reshape(F, H), gW) < REL_TOL and rel_err(g[F * H + H:], gbv) < REL_TOL
    for k in ('cost', 'ae_loss', 'triplet_loss'):
        assert rel_err(st[k], out[False][0][k]) < 1e-5, k
    assert rel_err(g[:F * H], out[False][1][:F * H]) < 1e-5 and rel_err(g[F * H + H:], out[False][1][F * H + H:]) < 1e-5
    assert rel_err(th, out[False][2]) < 1e-5


def test_cli_deterministic_runs_write_identical_outputs(tmp_path):
    outs = []
    for i in range(2):
        d = tmp_path / ('run%d' % i)
        d.mkdir()
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'main_autoencoder.py'), '--model_name', 'det', '--synthetic', '1500',
                            '--max_features', '2000', '--num_epochs', '2', '--batch_size', '300', '--seed', '0', '--deterministic',
                            '--triplet_strategy', 'batch_all', '--encode_full'], cwd=d, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        files = sorted(p for p in d.rglob('*.npy'))
        assert files
        outs.append({p.relative_to(d): p.read_bytes() for p in files})
    assert outs[0].keys() == outs[1].keys()
    for k in outs[0]:
        assert outs[0][k] == outs[1][k], k


@pytest.mark.parametrize('sweep', ['shared', 'tiled', 'blocked'])
def test_batch_all_anchors_without_triplets_add_nothing(sweep):
    """Anchors whose label is alone in the batch, and a batch of one label, have no valid triplet: their loss slots must add 0, as
    the atomic path does -- also after an earlier batch left other values in those slots.  The three batch_all sweeps: shared memory,
    the tiled sweep (forced), the tiled sweep on 128-row anchor blocks."""
    from dae_rnn_news_recommendation_b200._cabi import call
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    F, H, B = 1500, 64, 256
    x = make_sparse(3 * B, F, 30, 'binary', seed=81)
    keep = np.random.default_rng(82).random(x.nnz) >= 0.3
    rng = np.random.default_rng(83)
    lab = np.concatenate([rng.integers(0, 4, B),                          # batch 0: four classes (every slot written with a loss)
                          np.where(np.arange(B) < 40, 0, 1000 + np.arange(B)),   # batch 1: one class of 40, 216 singletons
                          np.full(B, 7)]).astype(np.float32)               # batch 2: one label (no negatives)
    W0 = xavier(F, H, 84)
    call('dae_triplet_config', 1 if sweep == 'tiled' else 0)
    try:
        logs = {}
        for det in (False, True):
            eng = TrainEngine(F, H, device=DEV, triplet_strategy='batch_all', deterministic=det,
                              mining_block_rows=128 if sweep == 'blocked' else None, **KW)
            eng.set_parameters(W0)
            eng.set_data(DeviceCSR(x, eng.device), _t((x.data * keep).astype(np.float32)), _t(lab))
            log = torch.zeros(3, 16, dtype=torch.float64, device=DEV)
            for s in range(3):
                eng.step(None, s * B, B, log[s])
            torch.cuda.synchronize()
            logs[det] = log.cpu().numpy()
            del eng
    finally:
        call('dae_triplet_config', 0)
    from dae_rnn_news_recommendation_b200._cabi import STAT
    d, a = logs[True], logs[False]
    assert np.isfinite(d).all()
    assert d[2, STAT['triplet_sum']] == 0.0 and d[2, STAT['triplet_loss']] == 0.0
    assert d[1, STAT['triplet_sum']] > 0.0
    for s in range(3):
        for k in ('cost', 'ae_loss', 'triplet_loss', 'triplet_sum', 'num', 'fraction'):
            assert abs(d[s, STAT[k]] - a[s, STAT[k]]) <= 1e-5 * max(1.0, abs(a[s, STAT[k]])), (s, k, d[s, STAT[k]], a[s, STAT[k]])
