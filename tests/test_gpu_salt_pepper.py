"""Salt-and-pepper noise on the device (dae_salt_pepper_csr, TrainEngine.corrupt_salt_pepper, fit with corr_type='salt_and_pepper'):
host-draw mode against utils.salt_and_pepper_noise bit for bit, Philox mode against the oracle's restated draws bit for bit, the
distribution, the C1 / C2 sizes and their memory, and the estimators' fits (numpy-mode parity, graph replay, determinism, triplets)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from helpers import REL_TOL, load_uci_c1, rel_err, random_csr, xavier
from salt_pepper_oracle import apply_draws, capacity, cases, philox_draws, value_range

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _corrupt(X, v, segs=None, draws=None, seed=0, epoch=0, base=0, cap=None):
    """dae_salt_pepper_csr over the row ranges segs = [(row0, n, lo, hi), ...] (default: all rows with X's lo / hi), appended.
    base: preset indptr_out[segs[0][0]].  Returns the output (indptr, indices, values) as NumPy arrays and the overflow flag."""
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    N, F = X.shape
    lo, hi = value_range(X)
    segs = [(0, N, lo, hi)] if segs is None else segs
    c = DeviceCSR(X, DEV)
    cap = capacity(X, v) + base if cap is None else cap
    ip = torch.zeros(N + 1, dtype=torch.int64, device=DEV)
    ip[segs[0][0]] = base
    ix = torch.full((max(cap, 1),), -7, dtype=torch.int32, device=DEV)
    va = torch.full((max(cap, 1),), float('nan'), dtype=torch.float32, device=DEV)
    ovf = torch.zeros(1, dtype=torch.int32, device=DEV)
    nmax = max(s[1] for s in segs)
    wsb = _cabi.query('dae_salt_pepper_workspace', nmax, ctype=ctypes.c_size_t)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    d = None if draws is None else torch.from_numpy(np.ascontiguousarray(draws, np.uint32).reshape(-1).view(np.int32)).to(DEV)
    st = torch.cuda.current_stream().cuda_stream
    for r0, n, l, h in segs:
        dp = None if d is None else d.data_ptr() + 4 * (r0 - segs[0][0]) * v
        _cabi.call('dae_salt_pepper_csr', c.indptr.data_ptr(), c.indices.data_ptr(), c.values.data_ptr(), r0, n, F, v, float(l), float(h),
                   dp, seed, epoch, ip.data_ptr(), ix.data_ptr(), va.data_ptr(), cap, ovf.data_ptr(), ws.data_ptr(), wsb, st)
    torch.cuda.synchronize()
    ipn = ip.cpu().numpy()
    top = int(ipn.max())
    return ipn, ix.cpu().numpy()[:top], va.cpu().numpy()[:top], int(ovf.item())


def _assert_rows_equal(got, want_rows, rows):
    """got = (indptr, indices, values) of the whole output; want_rows = (indptr, indices, values) of the oracle over `rows`."""
    ip, ix, va = got[:3]
    wp, wi, wv = want_rows
    for k, r in enumerate(rows):
        np.testing.assert_array_equal(ix[ip[r]:ip[r + 1]], wi[wp[k]:wp[k + 1]], err_msg='row %d' % r)
        np.testing.assert_array_equal(va[ip[r]:ip[r + 1]], wv[wp[k]:wp[k + 1]], err_msg='row %d' % r)


@pytest.mark.parametrize('name,X,v', cases(), ids=[c[0] for c in cases()])
def test_host_draws_equal_host_function(name, X, v):
    from dae_rnn_news_recommendation_b200.autoencoder import utils
    X = X.astype(np.float32)
    np.random.seed(99)
    want = utils.salt_and_pepper_noise(X, v)
    np.random.seed(99)
    draws = utils.salt_and_pepper_draws(X, v)
    ip, ix, va, ovf = _corrupt(X, v, draws=draws)
    assert ovf == 0
    np.testing.assert_array_equal(ip, want.indptr)
    np.testing.assert_array_equal(ix, want.indices)
    np.testing.assert_array_equal(va, want.data.astype(np.float32))


@pytest.mark.parametrize('name,X,v', cases(), ids=[c[0] for c in cases()])
def test_philox_equals_oracle(name, X, v):
    X = X.astype(np.float32)
    lo, hi = value_range(X)
    seed, epoch = (3 << 32) | 11, (1 << 32) | 4
    got = _corrupt(X, v, seed=seed, epoch=epoch)
    want = apply_draws(X, philox_draws(np.arange(X.shape[0]), X.shape[1], v, seed, epoch), lo, hi)
    assert got[3] == 0
    for a, b in zip(got[:3], want):
        np.testing.assert_array_equal(a, b)


def test_philox_many_windows():
    """F = 200 003 needs 13 slab windows of 16 384 columns: rows with clean entries and draws on both sides of every boundary."""
    N, F, v = 36, 200003, 60001
    rng = np.random.default_rng(1)
    X = random_csr(N, F, 40, kind='tfidf', seed=2)
    Xl = X.tolil()
    for r in range(N):                              # clean entries right at the window edges
        for b in (16383, 16384, 32767, 32768, 196607, 196608, F - 1):
            Xl[r, b] = 0.25 + 0.5 * rng.random()
    X = Xl.tocsr().astype(np.float32)
    X.sort_indices()
    lo, hi = value_range(X)
    got = _corrupt(X, v, seed=5, epoch=2)
    want = apply_draws(X, philox_draws(np.arange(N), F, v, 5, 2), lo, hi)
    for a, b in zip(got[:3], want):
        np.testing.assert_array_equal(a, b)
    assert got[0][-1] > N * 0.5 * F * (1 - np.exp(-v / F)) * 0.95


def test_row0_base_and_appended_segments():
    """Three appended calls with their own lo / hi form one stacked CSR; a call starting at row0 > 0 continues from the indptr_out entry
    the device holds (here preset to 17)."""
    N, F, v = 90, 3000, 700
    X = random_csr(N, F, 25, kind='tfidf', seed=7).astype(np.float32)
    segs = [(0, 30, -0.5, 1.0), (30, 30, 0.0, 2.0), (60, 30, 0.25, 0.0)]
    got = _corrupt(X, v, segs=segs, seed=9, epoch=1)
    assert got[3] == 0
    for r0, n, lo, hi in segs:
        rows = np.arange(r0, r0 + n)
        _assert_rows_equal(got, apply_draws(X, philox_draws(rows, F, v, 9, 1), lo, hi, rows), rows)
    assert set(np.unique(got[2][got[0][30]:got[0][60]])) - set(X.data[X.indptr[30]:X.indptr[60]]) == {2.0}
    # row0 > 0, base 17
    rows = np.arange(40, 65)
    got = _corrupt(X, v, segs=[(40, 25, -1.0, 1.0)], seed=9, epoch=1, base=17, cap=17 + capacity(X[40:65], v))
    assert got[0][40] == 17
    _assert_rows_equal(got, apply_draws(X, philox_draws(rows, F, v, 9, 1), -1.0, 1.0, rows), rows)
    # the draws of host mode are offset by row0 as well
    d = (np.arange(25 * v, dtype=np.uint32) * 7919) % F
    got = _corrupt(X, v, segs=[(40, 25, -1.0, 1.0)], draws=d, base=3, cap=3 + capacity(X[40:65], v))
    _assert_rows_equal(got, apply_draws(X, d.reshape(25, v), -1.0, 1.0, rows), rows)


def test_overflow_writes_no_entries():
    X = random_csr(50, 500, 10, seed=3).astype(np.float32)
    ip, ix, va, ovf = _corrupt(X, 100, seed=1, cap=200)
    assert ovf == 1 and (ip == 0).all()


def test_distribution_and_reproducibility():
    """Empty clean rows, lo = -1, hi = 1: a row stores every column some draw hit, F (1 - e^(-v/F)) on average, half of them hi, with
    no column bias.  The same (seed, epoch) reproduces the output; another epoch or seed draws another one."""
    N, F, v = 2000, 10000, 3000
    X = sp.csr_matrix(([1.0], ([N - 1], [0])), shape=(N, F), dtype=np.float32)   # one clean entry (= hi): the arrays are not empty
    segs = [(0, N, -1.0, 1.0)]
    ip, ix, va, _ = _corrupt(X, v, segs=segs, seed=1, epoch=0)
    frac = ip[-1] / (N * F)
    assert abs(frac - (1 - np.exp(-v / F))) < 2e-3
    assert abs(float((va == 1.0).mean()) - 0.5) < 2e-3 and set(np.unique(va)) == {-1.0, 1.0}
    per_col = np.bincount(ix, minlength=F).reshape(20, -1).sum(1) / (N * F / 20)
    assert np.abs(per_col - frac).max() < 5e-3
    again = _corrupt(X, v, segs=segs, seed=1, epoch=0)
    assert all(np.array_equal(a, b) for a, b in zip(again[:3], (ip, ix, va)))
    for other in (_corrupt(X, v, segs=segs, seed=1, epoch=1), _corrupt(X, v, segs=segs, seed=2, epoch=0)):
        dense_a = np.zeros((200, F), np.int8)
        dense_b = np.zeros((200, F), np.int8)
        for r in range(200):
            dense_a[r, ix[ip[r]:ip[r + 1]]] = va[ip[r]:ip[r + 1]]
            dense_b[r, other[1][other[0][r]:other[0][r + 1]]] = other[2][other[0][r]:other[0][r + 1]]
        p = 1 - np.exp(-v / F)                      # independent draws agree on (1-p)^2 + p^2 / 2 of the cells
        assert abs(float((dense_a == dense_b).mean()) - ((1 - p) ** 2 + p * p / 2)) < 0.01


def _engine(F, H=16, **kw):
    from dae_rnn_news_recommendation_b200.engine import TrainEngine
    base = dict(enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy', opt='gradient_descent', learning_rate=0.05,
                triplet_strategy='none')
    base.update(kw)
    return TrainEngine(F, H, device=DEV, **base)


def _engine_output(eng):
    c = eng.csr_c
    ip = c.indptr.cpu().numpy()
    return ip, c.indices[:ip[-1]].cpu().numpy(), c.values[:ip[-1]].cpu().numpy()


@pytest.mark.parametrize('which', ['C1', 'C2'])
def test_full_size_sets_sampled_rows_and_memory(which):
    """The C1 articles (8000 x 10 000 binary) and a 100 000-row C2-like tf-idf set, v = 3000: sampled rows equal the oracle, the engine's
    buffers hold sum_r min(F, nnz_r + v) entries, and the corruption's peak memory is those buffers plus the workspace."""
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    if which == 'C1':
        X = load_uci_c1()['train']
    else:
        X = make_sparse(100000, 10000, 100, 'tfidf', seed=0).astype(np.float32)
    X.sort_indices()
    N, F = X.shape
    v = int(round(0.3 * F))
    lo, hi = value_range(X)
    eng = _engine(F)
    eng.set_data(DeviceCSR(X, DEV), None, None)
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    eng.corrupt_salt_pepper(v, lo, hi, seed=4, epoch=3)
    torch.cuda.synchronize()
    cap = capacity(X, v)
    b = eng.salt_pepper_buffers(v)
    assert b['cap'] == cap and eng.csr_c.max_row_nnz == min(F, int(np.diff(X.indptr).max()) + v)
    stated = cap * 8 + (N + 1) * 8 + b['ws'].numel() + 4
    peak = torch.cuda.max_memory_allocated() - m0
    assert stated <= peak <= stated + (8 << 20), (peak, stated)
    got = _engine_output(eng)
    rows = np.sort(np.random.default_rng(0).choice(N, 300, replace=False))
    _assert_rows_equal(got, apply_draws(X, philox_draws(rows, F, v, 4, 3), lo, hi, rows), rows)
    assert got[0][-1] <= cap
    eng.check_corruption()
    print('%s: %d rows, cap %d entries (%.2f GB), %.1f stored per row' % (which, N, cap, cap * 8 / 1e9, got[0][-1] / N))


def test_engine_step_on_corrupted_copy_matches_oracle():
    """One training step on the device-corrupted copy (numpy draws) equals the oracle's step on utils.salt_and_pepper_noise's output."""
    from dae_rnn_news_recommendation_b200.autoencoder import utils
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    from oracle.dae_oracle import OracleDAE
    F, H, B = 300, 24, 80
    x = random_csr(B, F, 12, seed=51)
    labels = np.random.default_rng(52).integers(0, 3, B).astype(np.float32)
    W0 = xavier(F, H, 53) * 3
    kw = dict(enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy', opt='gradient_descent', learning_rate=0.05,
              triplet_strategy='batch_hard')
    np.random.seed(3)
    xc = utils.salt_and_pepper_noise(x, 9)
    np.random.seed(3)
    draws = utils.salt_and_pepper_draws(x, 9)
    eng = _engine(F, H, **kw)
    eng.set_parameters(W0)
    eng.set_data(DeviceCSR(x, eng.device), None, torch.from_numpy(labels).to(eng.device))
    lo, hi = value_range(x)
    eng.corrupt_salt_pepper(9, lo, hi, draws_host=draws)
    got = _engine_output(eng)
    np.testing.assert_array_equal(got[1], xc.indices)
    eng.step(None, 0, B)
    torch.cuda.synchronize()
    o = OracleDAE(W0, **kw).step(x, xc, labels)
    st = eng.read_stats()
    assert rel_err(st['cost'], o['cost']) < REL_TOL and rel_err(st['triplet_loss'], o['triplet_loss']) < REL_TOL
    g = eng.grad.cpu().numpy()
    assert rel_err(g[:F * H].reshape(F, H), o['grads'][0]) < REL_TOL


def _dae(**kw):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder
    base = dict(model_name='sp', main_dir='sp', compress_factor=10, enc_act_func='sigmoid', dec_act_func='sigmoid',
                loss_func='cross_entropy', num_epochs=3, batch_size=100, opt='gradient_descent', learning_rate=0.1, corr_type='salt_and_pepper',
                corr_frac=0.1, verbose=False, verbose_step=1, seed=5, triplet_strategy='batch_all')
    base.update(kw)
    return DenoisingAutoencoder(**base)


def _recording(monkeypatch):
    """Record the corrupted CSR of every corrupt_salt_pepper call."""
    from dae_rnn_news_recommendation_b200.engine import TrainEngine
    seen = []
    orig = TrainEngine.corrupt_salt_pepper

    def rec(self, *a, **k):
        orig(self, *a, **k)
        torch.cuda.synchronize()
        seen.append(_engine_output(self))
    monkeypatch.setattr(TrainEngine, 'corrupt_salt_pepper', rec)
    return seen


def test_fit_numpy_mode_epochs_equal_host_function(monkeypatch):
    from dae_rnn_news_recommendation_b200.autoencoder import utils
    N, F = 400, 300
    X = random_csr(N, F, 15, kind='tfidf', seed=11).astype(np.float32)
    labels = np.random.default_rng(1).integers(0, 4, N)
    seen = _recording(monkeypatch)
    m = _dae(rng_mode='numpy', W_init=xavier(F, 30, 2), loss_func='mean_squared')
    m.fit(X, train_set_label=labels)
    assert len(seen) == 3 and m.engine._graph is not None
    np.random.seed(5)
    for e in range(3):
        want = utils.salt_and_pepper_noise(X, 30)
        order = list(range(N))
        np.random.shuffle(order)
        for a, b in zip(seen[e], (want.indptr, want.indices, want.data.astype(np.float32))):
            np.testing.assert_array_equal(a, b)


def test_fit_replay_matches_eager(monkeypatch):
    N, F = 600, 400
    X = random_csr(N, F, 20, seed=12)
    labels = np.random.default_rng(2).integers(0, 4, N)
    res = []
    for graph in ('1', '0'):
        monkeypatch.setenv('DAE_CUDA_GRAPH', graph)
        m = _dae(W_init=xavier(F, 40, 3))
        m.fit(X, train_set_label=labels)
        assert (m.engine._graph is not None) == (graph == '1')
        res.append((np.concatenate(m.history), m.get_model_parameters()))
    assert rel_err(res[0][0][:, 0], res[1][0][:, 0]) < 1e-4
    assert rel_err(res[0][1]['enc_w'], res[1][1]['enc_w']) < 5e-3


def test_fit_deterministic_device_mode_bit_identical():
    N, F = 500, 300
    X = random_csr(N, F, 20, seed=13)
    labels = np.random.default_rng(3).integers(0, 4, N)
    out = []
    for _ in range(2):
        m = _dae(deterministic=True, rng_mode='device', W_init=xavier(F, 30, 4))
        m.fit(X, train_set_label=labels)
        out.append((m.get_model_parameters(), np.concatenate(m.history)))
    for k in ('enc_w', 'enc_b', 'dec_b'):
        assert np.array_equal(out[0][0][k], out[1][0][k])
    assert np.array_equal(out[0][1], out[1][1])


@pytest.mark.parametrize('rng_mode', ['numpy', 'device'])
def test_triplet_estimator(rng_mode, monkeypatch):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoderTriplet, utils
    N, F, v = 120, 200, 20
    data = {k: random_csr(N, F, 10, kind=kind, seed=s).astype(np.float32)
            for k, kind, s in (('org', 'binary', 61), ('pos', 'tfidf', 62), ('neg', 'binary', 63))}
    data['neg'] = data['neg'] * 3.0
    seen = _recording(monkeypatch)
    m = DenoisingAutoencoderTriplet(model_name='t', main_dir='t', compress_factor=10, enc_act_func='sigmoid', dec_act_func='sigmoid',
                                    loss_func='cross_entropy', num_epochs=2, batch_size=40.0, opt='gradient_descent', learning_rate=0.05,
                                    corr_type='salt_and_pepper', corr_frac=0.1, verbose=False, verbose_step=1, seed=5, alpha=2,
                                    W_init=xavier(F, 20, 64), rng_mode=rng_mode)
    m.fit(data)
    assert len(seen) == 2 and np.isfinite(m.train_cost_batch[0]).all() and m.engine._graph is not None
    keys = ('org', 'pos', 'neg')
    if rng_mode == 'numpy':
        np.random.seed(5)
        for e in range(2):
            want = sp.vstack([utils.salt_and_pepper_noise(data[k], v) for k in keys]).tocsr()
            order = list(range(N))
            np.random.shuffle(order)
            for a, b in zip(seen[e], (want.indptr, want.indices, want.data.astype(np.float32))):
                np.testing.assert_array_equal(a, b)
    else:
        stacked = sp.vstack([data[k] for k in keys]).tocsr()
        for e in range(2):
            for s, k in enumerate(keys):
                rows = np.arange(s * N, (s + 1) * N)
                lo, hi = value_range(data[k])
                _assert_rows_equal(seen[e], apply_draws(stacked, philox_draws(rows, F, v, 5, e), lo, hi, rows), rows)


def test_cli_salt_and_pepper():
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    model = cli.main(['--model_name', 'sp', '--synthetic', '4000', '--corr_type', 'salt_and_pepper', '--num_epochs', '2', '--seed', '3'])
    assert len(model.history) == 2 and np.isfinite(model.history[-1]).all()
