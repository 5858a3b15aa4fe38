"""The host-feed training path -- HostFeed, TrainEngine.run_feed and the streamed TrainEngine.run_feeds (three device feed buffers
with one captured graph each, H2D copies on a copy stream, the next batch staged from the next buffer's labels, the scalars through
a device log and a pinned ring, chunks of LOG_ROWS feeds) -- against the fp64 oracle on every strategy, and bit for bit against eager
single-stream steps in deterministic mode: feed counts around the three buffers, the log chunking, layout changes, the poisoned padding
of a feed, batches without triplets, the optimizer's step counter across eager and replayed steps, and feeds without labels."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from helpers import REL_TOL, rel_err, random_csr, xavier

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(autouse=True)
def _tensor_core_path(monkeypatch):
    monkeypatch.setenv('DAE_GEMM', 'tc')
    monkeypatch.delenv('DAE_CUDA_GRAPH', raising=False)
    monkeypatch.delenv('DAE_DETERMINISTIC', raising=False)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _engine(F, H, strategy, W0, opt='adam', lr=0.01, loss='cross_entropy', enc='sigmoid', dec='sigmoid', **kw):
    from dae_rnn_news_recommendation_b200.engine import TrainEngine
    eng = TrainEngine(F, H, device=DEV, enc_act_func=enc, dec_act_func=dec, loss_func=loss, opt=opt, learning_rate=lr, momentum=0.5,
                      alpha=1.0, triplet_strategy=strategy, **kw)
    eng.set_parameters(W0)
    return eng


def _batches(n, B, F, nnz_row, seed, kind='binary', labelled=True, n_classes=4, make=None):
    """n batches (x: canonical CSR, xc: masked values in x's entry order, labels or None); B rows each (explicit: 3 x B/3 stacked)."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(n):
        x = random_csr(B, F, nnz_row, kind=kind, seed=seed * 1000 + s) if make is None else make(B, F, nnz_row, kind, seed * 1000 + s)
        xc = (x.data * (rng.random(x.nnz) >= 0.3)).astype(np.float32)
        out.append((x, xc, rng.integers(0, n_classes, B).astype(np.float32) if labelled else None))
    return out


def _feeds(batches, cap):
    from dae_rnn_news_recommendation_b200.engine import HostFeed
    return [HostFeed(x, xc, lb, cap_nnz=cap) for x, xc, lb in batches]


def _state(eng):
    return [t.cpu().numpy().copy() for t in (eng.theta, eng.slot1, eng.slot2) if t is not None]


def _eager_step(eng, x, xc, lb):
    """One eager step on a DeviceCSR of the batch (what run_feed replays from the feed buffer)."""
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    eng.set_data(DeviceCSR(x, eng.device), _t(xc), None if lb is None else _t(lb))
    if eng.strategy == 3:
        n = x.shape[0] // 3
        eng.step_explicit(None, 0, n, n)
    else:
        eng.step(None, 0, x.shape[0])
    torch.cuda.synchronize()
    return eng.read_stats()


def _eager_run(make_engine, batches):
    """The reference trajectory: eager steps on ONE stream (no parallel branches)."""
    eng = make_engine()
    eng.fork_branches = False
    stats = [_eager_step(eng, *b) for b in batches]
    return stats, _state(eng)


def _run_schedule(eng, feeds, schedule):
    """schedule: n = one run_feeds call on the next n feeds, 'f' = one run_feed call on the next feed."""
    out, i = [], 0
    for s in schedule:
        if s == 'f':
            out.append(eng.run_feed(feeds[i]))
            i += 1
        else:
            out.extend(eng.run_feeds(feeds[i:i + s]))
            i += s
    assert i == len(feeds)
    return out


def _assert_same(got_stats, got_state, want_stats, want_state, what):
    assert len(got_stats) == len(want_stats), what
    for j, (g, w) in enumerate(zip(got_stats, want_stats)):
        for k in w:
            assert g[k] == w[k], (what, 'step %d' % j, k, g[k], w[k])
    assert len(got_state) == len(want_state)
    for name, g, w in zip(('theta', 'slot1', 'slot2'), got_state, want_state):
        assert np.array_equal(g, w), (what, name, float(np.abs(g - w).max()))


# ---- 1. every strategy against the fp64 oracle, feed by feed ------------------------------------------------------------------------
def _oracle_step(orc, strategy, x, xc, lb):
    xcm = x.copy()
    xcm.data = xc
    if strategy == 'explicit':
        n = x.shape[0] // 3
        o = orc.step_explicit([x[i * n:(i + 1) * n] for i in range(3)], [xcm[i * n:(i + 1) * n] for i in range(3)])
    else:
        o = orc.step(x, xcm, lb)
    f = lambda k: float(np.asarray(o[k]))
    want = {'cost': f('cost'), 'ae_loss': f('autoencoder_loss'), 'triplet_loss': 0.0, 'num': 0.0, 'fraction': 0.0}
    if strategy != 'none':
        want['triplet_loss'] = f('triplet_loss')
    if strategy in ('batch_all', 'batch_hard'):
        want.update(num=f('num'), fraction=f('fraction'))
    return want, o['grads']


def _check_scalars(st, want, what):
    assert rel_err(st['cost'], want['cost']) < REL_TOL, (what, st['cost'], want['cost'])
    assert rel_err(st['ae_loss'], want['ae_loss']) < REL_TOL, (what, st['ae_loss'], want['ae_loss'])
    assert abs(st['triplet_loss'] - want['triplet_loss']) <= REL_TOL * max(abs(want['triplet_loss']), 1e-3), \
        (what, st['triplet_loss'], want['triplet_loss'])
    assert st['num'] == pytest.approx(want['num'], rel=1e-3, abs=2.0), (what, st['num'], want['num'])
    assert st['fraction'] == pytest.approx(want['fraction'], rel=1e-3, abs=1e-5), (what, st['fraction'], want['fraction'])


def _check_grads(eng, grads, F, H, what, bh_scale=False):
    gW, gbh, gbv = grads
    g = eng.grad.cpu().numpy()
    assert rel_err(g[:F * H].reshape(F, H), gW) < REL_TOL, (what, 'dW')
    assert rel_err(g[F * H + H:], gbv) < REL_TOL, (what, 'dbv')
    if bh_scale:   # dbh = sum_i dA_i - f'(bh) sum_i dE_i cancels almost completely at bh = 0: compare against the scale of its terms
        assert np.abs(g[F * H:F * H + H] - gbh).max() < REL_TOL * max(float(np.abs(gW).max()), float(np.abs(gbh).max())), (what, 'dbh')
    else:
        assert rel_err(g[F * H:F * H + H], gbh) < REL_TOL, (what, 'dbh')


def _check_params(eng, orc, what, bh_scale=False):
    p, q = eng.get_parameters(), orc.get_parameters()
    for k in ('enc_w', 'dec_b') if bh_scale else ('enc_w', 'enc_b', 'dec_b'):   # (bh_scale: bh moves by the cancelling dbh)
        assert rel_err(p[k], q[k]) < REL_TOL, (what, k, rel_err(p[k], q[k]))


def _oracle_case(strategy, F, H, batches, W0, orc, kw, bh_scale=False):
    cap = max(b[0].nnz for b in batches) + 13
    eng = _engine(F, H, strategy, W0, **kw)
    traj = []
    for s, (b, f) in enumerate(zip(batches, _feeds(batches, cap))):
        st = eng.run_feed(f)
        want, grads = _oracle_step(orc, strategy, *b)
        _check_scalars(st, want, ('run_feed', s))
        _check_grads(eng, grads, F, H, ('run_feed', s), bh_scale)
        _check_params(eng, orc, ('run_feed', s), bh_scale)
        traj.append(want)
    assert eng.step_count == len(batches)
    del eng
    eng = _engine(F, H, strategy, W0, **kw)
    outs = eng.run_feeds(_feeds(batches, cap))
    assert len(outs) == len(batches) and eng.step_count == len(batches)
    for s, (st, want) in enumerate(zip(outs, traj)):
        _check_scalars(st, want, ('run_feeds', s))
    _check_params(eng, orc, 'run_feeds', bh_scale)


@pytest.mark.parametrize('strategy', ['none', 'batch_all', 'batch_hard', 'explicit'])
@pytest.mark.parametrize('loss,enc,dec,kind,opt', [('cross_entropy', 'sigmoid', 'sigmoid', 'binary', 'momentum'),
                                                   ('mean_squared', 'tanh', 'none', 'tfidf', 'gradient_descent')])
def test_feeds_follow_the_fp64_oracle(strategy, loss, enc, dec, kind, opt):
    from oracle.dae_oracle import OracleDAE
    F, H, B = 300, 24, 96
    batches = _batches(4, B, F, 10, seed=1, kind=kind, labelled=strategy != 'explicit')
    W0 = xavier(F, H, 2) * 3
    kw = dict(opt=opt, lr=0.05, loss=loss, enc=enc, dec=dec)
    orc = OracleDAE(W0, enc_act_func=enc, dec_act_func=dec, loss_func=loss, opt=opt, learning_rate=0.05, momentum=0.5, alpha=1.0,
                    triplet_strategy='none' if strategy == 'explicit' else strategy, dtype=torch.float64)
    _oracle_case(strategy, F, H, batches, W0, orc, kw)


def _bench_rows(B, F, nnz, kind, seed):
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    return make_sparse(B, F, nnz, kind, seed=seed)


def test_c2_feeds_follow_the_fp64_oracle():
    """BASELINE C2: B = 800, F = 10 000, H = 500, tf-idf, batch_all (the oracle mines in chunks, in fp64 on the GPU with torch ops)."""
    from oracle.chunked_oracle import ChunkedOracleDAE
    F, H, B = 10000, 500, 800
    batches = _batches(4, B, F, 100, seed=3, kind='tfidf', make=_bench_rows)
    W0 = xavier(F, H, 4)
    kw = dict(opt='gradient_descent', lr=0.1)
    orc = ChunkedOracleDAE(W0, device=DEV, enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy',
                           opt='gradient_descent', learning_rate=0.1, alpha=1.0, triplet_strategy='batch_all')
    _oracle_case('batch_all', F, H, batches, W0, orc, kw, bh_scale=True)


def test_c5_stacked_feeds_follow_the_fp64_oracle():
    """BASELINE C5: explicit triplets, 3 x 800 stacked [org; pos; neg] rows per feed, binary, F = 10 000, H = 500.  Learning rate 0.01:
    at C5's 0.1 these unrelated random rows make the cost diverge within three steps (20 792 -> 227 479), where the decode's sigmoid
    saturates and any fp32 computation, the fp32 oracle's included, leaves the fp64 trajectory by percents."""
    from oracle.dae_oracle import OracleDAE
    F, H, B = 10000, 500, 3 * 800
    batches = _batches(4, B, F, 100, seed=5, kind='binary', labelled=False, make=_bench_rows)
    W0 = xavier(F, H, 6)
    kw = dict(opt='gradient_descent', lr=0.01)
    orc = OracleDAE(W0, enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy', opt='gradient_descent',
                    learning_rate=0.01, alpha=1.0, triplet_strategy='none', dtype=torch.float64)
    _oracle_case('explicit', F, H, batches, W0, orc, kw, bh_scale=True)


# ---- 2. deterministic mode: streamed feeds == eager single-stream steps, bit for bit --------------------------------------------------
@pytest.mark.parametrize('strategy', ['batch_all', 'batch_hard', 'none', 'explicit'])
def test_deterministic_feeds_equal_eager_steps_bit_for_bit(strategy):
    """12 feeds in two call patterns: 1 feed (the first capture), 7 in one call (the three buffers wrap twice), run_feed in between,
    then 3; and 2, run_feed, 1 (one streamed feed), 4, run_feed, 3.  Adam, so the step counter on the device matters too."""
    F, H, B = 400, 32, 96
    batches = _batches(12, B, F, 12, seed=7, labelled=strategy != 'explicit')
    W0 = xavier(F, H, 8) * 3
    make = lambda: _engine(F, H, strategy, W0, deterministic=True)
    want = _eager_run(make, batches)
    feeds = _feeds(batches, max(b[0].nnz for b in batches) + 5)
    for schedule in ([1, 7, 'f', 3], [2, 'f', 1, 4, 'f', 3]):
        eng = make()
        got = _run_schedule(eng, feeds, schedule)
        assert eng.step_count == 12
        _assert_same(got, _state(eng), *want, (strategy, schedule))
        del eng


# ---- 3. the padding of a feed and the edges of a batch --------------------------------------------------------------------------------
def _gaps(f):
    """The byte ranges of f.host that carry no data: alignment gaps and the padding between the real nnz and cap_nnz."""
    n = int(f.host.numpy()[:8 * (f.B + 1)].view(np.int64)[-1])
    return n, [(8 * (f.B + 1), f.off_indices), (f.off_labels + 4 * f.B, f.nbytes)], \
        [(f.off_indices, f.off_values), (f.off_values, f.off_values_c), (f.off_values_c, f.off_labels)]


def _fill_padding(f, F, poison):
    """poison: column ids >= F and negative ones, NaN values, 0xFF bytes in the alignment gaps; else zeros everywhere."""
    hb = f.host.numpy()
    n, gaps, parts = _gaps(f)
    for a, b in gaps:
        hb[a:b] = 0xFF if poison else 0
    (ia, ib), (va, vb), (ca, cb) = parts
    idx = hb[ia:ib].view(np.int32)
    idx[n:] = np.where(np.arange(idx.size - n) % 2 == 0, F + 7, -5) if poison else 0
    for a, b in ((va, vb), (ca, cb)):
        hb[a:b].view(np.float32)[n:] = np.nan if poison else 0.0
    return f


def _drop_rows(x, rows):
    c = x.tocoo()
    keep = ~np.isin(c.row, rows)
    return sp.csr_matrix((c.data[keep], (c.row[keep], c.col[keep])), shape=x.shape)


@pytest.mark.parametrize('strategy', ['batch_all', 'batch_hard', 'none'])
def test_poisoned_padding_and_batch_edges(strategy):
    """Feeds of one layout: real nnz == cap_nnz; a batch far below the cap; empty rows; one class only (no valid triplet); then a
    two-row layout of two classes with one row each.  With the padding poisoned, every feed trains bit for bit as with zero padding
    and as eager steps on the batches themselves, and every output is finite."""
    F, H, B = 400, 32, 64
    rng = np.random.default_rng(9)
    full = random_csr(B, F, 24, seed=10)
    sparse = random_csr(B, F, 2, seed=11)
    holes = _drop_rows(random_csr(B, F, 12, seed=12), [0, 17, 63])
    one_class = random_csr(B, F, 12, seed=13)
    xs = [full, sparse, holes, one_class, random_csr(B, F, 3, seed=14)]
    labels = [rng.integers(0, 4, B).astype(np.float32) for _ in xs]
    labels[3][:] = 3.0
    main = [(x, (x.data * (rng.random(x.nnz) >= 0.3)).astype(np.float32), lb) for x, lb in zip(xs, labels)]
    cap = full.nnz
    assert all(x.nnz <= cap for x in xs) and sparse.nnz * 4 < cap and holes.indptr[1] == 0
    pairs = [random_csr(2, F, 12, seed=15 + i) for i in range(2)]
    two = [(x, x.data.astype(np.float32), np.array([0.0, 1.0], np.float32)) for x in pairs]
    cap2 = max(x.nnz for x in pairs) + 40
    W0 = xavier(F, H, 16) * 3
    make = lambda: _engine(F, H, strategy, W0, deterministic=True)
    want = _eager_run(make, main + two)
    for s in want[0]:
        assert all(np.isfinite(v) for v in s.values()), s
    assert all(np.isfinite(t).all() for t in want[1])
    results = {}
    for kind in ('clean', 'poisoned'):
        mk = lambda: [_fill_padding(f, F, kind == 'poisoned') for f in _feeds(main, cap)] + \
            [_fill_padding(f, F, kind == 'poisoned') for f in _feeds(two, cap2)]
        eng = make()
        fs = mk()
        results[kind, 'run_feeds'] = (eng.run_feeds(fs[:5]) + eng.run_feeds(fs[5:]), _state(eng))
        eng = make()
        results[kind, 'run_feed'] = ([eng.run_feed(f) for f in mk()], _state(eng))
    for k, (st, state) in results.items():
        _assert_same(st, state, *want, (strategy,) + k)


# ---- 4. streaming boundaries --------------------------------------------------------------------------------------------------------
def test_log_chunking_over_1026_feeds():
    """One run_feeds call of 1 026 feeds: the first captures the layout, the other 1 025 stream in chunks of LOG_ROWS = 1 024 and 1."""
    F, H, B, n = 400, 32, 64, 1026
    batches = _batches(n, B, F, 12, seed=17)
    W0 = xavier(F, H, 18) * 3
    make = lambda: _engine(F, H, 'batch_all', W0, deterministic=True)
    want = _eager_run(make, batches)
    eng = make()
    got = eng.run_feeds(_feeds(batches, max(b[0].nnz for b in batches)))
    assert eng.step_count == n
    _assert_same(got, _state(eng), *want, 'run_feeds(1026)')


def test_layout_changes_recapture():
    """run_feeds on layout A, then B (another batch size and cap), then A again: each call captures its layout anew and the whole run
    follows the eager trajectory."""
    F, H = 400, 32
    a1, b1, a2 = _batches(3, 64, F, 12, seed=19), _batches(3, 96, F, 12, seed=20), _batches(3, 64, F, 12, seed=21)
    cap_a, cap_b = max(b[0].nnz for b in a1 + a2) + 3, max(b[0].nnz for b in b1) + 50
    W0 = xavier(F, H, 22) * 3
    make = lambda: _engine(F, H, 'batch_hard', W0, deterministic=True)
    want = _eager_run(make, a1 + b1 + a2)
    eng = make()
    got, streams = [], []
    for batches, cap in ((a1, cap_a), (b1, cap_b), (a2, cap_a)):
        got += eng.run_feeds(_feeds(batches, cap))
        assert eng._feed_stream['owner'] is eng._feed_graph and eng._feed_graph[0][:2] == (batches[0][0].shape[0], cap)
        streams.append(eng._feed_stream)
    assert streams[0] is not streams[1] and streams[1] is not streams[2]
    _assert_same(got, _state(eng), *want, 'A -> B -> A')


def test_without_graphs_feeds_give_the_same_trajectory(monkeypatch):
    """DAE_CUDA_GRAPH=0: run_feed / run_feeds run every feed eagerly, with the same results as the replayed graphs."""
    F, H, B = 400, 32, 64
    batches = _batches(6, B, F, 12, seed=23)
    W0 = xavier(F, H, 24) * 3
    make = lambda: _engine(F, H, 'batch_all', W0, deterministic=True)
    want = _eager_run(make, batches)
    cap = max(b[0].nnz for b in batches) + 7
    feeds = _feeds(batches, cap)
    eng = make()
    _assert_same(_run_schedule(eng, feeds, [3, 'f', 2]), _state(eng), *want, 'graphs')
    monkeypatch.setenv('DAE_CUDA_GRAPH', '0')
    eng = make()
    _assert_same(_run_schedule(eng, feeds, [3, 'f', 2]), _state(eng), *want, 'DAE_CUDA_GRAPH=0')
    assert eng._feed_graph is None and eng._feed_stream is None


@pytest.mark.parametrize('strategy', ['batch_all', 'batch_hard'])
def test_block_mined_engine_streams_feeds(strategy):
    """mining_block_rows=128 at B = 800: the streamed step stages the next batch with dae_batch_prepare_next_blocked."""
    F, H, B = 1000, 32, 800
    batches = _batches(4, B, F, 12, seed=25)
    W0 = xavier(F, H, 26) * 3
    make = lambda: _engine(F, H, strategy, W0, deterministic=True, mining_block_rows=128)
    want = _eager_run(make, batches)
    eng = make()
    assert eng._prepare_next == 'dae_batch_prepare_next_blocked'
    got = _run_schedule(eng, _feeds(batches, max(b[0].nnz for b in batches)), [1, 3])
    _assert_same(got, _state(eng), *want, strategy)


# ---- 5. Adam's step counter across eager and replayed steps -----------------------------------------------------------------------------
def test_optimizer_step_counter_continues_across_eager_and_replayed_steps():
    """run_feed (replayed), 2 eager step() calls, run_feed (replayed), run_feed without cap_nnz (eager), run_feeds, run_feed (replayed):
    the replays must take Adam's step t from the steps taken so far, eager ones included."""
    F, H, B = 400, 32, 64
    batches = _batches(9, B, F, 12, seed=27)
    W0 = xavier(F, H, 28) * 3
    make = lambda: _engine(F, H, 'batch_all', W0, deterministic=True, lr=0.02)
    want = _eager_run(make, batches)
    from dae_rnn_news_recommendation_b200.engine import HostFeed
    feeds = _feeds(batches, max(b[0].nnz for b in batches) + 2)
    eng = make()
    got = [eng.run_feed(feeds[0])]
    got += [_eager_step(eng, *batches[1]), _eager_step(eng, *batches[2])]
    got.append(eng.run_feed(feeds[3]))
    got.append(eng.run_feed(HostFeed(*batches[4])))
    got += eng.run_feeds(feeds[5:8])
    got.append(eng.run_feed(feeds[8]))
    assert eng.step_count == 9
    _assert_same(got, _state(eng), *want, 'mixed')


# ---- 6. feeds without labels ------------------------------------------------------------------------------------------------------------
def test_feeds_without_labels():
    """Accepted by triplet_strategy='none' (and equal to the fp64 oracle); refused by the triplet strategies before anything is captured,
    after which the engine still trains on a labelled feed."""
    from oracle.dae_oracle import OracleDAE
    F, H, B = 300, 24, 64
    batches = _batches(6, B, F, 10, seed=29, labelled=False)
    W0 = xavier(F, H, 30) * 3
    kw = dict(enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy', opt='momentum', learning_rate=0.05,
              momentum=0.5, alpha=1.0)
    cap = max(b[0].nnz for b in batches)
    orc = OracleDAE(W0, triplet_strategy='none', dtype=torch.float64, **kw)
    eng = _engine(F, H, 'none', W0, opt='momentum', lr=0.05)
    feeds = _feeds(batches, cap)
    outs = [eng.run_feed(f) for f in feeds[:3]] + eng.run_feeds(feeds[3:])
    for s, (st, b) in enumerate(zip(outs, batches)):
        want, _ = _oracle_step(orc, 'none', *b)
        _check_scalars(st, want, s)
    _check_params(eng, orc, 'none, no labels')
    for strategy in ('batch_all', 'batch_hard'):
        eng = _engine(F, H, strategy, W0, opt='momentum', lr=0.05)
        with pytest.raises(ValueError, match='labels'):
            eng.run_feed(feeds[0])
        with pytest.raises(ValueError, match='labels'):
            eng.run_feeds(feeds[:3])
        assert eng._feed_graph is None and eng._feed_stream is None and eng.step_count == 0
        x, xc, _ = batches[0]
        lb = np.arange(B, dtype=np.float32) % 4
        orc = OracleDAE(W0, triplet_strategy=strategy, dtype=torch.float64, **kw)
        want, _ = _oracle_step(orc, strategy, x, xc, lb)
        _check_scalars(eng.run_feeds(_feeds([(x, xc, lb)], cap))[0], want, strategy)
        _check_params(eng, orc, strategy)
