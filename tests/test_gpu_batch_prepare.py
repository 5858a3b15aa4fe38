"""The batch preparation (dae_batch_prepare[_blocked], dae_batch_prepare_next[_blocked], dae_batch_commit) and the masking noise
(dae_mask_values) through the C ABI, every output bit for bit against the exact NumPy references of tests/batch_prepare_oracle.py.

The sizes cover the three sort paths and their edges: the register bitonic sort (B <= 1024; partners exchange by warp shuffle below
stride 32 and through shared memory above, so P = 32 / 64 on both sides of the switch), the shared-memory sort (B <= 4096) and the
global-memory sort inside the caller's buffers (B > 4096, up to DAE_MAX_BLOCKED_BATCH = 262 144 through the _blocked exports).  Every
output starts as a sentinel and has guard entries past B; the stats start non-zero and have two guard slots past the 16."""
import numpy as np
import pytest
import torch

import batch_prepare_oracle as bo
from helpers import REL_TOL, rel_err, random_csr, mask_csr, xavier

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GUARD = 5
F_SENT = 0x7fa5a5a5          # a NaN payload no kernel writes
I_SENT = -77
ST_SENT = 5.0
NAMES = ('rows', 'labels', 'lo', 'hi', 'w', 'stats')

REGISTER_B = [1, 2, 3, 31, 32, 33, 63, 64, 65, 511, 800, 1023, 1024]
SHARED_B = [1025, 2047, 2048, 2049, 4095, 4096]
GLOBAL_B = [4097, 8191, 8192, 8193, 32769, 131073, 262143, 262144]


def _call(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call(name, *args)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _exports(B):
    """(prepare, prepare_next): the plain exports up to DAE_MAX_TRIPLET_BATCH, the _blocked ones above."""
    return ('dae_batch_prepare', 'dae_batch_prepare_next') if B <= 32768 else \
        ('dae_batch_prepare_blocked', 'dae_batch_prepare_next_blocked')


class Out:
    """The six outputs of one batch, each with GUARD sentinel entries past B (stats: 16 slots + 2 guards); `null` names stay NULL."""

    def __init__(self, B, null=()):
        i32 = dict(dtype=torch.int32, device=DEV)
        self.B, self.null = B, set(null)
        self.t = {
            'rows': torch.full((B + GUARD,), I_SENT, **i32),
            'labels': torch.full((B + GUARD,), F_SENT, **i32).view(torch.float32),
            'lo': torch.full((B + GUARD,), I_SENT, **i32),
            'hi': torch.full((B + GUARD,), I_SENT, **i32),
            'w': torch.full((B + GUARD,), F_SENT, **i32).view(torch.float32),
            'stats': torch.full((bo.STAT_SLOTS + 2,), ST_SENT, dtype=torch.float64, device=DEV),
        }
        for n in self.null:
            self.t[n] = None

    def ptrs(self):
        return [_ptr(self.t[n]) for n in NAMES]

    def host(self):
        torch.cuda.synchronize()
        return {n: (None if v is None else v.cpu().numpy()) for n, v in self.t.items()}


def _bits(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _check(out, want, what=''):
    """out's first B entries equal `want` (the oracle's six arrays) bit for bit; the guards and the stats' two extra slots are intact."""
    h, B = out.host(), out.B
    for n, e in zip(NAMES, want):
        g = h[n]
        if g is None:
            continue
        if n == 'stats':
            assert np.array_equal(g[:bo.STAT_SLOTS], e), (what, n, g[:bo.STAT_SLOTS], e)
            assert (g[bo.STAT_SLOTS:] == ST_SENT).all(), (what, 'stats guard')
            continue
        eb, gb = _bits(e), _bits(g[:B])
        bad = np.flatnonzero(gb != eb)
        assert bad.size == 0, (what, n, B, bad[:8], g[bad[:8]], np.asarray(e)[bad[:8]])
        sent = F_SENT if g.dtype == np.float32 else I_SENT
        assert (_bits(g[B:]).astype(np.int64) == sent).all(), (what, n, 'guard')


def _untouched(out):
    h = out.host()
    for n in NAMES:
        if h[n] is None:
            continue
        if n == 'stats':
            assert (h[n] == ST_SENT).all()
        else:
            assert (_bits(h[n]).astype(np.int64) == (F_SENT if h[n].dtype == np.float32 else I_SENT)).all(), n


def _problem(B, kind, offset=17, extra=37, seed=0):
    """perm of n_all = offset + B + extra rows, the batch perm[offset : offset + B] labelled by kind, every other row NaN."""
    n_all = offset + B + extra
    perm = np.random.default_rng(B + seed).permutation(n_all).astype(np.int32)
    labels_all = bo.scatter_labels(n_all, perm, offset, bo.batch_labels(B, kind, seed=B + seed + 1))
    return perm, labels_all


def _run_sizes(B, kinds=bo.LABEL_KINDS):
    prep = _exports(B)[0]
    for kind in kinds:
        perm, labels_all = _problem(B, kind)
        perm_d, lab_d = _t(perm), _t(labels_all)
        for strategy in (bo.STRATEGY_BATCH_ALL, bo.STRATEGY_BATCH_HARD):
            want = bo.prepare(perm, 17, B, labels_all, strategy)
            outs = [Out(B), Out(B)]
            for o in outs:
                _call(prep, _ptr(perm_d), 17, None, B, _ptr(lab_d), strategy, *o.ptrs(), _st())
            _check(outs[0], want, (kind, strategy))
            for n in NAMES:                         # run to run: the same bits, guards included
                assert torch.equal(outs[0].t[n].view(torch.int32) if n in ('labels', 'w') else outs[0].t[n],
                                   outs[1].t[n].view(torch.int32) if n in ('labels', 'w') else outs[1].t[n]), (kind, strategy, n)


@pytest.mark.parametrize('B', REGISTER_B)
def test_register_sort_path(B):
    _run_sizes(B)


@pytest.mark.parametrize('B', SHARED_B)
def test_shared_memory_sort_path(B):
    _run_sizes(B)


@pytest.mark.parametrize('B', GLOBAL_B)
def test_global_memory_sort_path(B):
    _run_sizes(B)


@pytest.mark.parametrize('B', [1, 800, 4097, 10 ** 6])
def test_strategy_none(B):
    """batch_rows_kernel: the permutation order, labels 0, one segment [0, B), w = 1, SUM_W = B -- any B; optional outputs NULL."""
    perm, labels_all = _problem(B, 'nanmany')
    perm_d, lab_d = _t(perm), _t(labels_all)
    want = bo.prepare(perm, 17, B, labels_all, bo.STRATEGY_NONE)
    o = Out(B)
    _call('dae_batch_prepare', _ptr(perm_d), 17, None, B, _ptr(lab_d), bo.STRATEGY_NONE, *o.ptrs(), _st())
    _check(o, want, 'none')
    o = Out(B, null=('labels', 'lo', 'hi', 'w'))
    _call('dae_batch_prepare_blocked', None, 17, None, B, None, bo.STRATEGY_NONE, *o.ptrs(), _st())
    _check(o, bo.prepare(None, 17, B, None, bo.STRATEGY_NONE), 'none, NULL perm and outputs')


@pytest.mark.parametrize('B', [800, 3000, 9000])
def test_null_perm_and_optional_outputs(B):
    """perm NULL reads rows offset .. offset + B - 1; weight_out may be NULL on every path, labels_out up to 4096 rows (above, the
    batch is sorted inside it and a NULL is refused before any launch)."""
    from dae_rnn_news_recommendation_b200 import _cabi
    perm, labels_all = _problem(B, 'nanmany', seed=3)
    lab_d = _t(labels_all)
    for strategy in (bo.STRATEGY_BATCH_ALL, bo.STRATEGY_BATCH_HARD):
        want = bo.prepare(None, 29, B, labels_all, strategy)
        null = ('w', 'labels') if B <= 4096 else ('w',)
        o = Out(B, null=null)
        _call('dae_batch_prepare', None, 29, None, B, _ptr(lab_d), strategy, *o.ptrs(), _st())
        _check(o, want, ('identity', strategy, null))
        if B > 4096:
            o = Out(B, null=('labels',))
            with pytest.raises(_cabi.DaeError, match='labels_out'):
                _call('dae_batch_prepare', None, 29, None, B, _ptr(lab_d), strategy, *o.ptrs(), _st())
            _untouched(o)


@pytest.mark.parametrize('B', [800, 3000, 9000, 40000])
def test_device_cursor_and_staging_bounds(B):
    """offset + ctl[0] selects the batch; dae_batch_prepare_next stages the batch at ctl[0] + stride, writes when it ends exactly at
    n_perm and writes nothing (every sentinel intact) when it would end one row past it."""
    prep, nxt = _exports(B)
    perm, labels_all = _problem(B, 'nanmany', offset=0, extra=600, seed=5)
    n_all = perm.shape[0]
    perm_d, lab_d = _t(perm), _t(labels_all)
    ctl = torch.tensor([211, 0, 1, 0], dtype=torch.int64, device=DEV)
    o = Out(B)
    _call(prep, _ptr(perm_d), 40, _ptr(ctl), B, _ptr(lab_d), 1, *o.ptrs(), _st())
    _check(o, bo.prepare(perm, 251, B, labels_all, 1), 'offset + ctl[0]')
    stride = 300
    ctl[0] = n_all - B - stride                       # ctl[0] + stride + B == n_perm: the last batch of the epoch
    o = Out(B)
    _call(nxt, _ptr(perm_d), n_all, stride, _ptr(ctl), B, _ptr(lab_d), 2, *o.ptrs(), _st())
    _check(o, bo.prepare(perm, n_all - B, B, labels_all, 2), 'next at the end')
    ctl[0] = n_all - B - stride + 1                   # one row past the end: nothing is written
    o = Out(B)
    _call(nxt, _ptr(perm_d), n_all, stride, _ptr(ctl), B, _ptr(lab_d), 1, *o.ptrs(), _st())
    _untouched(o)
    assert ctl.tolist() == [n_all - B - stride + 1, 0, 1, 0]


@pytest.mark.parametrize('B', [800, 3000, 9000, 40000])
def test_staged_then_committed_equals_eager(B):
    """dae_batch_prepare_next + dae_batch_commit leaves the live buffers equal, bit for bit, to dae_batch_prepare at the same cursor."""
    prep, nxt = _exports(B)
    perm, labels_all = _problem(B, 'c300', offset=0, extra=1000, seed=7)
    labels_all[perm[500:500 + B:97]] = np.nan                 # a few NaN rows in the batch
    perm_d, lab_d = _t(perm), _t(labels_all)
    for strategy in (bo.STRATEGY_BATCH_ALL, bo.STRATEGY_BATCH_HARD):
        ctl = torch.tensor([200, 0, 1, 0], dtype=torch.int64, device=DEV)
        stage, live, eager = Out(B), Out(B), Out(B)
        _call(nxt, _ptr(perm_d), perm.shape[0], 300, _ptr(ctl), B, _ptr(lab_d), strategy, *stage.ptrs(), _st())
        _call('dae_batch_commit', B, *stage.ptrs(), *live.ptrs(), _st())
        _call(prep, _ptr(perm_d), 300, _ptr(ctl), B, _ptr(lab_d), strategy, *eager.ptrs(), _st())
        want = bo.prepare(perm, 500, B, labels_all, strategy)
        for o, what in ((stage, 'staged'), (live, 'committed'), (eager, 'eager')):
            _check(o, want, (what, strategy))


@pytest.mark.parametrize('strategy', ['batch_all', 'batch_hard'])
def test_engine_step_with_nan_labels(strategy):
    """A B = 800 training step whose batch holds NaN labels against OracleDAE, where (as with the reference's tf.equal) a NaN row is
    a class of one: it has no positive and is a negative of every other row."""
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from oracle.dae_oracle import OracleDAE
    F, H, B = 400, 32, 800
    x = random_csr(B, F, 12, kind='binary', seed=61)
    xc, _ = mask_csr(x, 0.3, seed=62)
    labels = np.random.default_rng(63).integers(0, 4, B).astype(np.float32)
    labels[[3, 250, 251, 799]] = np.nan
    W0 = xavier(F, H, 64) * 3.0
    kw = dict(enc_act_func='sigmoid', dec_act_func='sigmoid', loss_func='cross_entropy', opt='gradient_descent', learning_rate=0.05,
              alpha=1.0, triplet_strategy=strategy)
    eng = TrainEngine(F, H, device=DEV, **kw)
    eng.set_parameters(W0)
    eng.set_data(DeviceCSR(x, eng.device), _t(xc.data.astype(np.float32)), _t(labels))
    eng.step(None, 0, B)
    torch.cuda.synchronize()
    st = eng.read_stats()
    o = OracleDAE(W0, **kw).step(x, xc, labels)
    assert rel_err(st['cost'], o['cost']) < REL_TOL, (st['cost'], o['cost'])
    assert rel_err(st['ae_loss'], o['autoencoder_loss']) < REL_TOL
    assert rel_err(st['triplet_loss'], o['triplet_loss']) < REL_TOL
    assert st['num'] == pytest.approx(float(o['num']), rel=1e-3, abs=2.0)
    g = eng.grad.cpu().numpy()
    gW, gbh, gbv = o['grads']
    assert rel_err(g[:F * H].reshape(F, H), gW) < REL_TOL
    assert rel_err(g[F * H:F * H + H], gbh) < REL_TOL
    assert rel_err(g[F * H + H:], gbv) < REL_TOL
    rows = eng.rows.cpu().numpy()[:B]
    assert np.array_equal(np.sort(rows), np.arange(B))        # every row of the batch trained, each once


# ---------------------------------------------------------------------------------------------------------------------------------
# masking noise
# ---------------------------------------------------------------------------------------------------------------------------------
SEED, EPOCH = (0x9E3779B9 << 32) | 0x2545F491, (3 << 32) | 5        # both high words non-zero


def _values(nnz, seed=0):
    rng = np.random.default_rng(seed)
    v = rng.normal(0.0, 2.0, nnz).astype(np.float32)
    if nnz:
        idx = rng.permutation(nnz)
        v[idx[0::7]] = -0.0
        v[idx[1::11]] = np.uint32(0xffc0beef).view(np.float32)     # a negative NaN with a payload
        v[idx[2::13]] = 0.0
    return v


def _mask(values, keep, frac, seed, epoch):
    nnz = values.shape[0]
    out = torch.full((nnz + GUARD,), F_SENT, dtype=torch.int32, device=DEV).view(torch.float32)
    v_d = _t(values) if nnz else torch.zeros(1, device=DEV)
    k_d = None if keep is None else (_t(keep) if nnz else torch.zeros(1, dtype=torch.uint8, device=DEV))
    _call('dae_mask_values', v_d.data_ptr(), _ptr(k_d), nnz, float(frac), seed, epoch, out.data_ptr(), _st())
    torch.cuda.synchronize()
    got = out.view(torch.int32).cpu().numpy().view(np.uint32)
    assert (got[nnz:] == F_SENT).all(), 'guard'
    return got[:nnz]


def _three_passes():
    """One more quad than three passes of the grid (sm_count * 16 CTAs of 256 threads, one quad of 4 entries per thread)."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return 3 * sm * 16 * 256 * 4 + 7


@pytest.mark.parametrize('nnz', [0, 1, 3, 4, 5, 1003, 'passes'])
def test_mask_values_philox(nnz):
    nnz = _three_passes() if nnz == 'passes' else nnz
    vals = _values(nnz, seed=nnz)
    fracs = [0.0, 1.0, 0.5, 0.3]
    if nnz:
        u = bo.mask_uniforms(nnz, SEED, EPOCH)
        fracs.append(float(u[nnz // 2]))             # some u exactly: that entry is kept (u >= corr_frac)
    for frac in fracs:
        for seed, epoch in ((SEED, EPOCH), (7, 0)):
            want = bo.mask_values(vals, None, frac, seed, epoch).view(np.uint32)
            got = _mask(vals, None, frac, seed, epoch)
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, (nnz, frac, seed, epoch, bad[:8])
    if nnz:
        assert got.shape == (nnz,)


def test_mask_values_exact_threshold_entries_are_kept():
    """corr_frac equal to the draws of many entries: all of them are kept, so `>` in place of `>=` would drop each."""
    nnz = 40000
    vals = np.arange(1, nnz + 1, dtype=np.float32)
    u = bo.mask_uniforms(nnz, SEED, EPOCH)
    for p in (5, 123, 39999):
        got = _mask(vals, None, u[p], SEED, EPOCH).view(np.float32)
        assert got[p] == vals[p]
        assert np.array_equal(got.view(np.uint32), bo.mask_values(vals, None, u[p], SEED, EPOCH).view(np.uint32))


@pytest.mark.parametrize('nnz', [1, 5, 1003, 'passes'])
def test_mask_values_host_mask(nnz):
    """keep bytes 0, 1 and 255: kept iff non-zero, whatever corr_frac says."""
    nnz = _three_passes() if nnz == 'passes' else nnz
    vals = _values(nnz, seed=nnz + 1)
    keep = np.random.default_rng(nnz).choice(np.array([0, 1, 255], np.uint8), nnz)
    for frac in (0.0, 1.0):
        got = _mask(vals, keep, frac, SEED, EPOCH)
        assert np.array_equal(got, bo.mask_values(vals, keep, frac).view(np.uint32))


def test_mask_values_zero_nnz_writes_nothing():
    got = _mask(np.zeros(0, np.float32), None, 0.3, SEED, EPOCH)
    assert got.shape == (0,)
