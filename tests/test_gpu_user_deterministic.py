"""The user encoders' deterministic mode on the GPU (DESIGN 4.21): the *_det loss kernels against the default instances and fp64,
dae_loss_slots_sum and dae_ordered_rows against their NumPy restatements, whole seeded fits bit for bit in one process and across
processes, one batch's gradients against the fp64 oracles, the GRU learning check, the default mode's launches and the CLI."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import user_deterministic_oracle as do  # noqa: E402
from helpers import rel_err  # noqa: E402

from dae_rnn_news_recommendation_b200 import _cabi, article_encoder, user_model  # noqa: E402
from dae_rnn_news_recommendation_b200._cabi import call  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import UserAttention, UserGRU, UserLSTM  # noqa: E402

D = torch.device('cuda:0')
CELLS = {'gru': UserGRU, 'lstm': UserLSTM, 'attention': UserAttention}
REL_TOL = 1e-5


def _st():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(D)


def _impressions(rng, P, N, per_pos=2, m=(2, 9)):
    from test_gpu_user_articles import _impressions as imp
    return imp(rng, P, N, per_pos, m)


# ---------------------------------------------------------------------------------------------------------------------------
# the loss kernels
# ---------------------------------------------------------------------------------------------------------------------------
def _loss_case(kind, H=37):
    rng = np.random.default_rng(len(kind) + H)
    P, N = 300, 40
    h, emb = rng.normal(0, .5, (P, H)).astype(np.float32), rng.normal(0, .5, (N, H)).astype(np.float32)
    if kind == 'rank':
        pos = rng.integers(0, N, P).astype(np.int32)
        pos[::7] = -1
        neg = ((pos + 1 + rng.integers(0, N - 1, P)) % N).astype(np.int32)
        neg[pos < 0] = -1
        return h, emb, (pos, neg)
    pos_indptr, indptr, items, clicked = _impressions(rng, P, N)
    clicked[indptr[3]:indptr[4]] = 1   # one impression without a non-click: its triples add nothing
    ids = np.arange(indptr.size - 1, dtype=np.int64) * 7 + 3
    return h, emb, (pos_indptr, indptr, items, clicked, ids)


def _run_loss(kind, h, emb, data, det, grad, K=2):
    """dh, the loss (stats[0] after the slot sum in the mode), the slots and the triples / demb of one call."""
    P, H = h.shape
    N = emb.shape[0]
    a = [_dev(x) for x in (h, emb) + tuple(data)]
    dh = torch.empty(P, H, device=D)
    stats = torch.zeros(1, dtype=torch.float64, device=D)
    slots = torch.full((P,), np.nan, dtype=torch.float64, device=D)
    n_trip = 2 * P if kind == 'rank' else int(data[2].size)
    trip = (torch.full((n_trip,), -7, dtype=torch.int32, device=D), torch.empty(n_trip, dtype=torch.int32, device=D),
            torch.empty(n_trip, dtype=torch.float32, device=D))
    demb = torch.zeros(N, H, device=D)
    out = slots if det else stats
    extra = ()
    if grad:
        extra = tuple(t.data_ptr() for t in trip) if det else (demb.data_ptr(), H)
    sfx = ('_grad' if grad else '') + ('_det' if det else '')
    if kind == 'rank':
        call('dae_seq_rank_loss' + sfx, a[0].data_ptr(), H, a[1].data_ptr(), H, H, a[2].data_ptr(), a[3].data_ptr(), P, 0.01,
             dh.data_ptr(), H, out.data_ptr(), *extra, _st())
    else:
        head = (a[0].data_ptr(), H, a[1].data_ptr(), H, H, a[2].data_ptr(), P, a[3].data_ptr(), a[4].data_ptr(), a[5].data_ptr())
        if kind == 'pairwise':
            call('dae_impression_rank_loss' + sfx, *head, 0.5, dh.data_ptr(), H, out.data_ptr(), *extra, _st())
        else:
            ws = torch.empty(2 * data[2].size, dtype=torch.int32, device=D)
            call('dae_impression_softmax_loss' + sfx, *head, a[6].data_ptr(), K, 5, 1, 0.5, dh.data_ptr(), H, out.data_ptr(),
                 ws.data_ptr(), *extra, _st())
    if det:
        call('dae_loss_slots_sum', slots.data_ptr(), P, stats.data_ptr(), _st())
    torch.cuda.synchronize()
    return dh, float(stats), slots.cpu().numpy(), tuple(t.cpu().numpy() for t in trip), demb


LOSS_KINDS = ['rank', 'pairwise', 'softmax0', 'softmax2']


@pytest.mark.parametrize('grad', [False, True])
@pytest.mark.parametrize('kind', LOSS_KINDS)
def test_det_loss_kernels(kind, grad):
    K = 0 if kind == 'softmax0' else 2
    base = 'softmax' if kind.startswith('softmax') else kind
    h, emb, data = _loss_case(kind)
    dh0, loss0, _, _, demb0 = _run_loss(base, h, emb, data, False, grad, K)
    dh1, loss1, slots, trip, _ = _run_loss(base, h, emb, data, True, grad, K)
    assert torch.equal(dh0, dh1)                                       # the flag does not touch dh's arithmetic
    if base == 'rank':
        want = do.rank_loss_slots(h, emb, *data)
    else:
        want = do.impression_loss_slots(h, emb, *data[:4], base, ids=data[4], K=K, seed=5, epoch=1)
    assert np.abs(slots - want).max() <= 1e-5 * max(1.0, np.abs(want).max())
    assert loss1 == do.slot_sum(slots)                                 # the stated order, bit for bit
    assert loss1 == pytest.approx(loss0, rel=1e-12)
    again = _run_loss(base, h, emb, data, True, grad, K)
    assert np.array_equal(again[2], slots) and again[1] == loss1
    if grad:
        t_slot, t_row, t_coef = trip
        assert (t_slot != -7).all()                                    # every triple is written
        n_slots = emb.shape[0]
        got = torch.empty(n_slots, h.shape[1], device=D)
        _ordered(trip, _dev(h), None, n_slots, got)
        mine = do.ordered_rows(t_slot, t_row, t_coef, h, [], h[:0], n_slots)
        assert np.array_equal(got.cpu().numpy(), mine)
        assert rel_err(got.cpu().numpy(), demb0.cpu().numpy()) < REL_TOL


# ---------------------------------------------------------------------------------------------------------------------------
# dae_ordered_rows
# ---------------------------------------------------------------------------------------------------------------------------
def _ordered(trip, src_a, b, n_slots, dst):
    """dst = dae_ordered_rows of the triples over src_a and the implicit (b_slot[p], p, 1) over src_b (b = (b_slot, src_b))."""
    t_slot, t_row, t_coef = (x if isinstance(x, torch.Tensor) else _dev(x) for x in trip)
    n_a = t_slot.numel()
    b_slot, src_b = (None, None) if b is None else b
    n_b = 0 if b is None else b_slot.numel()
    nb = _cabi.query('dae_ordered_rows_workspace', n_a, n_b, n_slots)
    assert nb >= 16 * (n_a + n_b)
    ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=D)
    call('dae_ordered_rows', t_slot.data_ptr(), t_row.data_ptr(), t_coef.data_ptr(), n_a, src_a.data_ptr() if n_a else None,
         src_a.stride(0) if n_a else 0, None if b is None else b_slot.data_ptr(), n_b, None if b is None else src_b.data_ptr(),
         0 if b is None else src_b.stride(0), n_slots, dst.shape[1], dst.data_ptr(), dst.stride(0), ws.data_ptr(), ws.numel(), _st())
    torch.cuda.synchronize()
    return dst


@pytest.mark.parametrize('cols', [1, 37, 129, 500])
def test_ordered_rows_against_restatement(cols):
    rng = np.random.default_rng(cols)
    n_a, n_b, n_slots, P = 3000, 700, 60, 900
    src_a = rng.normal(size=(P, cols)).astype(np.float32)
    src_b = rng.normal(size=(n_b, cols)).astype(np.float32)
    a_slot = rng.integers(-1, n_slots - 1, n_a).astype(np.int32)   # slot n_slots - 1 only from the dX rows below
    a_row = rng.integers(0, P, n_a).astype(np.int32)
    a_coef = rng.normal(size=n_a).astype(np.float32)
    b_slot = rng.integers(-1, n_slots, n_b).astype(np.int32)
    b_slot[:3] = n_slots - 1
    dst = torch.full((n_slots, cols + 3), np.nan, device=D)[:, :cols]
    got = _ordered((a_slot, a_row, a_coef), _dev(src_a), (_dev(b_slot), _dev(src_b)), n_slots, dst).cpu().numpy()
    assert np.array_equal(got, do.ordered_rows(a_slot, a_row, a_coef, src_a, b_slot, src_b, n_slots))
    exact = do.ordered_rows_fp64(a_slot, a_row, a_coef, src_a, b_slot, src_b, n_slots)
    assert rel_err(got, exact) < REL_TOL


def test_ordered_rows_zipf_is_run_to_run_identical():
    rng = np.random.default_rng(3)
    P, H, n_slots = 60000, 64, 40
    src = torch.randn(P, H, device=D)
    dX = torch.randn(P, H, device=D)
    slot = np.minimum(rng.zipf(1.3, 2 * P) - 1, n_slots - 1).astype(np.int32)    # thousands of terms on the first few slots
    coef = rng.normal(size=2 * P).astype(np.float32)
    row = np.repeat(np.arange(P), 2).astype(np.int32)
    b_slot = _dev(np.minimum(rng.zipf(1.3, P) - 1, n_slots - 1).astype(np.int32))
    assert np.bincount(slot)[0] > 10000
    outs = [_ordered((slot, row, coef), src, (b_slot, dX), n_slots, torch.empty(n_slots, H, device=D)) for _ in range(3)]
    assert all(torch.equal(outs[0], o) for o in outs[1:])
    want = do.ordered_rows_fp64(slot, row, coef, src.cpu().numpy(), b_slot.cpu().numpy(), dX.cpu().numpy(), n_slots)
    assert rel_err(outs[0].cpu().numpy(), want) < 1e-4   # tens of thousands of fp32 terms per row


def test_ordered_rows_edge_cases():
    H = 8
    src = torch.randn(4, H, device=D)
    # no terms at all: every row is stored as zero
    z = _ordered((np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32)), src, None, 3,
                 torch.full((3, H), 5.0, device=D))
    assert torch.equal(z, torch.zeros(3, H, device=D))
    # slot -1 adds nothing; an article that only appears as a negative (slot 2, never in the dX list) gets its loss terms alone
    trip = (np.array([-1, 2, 0, 2], np.int32), np.array([0, 1, 2, 3], np.int32), np.array([9.0, 0.5, 1.0, -2.0], np.float32))
    b = (_dev(np.array([0, -1, 1], np.int32)), torch.randn(3, H, device=D))
    got = _ordered(trip, src, b, 3, torch.empty(3, H, device=D)).cpu().numpy()
    s, x = src.cpu().numpy(), b[1].cpu().numpy()
    assert np.array_equal(got, do.ordered_rows(*trip, s, [0, -1, 1], x, 3))
    assert np.array_equal(got[1], x[2]) and np.array_equal(got[2], (np.float32(0.5) * s[1] + np.float32(-2.0) * s[3]))


def test_slot_sum_against_restatement():
    x = np.random.default_rng(0).standard_normal(100003) * 1e3
    out = torch.tensor([0.75], dtype=torch.float64, device=D)
    call('dae_loss_slots_sum', _dev(x).data_ptr(), x.size, out.data_ptr(), _st())
    call('dae_loss_slots_sum', _dev(x).data_ptr(), 0, out.data_ptr(), _st())       # no slots: adds +0
    assert float(out) == do.slot_sum(x, 0.75)


# ---------------------------------------------------------------------------------------------------------------------------
# whole runs
# ---------------------------------------------------------------------------------------------------------------------------
def _workload(seed=0, N=300, users=400):
    from test_gpu_user_articles import _workload as w
    return w(N, np.random.default_rng(seed), users=users)


def _article_encoder(N=300):
    from test_gpu_user_articles import _art
    art, _, _ = _art(N=N, F=150, H=32, act='tanh', seed=1, learning_rate=1e-2)
    return art


FIT_CASES = [(c, loss, arts, False) for c in CELLS for loss in ('negatives', 'pairwise', 'softmax') for arts in ('frozen', 'joint')]
FIT_CASES += [('gru', 'pairwise', 'joint', True), ('lstm', 'negatives', 'frozen', True), ('lstm', 'softmax', 'joint', True)]


def _case_id(c):
    return '-'.join(map(str, c[:3])) + ('-long_term' if c[3] else '')


def fit_case(cell, loss, arts, long_term, deterministic=True):
    """One seeded fit: everything the mode's contract lists, as NumPy arrays."""
    indptr, items, imp = _workload()
    kw = dict(max_len=6, batch_users=128, num_epochs=2, seed=3, learning_rate=1e-2, deterministic=deterministic,
              impression_loss='softmax' if loss == 'softmax' else 'pairwise', impression_negatives=2)
    if long_term:
        kw.update(long_term_users=len(indptr) - 1, long_term_mask=0.3)
    m = CELLS[cell](32, **kw)
    rng = np.random.default_rng(7)
    emb = rng.normal(0, .5, (300, 32)).astype(np.float32)
    a = _article_encoder() if arts == 'joint' else emb
    m.fit((indptr, items), a, impressions=None if loss == 'negatives' else imp)
    out = {'theta': m.theta, 'slot1': m.slot1, 'slot2': m.slot2, 'steps': np.array(m.steps), 'train_loss': np.array(m.train_loss),
           'transform': m.transform((indptr, items), a), 'states': m.impression_states((indptr, items), a, imp),
           'rec_index': m.recommend((indptr, items), a, k=5)[0], 'rec_score': m.recommend((indptr, items), a, k=5)[1]}
    if long_term:
        out.update(lt=m._lt, lt1=m._lt_slot1, lt2=m._lt_slot2, ltc=m._lt_count)
    if arts == 'joint':
        out.update(art_theta=a.theta, art1=a.slot1, art2=a.slot2, art_steps=np.array(a.steps))
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in out.items() if v is not None}


def _same(a, b):
    assert set(a) == set(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert a[k].tobytes() == b[k].tobytes(), k


@pytest.fixture(scope='module')
def other_process(tmp_path_factory):
    """Every FIT_CASE fitted once more in a fresh process, saved to .npz files."""
    d = tmp_path_factory.mktemp('det')
    code = ('import sys, json, numpy as np; sys.path[:0] = %r; import test_gpu_user_deterministic as t\n'
            'for c in t.FIT_CASES:\n'
            '    np.savez(%r + "/" + t._case_id(c) + ".npz", **t.fit_case(*c))\n' % ([ROOT, os.path.join(ROOT, 'tests')], str(d)))
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    return d


@pytest.mark.parametrize('case', FIT_CASES, ids=[_case_id(c) for c in FIT_CASES])
def test_fits_are_bit_identical(case, other_process):
    a, b = fit_case(*case), fit_case(*case)
    _same(a, b)
    z = np.load(other_process / (_case_id(case) + '.npz'))
    _same(a, {k: z[k] for k in z.files})


@pytest.mark.parametrize('cell', list(CELLS))
def test_default_mode_issues_no_det_export(cell, monkeypatch):
    names = []

    def rec(name, *args):
        names.append(name)
        return _cabi.call(name, *args)
    monkeypatch.setattr(user_model, 'call', rec)
    monkeypatch.setattr(article_encoder, 'call', rec)
    indptr, items, imp = _workload()
    for det in (False, True):
        names.clear()
        m = CELLS[cell](32, max_len=6, batch_users=128, num_epochs=1, seed=3, deterministic=det)
        m.fit((indptr, items), _article_encoder(), impressions=imp)
        m.fit((indptr, items), np.random.default_rng(0).normal(size=(300, 32)).astype(np.float32))
        new = {n for n in names if n.endswith('_det') or n in ('dae_loss_slots_sum', 'dae_ordered_rows')}
        if det:
            assert {'dae_gemm_bf16x3_det', 'dae_loss_slots_sum', 'dae_ordered_rows', 'dae_encode_csr_bwd_det'} <= new
            assert 'dae_rows_scatter_add' not in names and 'dae_encode_csr_bwd_gather' not in names
        else:
            assert not new and 'dae_rows_scatter_add' in names


# ---------------------------------------------------------------------------------------------------------------------------
# accuracy of one deterministic batch
# ---------------------------------------------------------------------------------------------------------------------------
ACC_CASES = [(c, k, 37) for c in CELLS for k in ('random', 'pairwise', 'softmax')] + [('gru', 'random', 'long_term'),
                                                                                       ('lstm', 'pairwise', 'long_term')]


@pytest.mark.parametrize('cell,kind,H', ACC_CASES)
def test_joint_batch_against_oracle(cell, kind, H, monkeypatch):
    """test_gpu_user_articles' one-batch check against the fp64 joint oracle (which builds on the GRU / LSTM / attention,
    impression, softmax and long-term oracles), with deterministic=True, and the gradients against the default mode's."""
    import test_gpu_user_articles as ua
    for name in CELLS:
        monkeypatch.setitem(ua.CELLS, name, functools.partial(CELLS[name], deterministic=True))
    ua.test_joint_batch_against_oracle(cell, kind, H)
    g = {}
    for det in (True, False):
        indptr, items, imp = _workload(seed=1, N=80, users=24)
        lt = dict(long_term_users=len(indptr) - 1, long_term_mask=0.0) if H == 'long_term' else {}
        m = CELLS[cell](32, max_len=6, batch_users=4096, num_epochs=1, seed=2, learning_rate=0.0,
                        impression_loss='softmax' if kind == 'softmax' else 'pairwise', impression_negatives=2, deterministic=det, **lt)
        art = _article_encoder(80)
        art.learning_rate = 0.0
        m.fit((indptr, items), art, impressions=None if kind == 'random' else imp)
        g[det] = (m.grad.cpu().numpy(), art.grad.cpu().numpy(), m.article_batch['dE'].cpu().numpy())
    for a, b in zip(g[True], g[False]):
        assert rel_err(a, b) < 2e-4


def test_gru_learning_check_deterministic(monkeypatch):
    import test_gpu_user_gru as tg
    monkeypatch.setattr(tg, 'UserGRU', functools.partial(UserGRU, deterministic=True))
    gru, mean, losses = tg._learning_numbers()
    print('deterministic hit@10: GRU %.4f, mean profile %.4f' % (gru, mean))
    assert losses[-1] < losses[0]
    assert gru - mean > tg.LEARNING_MARGIN, (gru, mean)


# ---------------------------------------------------------------------------------------------------------------------------
# the CLI
# ---------------------------------------------------------------------------------------------------------------------------
def test_cli_user_deterministic_runs_repeat(tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.synth import make_sequences
    base = ['--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200', '--seed', '3', '--top_k', '5',
            '--deterministic']
    _, _, trL, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(['--model_name', 'x'] + base)))
    indptr, items, targets = make_sequences(300, trL, mean_len=8, seed=4)
    np.savez(tmp_path / 's.npz', indptr=indptr, items=items, targets=targets)
    dirs = []
    for run in ('a', 'b'):
        model = cli.main(['--model_name', 'det_' + run] + base + ['--user_sequences', str(tmp_path / 's.npz'), '--user_epochs', '2',
                                                                  '--user_deterministic', '--user_fine_tune_articles'])
        dirs.append(model.data_dir)
    for f in ('user_gru.npz', 'user_gru_top_k_index.npy', 'user_gru_top_k_score.npy', 'user_gru_article_encoder.npz'):
        a, b = (np.load(d + f) for d in dirs)
        if f.endswith('.npz'):
            _same({k: a[k] for k in a.files}, {k: b[k] for k in b.files})
        else:
            assert a.tobytes() == b.tobytes(), f
