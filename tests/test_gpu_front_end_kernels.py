"""The kernels around the dense similarity GEMM (dae_rownorm_split_bf16, dae_row_argmax), nearest_neighbors' diagonal rule, and
the training step's plumbing exports (dae_step_advance, dae_batch_commit, dae_batch_prepare_explicit, dae_col_scan) through the
C ABI, against tests/gru_kernel_oracle.py and the contracts in include/dae_sm100.h.  Outputs start as sentinels."""
import numpy as np
import pytest
import torch

import gru_kernel_oracle as go

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF16_SENT = 0x7F7F
f32 = np.float32


def _call(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call(name, *args)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _np(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _bits(t):
    torch.cuda.synchronize()
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


# ---------------------------------------------------------------------------------------------------------------------------
# dae_rownorm_split_bf16
# ---------------------------------------------------------------------------------------------------------------------------
def _rows(rng, rows, cols):
    X = (rng.standard_normal((rows, cols)) * rng.choice([1e-6, 1.0, 1e6], (rows, 1))).astype(f32)
    X[0] = 0                                        # untouched
    X[1] = 0
    X[1, cols // 2] = -3.5                          # one non-zero entry
    X[2] = np.abs(X[2])
    return X


@pytest.mark.parametrize('cols', [1, 31, 32, 33, 500, 4097])
@pytest.mark.parametrize('kind', [0, 1, 2, 3])
def test_rownorm_split(kind, cols):
    rng = np.random.default_rng(kind * 10000 + cols)
    rows = 203                                      # not a multiple of 8 (one warp per row, 8 per CTA)
    X = _rows(rng, rows, cols)
    ld, ld_dst, ld_out = cols + 3, (cols + 7) // 8 * 8 + 8, cols + 5
    Xp = np.full((rows, ld), -7.0, f32)
    Xp[:, :cols] = X
    X_d = _dev(Xp)
    want, s = go.rownorm(X, kind)
    for mode in ('x_out', 'hi', 'both'):
        hi = torch.full((rows + 1, ld_dst), BF16_SENT, dtype=torch.int16, device=DEV)
        lo = torch.full_like(hi, BF16_SENT)
        xo = torch.full((rows + 1, ld_out), float('nan'), dtype=torch.float32, device=DEV)
        split, out = mode != 'x_out', mode != 'hi'
        _call('dae_rownorm_split_bf16', X_d.data_ptr(), rows, cols, ld, kind, hi.data_ptr() if split else None,
              lo.data_ptr() if split else None, ld_dst, xo.data_ptr() if out else None, ld_out, _st())
        g_hi, g_lo, g = _bits(hi), _bits(lo), _np(xo)
        tag = 'rownorm kind=%d cols=%d %s' % (kind, cols, mode)
        if out:
            go.check(tag, g[:rows, :cols], want, s, go.C_FP32)
            assert (g[0, :cols] == 0).all()
            assert np.isnan(g[:rows, cols:]).all() and np.isnan(g[rows:]).all()
        else:
            assert np.isnan(g).all()
        if split:
            if out:
                w_hi, w_lo = go.bf16_split(g[:rows, :cols])
                assert np.array_equal(g_hi[:rows, :cols], w_hi) and np.array_equal(g_lo[:rows, :cols], w_lo), tag
            else:
                go.check_pair(tag, g_hi[:rows, :cols], g_lo[:rows, :cols], want, s, go.C_FP32)
            assert (g_hi[:rows, cols:] == 0).all() and (g_lo[:rows, cols:] == 0).all(), tag    # padding exactly 0
            assert (g_hi[rows:] == BF16_SENT).all() and (g_lo[rows:] == BF16_SENT).all()
        else:
            assert (g_hi == BF16_SENT).all() and (g_lo == BF16_SENT).all()


# ---------------------------------------------------------------------------------------------------------------------------
# dae_row_argmax
# ---------------------------------------------------------------------------------------------------------------------------
def _scores(rng, rows, cols):
    S = rng.integers(-3, 4, (rows, cols)).astype(f32)      # small integers: ties within a lane and across lanes
    S[rng.random(S.shape) < 0.1] = np.nan
    S[0] = -np.inf                                          # every candidate -inf: the first one wins
    S[1] = np.nan                                           # no candidate
    if rows > 2:
        S[2] = -np.abs(S[2]) - 1                            # every score negative
    if rows > 3:
        S[3] = np.nan
        S[3, cols - 1] = -np.inf
    return S


@pytest.mark.parametrize('cols', [1, 2, 33, 1000])
def test_row_argmax(cols):
    rng = np.random.default_rng(cols)
    rows = 37
    ld = cols + 3
    S = _scores(rng, rows, cols)
    for off in (0, 16, -5, cols, cols + 7):
        w_idx, w_val = go.row_argmax(S, off)
        for zero_diag in (0, 1):
            for outs in ('both', 'idx', 'val'):
                Sp = np.full((rows, ld), -7.0, f32)
                Sp[:, :cols] = S
                S_d = _dev(Sp)
                idx = torch.full((rows + 1,), -7, dtype=torch.int32, device=DEV)
                val = torch.full((rows + 1,), 1234.5, dtype=torch.float32, device=DEV)
                _call('dae_row_argmax', S_d.data_ptr(), rows, cols, ld, off, zero_diag, idx.data_ptr() if outs != 'val' else None,
                      val.data_ptr() if outs != 'idx' else None, _st())
                gi, gv = _np(idx), _np(val)
                tag = 'cols=%d off=%d zero=%d %s' % (cols, off, zero_diag, outs)
                if outs != 'val':
                    assert np.array_equal(gi[:rows], w_idx), (tag, np.flatnonzero(gi[:rows] != w_idx)[:5])
                else:
                    assert (gi == -7).all()
                if outs != 'idx':
                    assert np.array_equal(gv[:rows].view(np.uint32), w_val.view(np.uint32)), tag     # bit for bit, -inf included
                else:
                    assert (gv == 1234.5).all()
                assert gi[rows] == -7 and gv[rows] == 1234.5
                after = _np(S_d)
                expect = Sp.copy()
                if zero_diag:
                    r = np.arange(rows)
                    d = r + off
                    ok = (d >= 0) & (d < cols)
                    expect[r[ok], d[ok]] = 0.0
                assert np.array_equal(after.view(np.uint32), expect.view(np.uint32)), tag


def test_row_argmax_no_candidate_and_all_minus_inf():
    """Rows whose candidates are all -inf return the first of them; a row without a candidate returns -1 / -inf."""
    S = np.array([[-np.inf, -np.inf, -np.inf], [np.nan, -np.inf, np.nan], [np.nan, np.nan, np.nan]], f32)
    S_d = _dev(S)
    idx = torch.full((3,), -7, dtype=torch.int32, device=DEV)
    val = torch.zeros(3, dtype=torch.float32, device=DEV)
    _call('dae_row_argmax', S_d.data_ptr(), 3, 3, 3, 0, 0, idx.data_ptr(), val.data_ptr(), _st())
    assert _np(idx).tolist() == [1, -1, -1]
    assert np.isneginf(_np(val)).all()
    one = _dev(np.array([[0.5]], f32))
    _call('dae_row_argmax', one.data_ptr(), 1, 1, 1, 0, 0, idx.data_ptr(), val.data_ptr(), _st())
    assert _np(idx)[0] == -1 and np.isneginf(_np(val)[0])


def test_nearest_neighbors_never_returns_the_row_itself():
    """Row 0's similarities to every other row are negative: the best of them is returned, not row 0 with score 0."""
    from dae_rnn_news_recommendation_b200.helpers import nearest_neighbors, top_k_similar
    E = np.array([[1.0, 0.0], [-1.0, 0.3], [-1.0, -0.1], [-0.2, -1.0], [-1.0, 0.05]], f32)
    idx, val = nearest_neighbors(E, chunk=2)
    cos = (E / np.linalg.norm(E, axis=1, keepdims=True)) @ (E / np.linalg.norm(E, axis=1, keepdims=True)).T
    np.fill_diagonal(cos, -np.inf)
    assert idx[0] == 3 and idx[0] == np.argmax(cos[0]) and val[0] < 0
    assert (idx != np.arange(5)).all()
    np.testing.assert_allclose(val, cos.max(1), rtol=1e-4, atol=1e-4)     # the bf16x3 GEMM's accuracy
    ti, tv = top_k_similar(E, k=1)
    assert np.array_equal(ti[:, 0], idx)
    i1, v1 = nearest_neighbors(E[:1])
    assert i1[0] == -1 and np.isneginf(v1[0])


# ---------------------------------------------------------------------------------------------------------------------------
# step plumbing
# ---------------------------------------------------------------------------------------------------------------------------
def test_step_advance():
    ctl = _dev(np.array([5, 7, 9, 123], np.int64))
    _call('dae_step_advance', ctl.data_ptr(), 800, _st())
    _call('dae_step_advance', ctl.data_ptr(), -3, _st())
    assert _np(ctl).tolist() == [802, 9, 11, 123]


def test_batch_commit():
    rng = np.random.default_rng(0)
    B = 1000
    src = [rng.integers(-10 ** 6, 10 ** 6, B).astype(np.int32), rng.standard_normal(B).astype(f32),
           rng.integers(0, B, B).astype(np.int32), rng.integers(0, B, B).astype(np.int32), rng.standard_normal(B).astype(f32),
           rng.standard_normal(16)]
    dst = [torch.full((B + 3,), -7, dtype=torch.int32, device=DEV), torch.full((B + 3,), -7.0, device=DEV),
           torch.full((B + 3,), -7, dtype=torch.int32, device=DEV), torch.full((B + 3,), -7, dtype=torch.int32, device=DEV),
           torch.full((B + 3,), -7.0, device=DEV), torch.full((18,), -7.0, dtype=torch.float64, device=DEV)]
    s_d = [_dev(a) for a in src]
    _call('dae_batch_commit', B, *[t.data_ptr() for t in s_d], *[t.data_ptr() for t in dst], _st())
    for a, t in zip(src, dst):
        g = _np(t)
        assert np.array_equal(g[:len(a)], a) and (g[len(a):] == -7).all()


@pytest.mark.parametrize('with_perm', [True, False])
def test_batch_prepare_explicit(with_perm):
    rng = np.random.default_rng(1)
    B, n_each, offset, cur = 300, 4000, 100, 37
    perm = rng.permutation(n_each).astype(np.int32)
    ctl = _dev(np.array([cur, 0, 0], np.int64))
    rows = torch.full((3 * B + 3,), -7, dtype=torch.int32, device=DEV)
    stats = torch.full((18,), -7.0, dtype=torch.float64, device=DEV)
    perm_d = _dev(perm)
    _call('dae_batch_prepare_explicit', perm_d.data_ptr() if with_perm else None, offset, ctl.data_ptr(), B, n_each,
          rows.data_ptr(), stats.data_ptr(), _st())
    base = perm[offset + cur:offset + cur + B].astype(np.int64) if with_perm else np.arange(offset + cur, offset + cur + B)
    g = _np(rows)
    assert np.array_equal(g[:3 * B], np.concatenate([base, base + n_each, base + 2 * n_each])) and (g[3 * B:] == -7).all()
    want = np.zeros(16)
    want[5] = B                                      # DAE_STAT_SUM_W
    st = _np(stats)
    assert np.array_equal(st[:16], want) and (st[16:] == -7).all()


@pytest.mark.parametrize('F', [1, 1023, 1024, 1025, 200003])
def test_col_scan(F):
    rng = np.random.default_rng(F)
    cnt = rng.integers(0, 6, F).astype(np.int32)
    cnt[rng.random(F) < 0.3] = 0
    if F > 8200:
        cnt[8190:8195] = 1000                        # a carry across the 8192-element chunks
    start = torch.full((F + 3,), -7, dtype=torch.int32, device=DEV)
    cursor = torch.full((F + 2,), -7, dtype=torch.int32, device=DEV)
    cnt_d = _dev(cnt)
    _call('dae_col_scan', cnt_d.data_ptr(), F, start.data_ptr(), cursor.data_ptr(), _st())
    want = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    s, c = _np(start), _np(cursor)
    assert np.array_equal(s[:F + 1], want) and (s[F + 1:] == -7).all()
    assert np.array_equal(c[:F], want[:F]) and (c[F:] == -7).all()
