"""The training step's kernels called one by one through the C ABI, against the fp64 references of step_kernel_oracle.py, element
by element (|got - want| <= c * scale + tiny; c and the scales are derived there): the encoder (K1, its hot-rows variant, the atomic,
gather and deterministic backward), the fused and unfused decode loss, and the optimizer.  Shapes are picked to reach every
compiled instantiation and the tile, chunk and alignment edges of each kernel."""
import numpy as np
import pytest
import torch

import step_kernel_oracle as so

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ERR_UNSUPPORTED = -3
SENT = -7.0          # sentinel for memory a kernel must not touch
BF16_SENT = 0x7F7F   # a bf16 bit pattern no kernel writes here (3.4e38)


def _cabi():
    from dae_rnn_news_recommendation_b200 import _cabi
    return _cabi


def _st():
    return torch.cuda.current_stream().cuda_stream


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev_csr(m):
    return (torch.from_numpy(m.indptr.astype(np.int64)).to(DEV), torch.from_numpy(m.indices.astype(np.int32)).to(DEV),
            torch.from_numpy(m.data.astype(np.float32)).to(DEV))


def _np(t):
    torch.cuda.synchronize()
    return t.detach().cpu().numpy().astype(np.float64)


def _check(name, got, want, scale, c, tiny=1e-30):
    got = np.asarray(got, np.float64)
    err = np.abs(got - want)
    bound = c * scale + tiny
    bad = ~(err <= bound)
    if bad.any():
        idx = np.argwhere(bad)[:5]
        worst = np.unravel_index(np.argmax(np.where(np.isfinite(err), err / bound, np.inf)), err.shape)
        raise AssertionError('%s: %d of %d elements outside c*scale (c=%g); first %s; worst at %s: got %r want %r scale %r' %
                             (name, int(bad.sum()), bad.size, c, idx.tolist(), worst, got[worst], want[worst], scale[worst]))


def _bits16(t):
    torch.cuda.synchronize()
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def _bf16_sentinel(rows, cols):
    return torch.full((rows, cols), BF16_SENT, dtype=torch.int16, device=DEV).view(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------------------------------------
# K1: dae_encode_csr_fwd
# ---------------------------------------------------------------------------------------------------------------------------------
def _encode_fwd(x_dev, rows, n_rows, F, H, in_scale, W, bh, act, ldE, ld_split=0, col_count=None):
    ip, ix, vv = x_dev
    E = torch.full((n_rows, ldE), SENT, device=DEV)
    hi = lo = None
    if ld_split:
        hi, lo = _bf16_sentinel(n_rows, ld_split), _bf16_sentinel(n_rows, ld_split)
    rc = getattr(_cabi().lib(), 'dae_encode_csr_fwd')(ip.data_ptr(), ix.data_ptr(), vv.data_ptr(), None if rows is None else rows.data_ptr(),
                                          n_rows, F, H, in_scale, W.data_ptr(), bh.data_ptr(), _cabi().ACT[act], E.data_ptr(), ldE,
                                          None if col_count is None else col_count.data_ptr(), None if hi is None else hi.data_ptr(),
                                          None if lo is None else lo.data_ptr(), ld_split, _st())
    return rc, E, hi, lo


# (H, W pointer offset in floats): H picks the vector width (H % 4, H % 2) and the number of 128-thread column slices NC; a W
# pointer 4 bytes off its 16-byte alignment forces the scalar width.  Together with the two row counts (G = 4 thread groups per
# row up to 32 x SM count rows, G = 1 above) this runs every (VW, NC, G) instantiation:
#   VW 4: 52/128/500 (NC 1), 1000/1024 (2), 2048 (4), 4000 (8);  VW 2: 50 (1), 510 (2), 1022 (4), 2046 (8);
#   VW 1: 7 (1), 129 / offset 200 (2), offset 500 (4), 513 / offset 1000 (8).
FWD_SHAPES = [(7, 0), (50, 0), (52, 0), (128, 0), (129, 0), (500, 0), (510, 0), (513, 0), (1000, 0), (1022, 0), (1024, 0),
              (2046, 0), (2048, 0), (4000, 0), (200, 1), (500, 1), (1000, 1)]


@pytest.mark.parametrize('many_rows', [False, True], ids=['G4', 'G1'])
@pytest.mark.parametrize('H,w_off', FWD_SHAPES)
def test_encode_fwd_every_instantiation(H, w_off, many_rows):
    """E element-wise against fp64, with row indirection, in_scale != 1, ldE > H, rows longer than 512 entries, empty and fully
    masked rows; the fused bf16 hi / lo copy equals the bf16 split of the returned E bit for bit and leaves its padding alone;
    col_count is exact."""
    F = 3000
    i = FWD_SHAPES.index((H, w_off))
    act = so.ACTS[i % 3]
    n_rows = 32 * _sms() + 1 if many_rows else 37
    n_src = n_rows + 11
    x = so.mask_values(so.edge_csr(n_src, F, mean_nnz=12, seed=H + w_off), 0.25, seed=H, masked_rows=(5, 9))
    rng = np.random.default_rng(H * 3 + w_off)
    rows = np.sort(rng.choice(n_src, n_rows, replace=False)).astype(np.int32)
    rows[:6] = [3, 5, 4, 1, 2, 9]          # the empty, masked, long, full-half and chunk rows first
    rows_t = torch.from_numpy(rows).to(DEV)
    W = rng.normal(0, 0.3, (F, H)).astype(np.float32)
    bh = rng.normal(0, 0.5, H).astype(np.float32)
    W_buf = torch.empty(F * H + 4, device=DEV)
    W_buf[w_off:w_off + F * H] = torch.from_numpy(W.ravel()).to(DEV)
    W_dev = W_buf[w_off:]
    in_scale = 0.8 if i % 2 else 1.0
    ldE, ld_split = H + 3, H + 5
    cc = torch.full((F,), -1, dtype=torch.int32, device=DEV)
    rc, E, hi, lo = _encode_fwd(_dev_csr(x), rows_t, n_rows, F, H, in_scale, W_dev, torch.from_numpy(bh).to(DEV), act, ldE,
                                ld_split, cc)
    assert rc == 0, _cabi().last_error()
    want, scale, _ = so.encode_fwd(x[rows], W, bh, act, in_scale)
    En = _np(E)
    _check('E', En[:, :H], want, scale, so.C_FP32)
    assert np.all(En[:, H:] == SENT)
    h_bits, l_bits = _bits16(hi), _bits16(lo)
    eh, el = so.bf16_split(En[:, :H].astype(np.float32))
    assert np.array_equal(h_bits[:, :H], eh) and np.array_equal(l_bits[:, :H], el)
    assert np.all(h_bits[:, H:] == BF16_SENT) and np.all(l_bits[:, H:] == BF16_SENT)
    xb = x[rows]
    kept = xb.indices[xb.data * np.float32(in_scale) != 0]
    assert np.array_equal(_np(cc).astype(np.int64), np.bincount(kept, minlength=F))


def test_encode_fwd_row_count_boundary():
    """n_rows = 32 x SM count exactly, the largest batch that still splits each row over 4 thread groups, against fp64."""
    F, H = 2000, 500
    n = 32 * _sms()
    x = so.mask_values(so.edge_csr(n, F, seed=4), 0.2)
    rng = np.random.default_rng(1)
    W = rng.normal(0, 0.3, (F, H)).astype(np.float32)
    bh = rng.normal(0, 0.5, H).astype(np.float32)
    rc, E, _, _ = _encode_fwd(_dev_csr(x), None, n, F, H, 1.0, torch.from_numpy(W).to(DEV), torch.from_numpy(bh).to(DEV), 'sigmoid', H)
    assert rc == 0
    want, scale, _ = so.encode_fwd(x, W, bh, 'sigmoid')
    _check('E', _np(E), want, scale, so.C_FP32)


@pytest.mark.parametrize('H', [1025, 2050])
def test_encode_fwd_unsupported_h(H):
    """H = 1025 (odd: scalar width, 9 slices) and 2050 (H % 4 != 0: width 2, 9 slices) exceed the 8 compiled column slices."""
    F = 50
    x = so.edge_csr(4, F, mean_nnz=5, seed=0)
    W = torch.zeros(F, H, device=DEV)
    bh = torch.zeros(H, device=DEV)
    rc, _, _, _ = _encode_fwd(_dev_csr(x), None, 4, F, H, 1.0, W, bh, 'sigmoid', H)
    assert rc == ERR_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------------------------------------
# K1 hot rows: dae_encode_csr_fwd_hot
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,K,hot,groups,F', [(500, 1, 'top', 4, 3000), (500, 102, 'top', 8, 3000), (500, 100, 'all', 4, 100),
                                              (500, 102, 'none', 8, 3000), (1024, 50, 'top', 4, 3000), (1024, 1, 'all', 8, 1),
                                              (1024, 50, 'none', 8, 3000)])
def test_encode_fwd_hot_bit_equal_to_row_kernel(H, K, hot, groups, F):
    """The hot-rows kernel adds a row's entries in CSR order, as the row kernel does with one thread group per row (n_rows above
    32 x SM count): the two are bit-identical.  K = 1 and K at the 200 KB limit, every stored column hot or none, 4 and 8 row
    groups with n_rows not a multiple of either, H = 1024 (two column slices)."""
    n = 32 * _sms() + 7
    x = so.mask_values(so.edge_csr(n, F, mean_nnz=15, seed=K + H, long_row=F > 600, planted=F > 8), 0.2)
    rng = np.random.default_rng(K)
    W = torch.from_numpy(rng.normal(0, 0.3, (F, H)).astype(np.float32)).to(DEV)
    bh = torch.from_numpy(rng.normal(0, 0.5, H).astype(np.float32)).to(DEV)
    assert K * H * 4 <= 200 * 1024
    freq = np.bincount(x.indices, minlength=F)
    hot_cols = np.argsort(-freq, kind='stable')[:K].astype(np.int32)
    slot = np.full(F, -1, np.int32)
    if hot != 'none':
        slot[hot_cols] = np.arange(K, dtype=np.int32)
    if hot == 'all':
        assert K >= F
    xd = _dev_csr(x)
    for act in so.ACTS:
        rc, E_row, _, _ = _encode_fwd(xd, None, n, F, H, 0.9, W, bh, act, H)
        assert rc == 0
        E_hot = torch.full((n, H), SENT, device=DEV)
        hc, hs = torch.from_numpy(np.resize(hot_cols, K)).to(DEV), torch.from_numpy(slot).to(DEV)
        _cabi().call('dae_encode_csr_fwd_hot', xd[0].data_ptr(), xd[1].data_ptr(), xd[2].data_ptr(), n, F, H, 0.9, W.data_ptr(),
                     bh.data_ptr(), _cabi().ACT[act], E_hot.data_ptr(), H, hc.data_ptr(), hs.data_ptr(), K, groups, _st())
        torch.cuda.synchronize()
        assert torch.equal(E_hot.view(torch.int32), E_row.view(torch.int32)), act


# ---------------------------------------------------------------------------------------------------------------------------------
# K5: dae_encode_csr_bwd (atomic), dae_encode_csr_bwd_gather, dae_encode_csr_bwd_det + dae_encode_sparse_dw_add
# ---------------------------------------------------------------------------------------------------------------------------------
def _encode_bwd_all(x, rows, n, F, H, in_scale, act, E, dE0, dE_add, bh, dW0, dbh_zeroed, gather_ok=True):
    """Runs the three backward variants on copies of the same inputs; returns {variant: (dA, dbh, dW)}.  gather_ok = False: H
    needs more than two column slices, and the gather must refuse it with DAE_ERR_UNSUPPORTED."""
    c = _cabi()
    ip, ix, vv = _dev_csr(x)
    rows_p = None if rows is None else rows.data_ptr()
    add_p = None if dE_add is None else dE_add.data_ptr()
    cc = torch.zeros(F, dtype=torch.int32, device=DEV)
    Etmp = torch.empty(n, H, device=DEV)
    # col_count of the batch comes from the forward, as in the step
    assert c.lib().dae_encode_csr_fwd(ip.data_ptr(), ix.data_ptr(), vv.data_ptr(), rows_p, n, F, H, in_scale, dW0.data_ptr(), bh.data_ptr(),
                                      c.ACT[act], Etmp.data_ptr(), H, cc.data_ptr(), None, None, 0, _st()) == 0
    cap = max(1, int(x.nnz))
    out = {}

    def fresh():
        dbh = torch.zeros(H, device=DEV) if dbh_zeroed else torch.full((H,), float('nan'), device=DEV)
        return dE0.clone(), dW0.clone(), dbh

    dE, dW, dbh = fresh()
    c.call('dae_encode_csr_bwd', ip.data_ptr(), ix.data_ptr(), vv.data_ptr(), rows_p, n, F, H, in_scale, E.data_ptr(), bh.data_ptr(),
           c.ACT[act], dE.data_ptr(), add_p, H, dW.data_ptr(), dbh.data_ptr(), int(dbh_zeroed), _st())
    out['atomic'] = (dE, dbh, dW)

    dE, dW, dbh = fresh()
    cs, cur = torch.empty(F + 1, dtype=torch.int32, device=DEV), torch.empty(F, dtype=torch.int32, device=DEV)
    ec, er, ev = (torch.empty(cap, dtype=torch.int32, device=DEV), torch.empty(cap, dtype=torch.int32, device=DEV),
                  torch.empty(cap, device=DEV))
    rc = getattr(c.lib(), 'dae_encode_csr_bwd_gather')(ip.data_ptr(), ix.data_ptr(), vv.data_ptr(), rows_p, n, F, H, in_scale, E.data_ptr(),
                                           bh.data_ptr(), c.ACT[act], dE.data_ptr(), add_p, H, dW.data_ptr(), dbh.data_ptr(),
                                           int(dbh_zeroed), cc.data_ptr(), cs.data_ptr(), cur.data_ptr(), ec.data_ptr(), er.data_ptr(),
                                           ev.data_ptr(), _st())
    if gather_ok:
        assert rc == 0, c.last_error()
        out['gather'] = (dE, dbh, dW)
        torch.cuda.synchronize()
        assert np.array_equal(cs.cpu().numpy()[1:], np.cumsum(cc.cpu().numpy()))   # col_scan over several 8192-column chunks
    else:   # more than two column slices: the gather is not compiled for them and says so before any launch
        assert rc == ERR_UNSUPPORTED

    dE, dW, dbh = fresh()
    wsb = c.query('dae_encode_csr_bwd_det_workspace', n, F, H, cap)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    c.call('dae_encode_csr_bwd_det', ip.data_ptr(), ix.data_ptr(), vv.data_ptr(), rows_p, n, F, H, in_scale, E.data_ptr(),
           bh.data_ptr(), c.ACT[act], dE.data_ptr(), add_p, H, dbh.data_ptr(), cc.data_ptr(), cap, ws.data_ptr(), wsb, _st())
    c.call('dae_encode_sparse_dw_add', n, F, H, cap, ws.data_ptr(), wsb, dW.data_ptr(), _st())
    out['det'] = (dE, dbh, dW)
    torch.cuda.synchronize()
    return out


# (F, H): F at and around the 8192-column chunks of col_scan and far past them; H reaches every compiled backward instantiation.
# The dispatch picks the vector width VW from H (H % 4, H % 2) and the column slices NC = ceil(H / (128 VW)):
#   atomic encode_bwd_kernel, VW x NC = 4 x {1, 2, 4, 8}: 100, 1000, 2048, 4000;  2 x {1, 2, 4, 8}: 130, 510, 1022, 2046;
#                                       1 x {1, 2, 4, 8}: 7, 129, 385, 513;
#   gather (NC <= 2 only; above, DAE_ERR_UNSUPPORTED): 4 x {1, 2}: 100, 1000;  2 x {1, 2}: 130, 510;  1 x {1, 2}: 7, 129;
#   det gather, one width per VW, with 1 to 8 passes of its 128 VW-column loop (H = 1000: two passes at VW 4).
BWD_SHAPES = [(8191, 100), (8192, 1000), (8193, 2048), (8193, 4000), (8191, 130), (8192, 510), (8193, 1022), (8191, 2046),
              (50000, 7), (8192, 129), (8193, 385), (8191, 513), (50000, 64)]


@pytest.mark.parametrize('F,H', BWD_SHAPES)
def test_encode_bwd_three_variants(F, H):
    """dA, dbh and dW (accumulated onto a non-zero dense dW) of the atomic, gather and deterministic backward against fp64: dE_add,
    n_rows % 4 != 0, row indirection, several col_scan chunks, a column of 150 entries (its run crosses gather chunks of 32 and det
    chunks of 64 entries).  dA is the same expression in the three kernels and is compared bit for bit."""
    i = BWD_SHAPES.index((F, H))
    act, n = so.ACTS[i % 3], 203
    vw = 4 if H % 4 == 0 else (2 if H % 2 == 0 else 1)
    gather_ok = -(-H // (128 * vw)) <= 2
    x_src = so.mask_values(so.edge_csr(n + 20, F, mean_nnz=25, seed=F), 0.3, masked_rows=(5, 30))
    rng = np.random.default_rng(F)
    rows = np.concatenate([np.arange(6), rng.choice(np.arange(6, n + 20), n - 6, replace=False)]).astype(np.int32)
    x = x_src[rows]
    in_scale = 0.85
    W = rng.normal(0, 0.2, (F, H)).astype(np.float32)
    bh = rng.normal(0, 0.5, H).astype(np.float32)
    E_ref = so.encode_fwd(x, W, bh, act, in_scale)[0].astype(np.float32)
    dE0 = rng.normal(0, 1, (n, H)).astype(np.float32)
    dEa = rng.normal(0, 0.5, (n, H)).astype(np.float32)
    dW0 = rng.normal(0, 1, (F, H)).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    out = _encode_bwd_all(x_src, T(rows), n, F, H, in_scale, act, T(E_ref), T(dE0), T(dEa), T(bh), T(dW0), dbh_zeroed=i % 2 == 0,
                          gather_ok=gather_ok)
    assert ('gather' in out) == gather_ok
    ref = so.encode_bwd(x, E_ref, dE0, dEa, bh, act, in_scale, dW0)
    a_bits = out['atomic'][0].view(torch.int32)
    for name, (dA, dbh, dW) in out.items():
        assert torch.equal(dA.view(torch.int32), a_bits), name
        _check(name + ' dA', _np(dA), *ref['dA'], so.C_FP32)
        _check(name + ' dbh', _np(dbh), *ref['dbh'], so.C_FP32)
        _check(name + ' dW', _np(dW), *ref['dW'], so.C_FP32)


def test_encode_bwd_all_masked_leaves_dw():
    """Every entry of the batch masked: dW is left bit for bit, dA and dbh are still computed."""
    F, H, n = 8193, 100, 41
    x = so.edge_csr(n, F, mean_nnz=10, seed=2)
    x.data[:] = 0.0
    rng = np.random.default_rng(3)
    E = rng.normal(0, 0.2, (n, H)).astype(np.float32)
    dE0 = rng.normal(0, 1, (n, H)).astype(np.float32)
    bh = rng.normal(0, 0.5, H).astype(np.float32)
    dW0 = rng.normal(0, 1, (F, H)).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    out = _encode_bwd_all(x, None, n, F, H, 1.0, 'tanh', T(E), T(dE0), None, T(bh), T(dW0), dbh_zeroed=False)
    ref = so.encode_bwd(x, E, dE0, None, bh, 'tanh', 1.0, dW0)
    for name, (dA, dbh, dW) in out.items():
        assert np.array_equal(dW.cpu().numpy().view(np.int32), dW0.view(np.int32)), name
        _check(name + ' dA', _np(dA), *ref['dA'], so.C_FP32)
        _check(name + ' dbh', _np(dbh), *ref['dbh'], so.C_FP32)


# ---------------------------------------------------------------------------------------------------------------------------------
# fused decode: dae_decode_fused_bf16x3 and dae_decode_fused_bf16x3_det
# ---------------------------------------------------------------------------------------------------------------------------------
def _split(x, ld):
    rows, cols = x.shape
    hi = torch.zeros(rows, ld, dtype=torch.bfloat16, device=DEV)
    lo = torch.zeros(rows, ld, dtype=torch.bfloat16, device=DEV)
    _cabi().call('dae_split_bf16', x.data_ptr(), rows, cols, x.stride(0), hi.data_ptr(), lo.data_ptr(), ld, -1, 1.0, _st())
    return hi, lo


def _decode_inputs(act, loss, Brows, F, K, seed, indirect, saturate):
    rng = np.random.default_rng(seed)
    n_src = Brows + (9 if indirect else 0)
    x_src = so.edge_csr(n_src, F, mean_nnz=min(30, max(2, F // 8)), kind='binary' if loss == 'cross_entropy' else 'tfidf', seed=seed,
                        long_row=F > 600)
    rows = np.arange(Brows, dtype=np.int32)
    if indirect:   # a shuffled subset that keeps edge_csr's full-half (1), dense-chunk (2), empty (3) and long (4) rows
        edge = np.array([1, 2, 3, 4])
        rest = rng.permutation(np.setdiff1d(np.arange(n_src), edge))[:Brows - len(edge)]
        rows = rng.permutation(np.concatenate([edge, rest])).astype(np.int32)
    if loss == 'cross_entropy' and act != 'sigmoid':     # D inside (0, 1): pre-activations in (0.25, 0.75)
        E = rng.uniform(-1, 1, (Brows, K)).astype(np.float32)
        W = (rng.uniform(-1, 1, (F, K)) * (0.25 / K)).astype(np.float32)
        bv = rng.uniform(0.3, 0.7, F).astype(np.float32)
    else:
        E = rng.normal(0, 1, (Brows, K)).astype(np.float32)
        W = (rng.normal(0, 1, (F, K)) * (1.5 / np.sqrt(K))).astype(np.float32)
        bv = rng.normal(0, 0.3, F).astype(np.float32)
    if saturate:   # +-90 next to ordinary chunks: every third 16-column chunk holds one saturated column
        cols = np.arange(5, F, 48)
        bv[cols] = np.where(np.arange(len(cols)) % 2 == 0, 90.0, -90.0).astype(np.float32)
    w = (rng.random(Brows) * 3).astype(np.float32)
    w[::7] = 0.0
    return x_src, rows, E, W, bv, w


def _run_decode(det, Brows, F, K, Ehl, Whl, ldk, xd, rows_t, bv, act, loss, w, stats, prepared):
    c = _cabi()
    ld_dz = (F + 31) // 32 * 32
    n_parts = 2 * ((F + 127) // 128)
    dzh, dzl = _bf16_sentinel(Brows + 2, ld_dz), _bf16_sentinel(Brows + 2, ld_dz)
    parts = torch.full((n_parts if det else 1, Brows), SENT, device=DEV)
    tptr = torch.full((Brows, n_parts + 1), -1, dtype=torch.int32, device=DEV)
    if prepared:
        c.call('dae_decode_prepare', Brows, F, xd[0].data_ptr(), xd[1].data_ptr(), _cabi().ptr(rows_t), parts.data_ptr(), tptr.data_ptr(),
               _st())
    c.call('dae_decode_fused_bf16x3_det' if det else 'dae_decode_fused_bf16x3', Brows, F, K, Ehl[0].data_ptr(), Ehl[1].data_ptr(), ldk,
           Whl[0].data_ptr(), Whl[1].data_ptr(), ldk, xd[0].data_ptr(), xd[1].data_ptr(), xd[2].data_ptr(), _cabi().ptr(rows_t),
           bv.data_ptr(), c.ACT[act], c.LOSS[loss], w.data_ptr(), stats.data_ptr(), dzh.data_ptr(), dzl.data_ptr(), ld_dz,
           parts.data_ptr(), tptr.data_ptr(), int(prepared), _st())
    torch.cuda.synchronize()
    return dzh, dzl, parts


# (act, loss, Brows, F, K, rows indirection, +-90 pre-activations): all six ACT x LOSS instantiations; Brows on both sides of the
# 128-row tile; F below, on and past the 64- and 128-column boundaries; K below, on and past the 32-wide k-block and several ring
# cycles (4 stages of 32); tile counts from 1 to above the SM count (800 x 10 000: 553 tiles; F = 50 000: 391 per 128 rows).
DECODE_CASES = [
    ('sigmoid', 'cross_entropy', 1, 8, 8, False, False),
    ('tanh', 'cross_entropy', 127, 63, 31, True, False),
    ('none', 'cross_entropy', 128, 64, 32, False, False),
    ('sigmoid', 'mean_squared', 129, 65, 33, True, False),
    ('tanh', 'mean_squared', 800, 127, 52, False, True),
    ('none', 'mean_squared', 129, 128, 129, True, False),
    ('sigmoid', 'cross_entropy', 800, 129, 500, True, True),
    ('sigmoid', 'cross_entropy', 128, 1000, 1000, False, True),
    ('tanh', 'cross_entropy', 129, 1000, 129, True, False),
    ('none', 'cross_entropy', 1, 1000, 33, False, False),
    ('sigmoid', 'mean_squared', 800, 1000, 8, True, True),
    ('tanh', 'mean_squared', 127, 10000, 52, True, False),
    ('sigmoid', 'cross_entropy', 800, 10000, 500, True, True),
    ('sigmoid', 'cross_entropy', 129, 50000, 52, False, True),
]


@pytest.mark.parametrize('act,loss,Brows,F,K,indirect,saturate', DECODE_CASES)
def test_fused_decode_against_fp64(act, loss, Brows, F, K, indirect, saturate):
    """dZ (bf16 hi + lo) element-wise and the row losses against fp64; the _det variant's partial of every 64-column half tile
    against the fp64 loss of that half tile; dZ bits equal between the plain and _det variants and between prepared = 0 and 1;
    columns [F, ld_dz) zero; the guard rows past Brows untouched.  Rows with more than three stored entries in one 16-column chunk
    and a fully stored 64-column half come from edge_csr; some rows have weight 0."""
    seed = Brows * 7 + F + K
    x_src, rows, E, W, bv, w = _decode_inputs(act, loss, Brows, F, K, seed, indirect, saturate)
    ldk = (K + 7) // 8 * 8
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    Ehl, Whl = _split(T(E), ldk), _split(T(W), ldk)
    xd = _dev_csr(x_src)
    rows_t, bv_t, w_t = (T(rows) if indirect else None), T(bv), T(w)   # rows == NULL: batch row r is CSR row r
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    sum_w = float(np.sum(w.astype(np.float64)))
    stats[_cabi().STAT['sum_w']] = sum_w
    args = (Brows, F, K, Ehl, Whl, ldk, xd, rows_t, bv_t, act, loss, w_t, stats)
    h0, l0, p0 = _run_decode(False, *args, prepared=False)
    h1, l1, p1 = _run_decode(True, *args, prepared=False)
    h2, l2, _ = _run_decode(False, *args, prepared=True)
    hb, lb = _bits16(h0), _bits16(l0)
    assert np.array_equal(hb, _bits16(h1)) and np.array_equal(lb, _bits16(l1)), 'plain vs _det dZ bits'
    assert np.array_equal(hb, _bits16(h2)) and np.array_equal(lb, _bits16(l2)), 'prepared = 0 vs 1 dZ bits'
    assert np.all(hb[Brows:] == BF16_SENT) and np.all(lb[Brows:] == BF16_SENT), 'guard rows'
    assert np.all(hb[:Brows, F:] == 0) and np.all(lb[:Brows, F:] == 0), 'columns [F, ld_dz)'

    z, zs = so.fused_decode_z(E, W, bv)
    dZ, s_dZ, lt, s_l = so.decode_loss(z, x_src[rows], w, sum_w, act, loss, zs)
    got = (h0.float() + l0.float())[:Brows, :F]
    # 1e-20: where the MUFU sigmoid of z = -90 comes out as an fp32 denormal rather than 0, dZ of a stored entry is
    # sc * D / 1e-16 ~ 1e-24 against the reference's 0
    _check('dZ', _np(got), dZ, s_dZ, so.C_BF16X3, 1e-20)
    tiny_col = 2.0 ** -20
    _check('row loss', _np(p0)[0], lt.sum(1), s_l.sum(1), so.C_BF16X3, F * tiny_col)
    parts = _np(p1)
    n_half = parts.shape[0]
    for t in range(n_half):
        c0, c1 = 64 * t, min(F, 64 * t + 64)
        if c0 >= F:
            want, sc = np.zeros(Brows), np.zeros(Brows)
        else:
            want, sc = lt[:, c0:c1].sum(1), s_l[:, c0:c1].sum(1)
        _check('half tile %d loss' % t, parts[t], want, sc, so.C_BF16X3, 64 * tiny_col)


def test_decode_prepare_many_rows():
    """dae_decode_prepare at 70 000 rows (more than grid.y's 65 535: the rows loop) with row indirection: tile_ptr exactly the
    number of stored entries of each row below every 64-column boundary, and the row-loss vector zeroed."""
    B, F = 70000, 300
    n_src = B + 100
    x = so.edge_csr(n_src, F, mean_nnz=6, seed=9, long_row=False, planted=False)
    rows = np.random.default_rng(0).permutation(n_src)[:B].astype(np.int32)
    xd = _dev_csr(x)
    n_half = 2 * ((F + 127) // 128)
    tptr = torch.full((B, n_half + 1), -1, dtype=torch.int32, device=DEV)
    rl = torch.full((B,), SENT, device=DEV)
    rows_t = torch.from_numpy(rows).to(DEV)
    _cabi().call('dae_decode_prepare', B, F, xd[0].data_ptr(), xd[1].data_ptr(), rows_t.data_ptr(), rl.data_ptr(), tptr.data_ptr(), _st())
    got = tptr.cpu().numpy()
    want = np.empty_like(got)
    for r_i, r in enumerate(rows):
        want[r_i] = np.searchsorted(x.indices[x.indptr[r]:x.indptr[r + 1]], np.arange(n_half + 1) * 64)
    assert np.array_equal(got, want)
    assert float(rl.abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------------------------------------------
# unfused decode loss: dae_decode_loss_bwd + dae_colsum
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('F', [300, 8192, 8193, 20000])
@pytest.mark.parametrize('loss', so.LOSSES)
def test_decode_loss_bwd_against_fp64(loss, F):
    """dZ element-wise and the row losses against fp64 for every activation, at one and several 8192-float chunks of the densified
    target row (cosine needs whole-row sums across them); rows with an all-zero target (cosine: the clamp branch); zero weights;
    row indirection.  dae_colsum of dZ against the fp64 column sums of the same dZ."""
    c = _cabi()
    B = 45
    n_src = B + 5
    x_src = so.edge_csr(n_src, F, mean_nnz=40, kind='binary' if loss == 'cross_entropy' else 'tfidf', seed=F, long_row=True)
    rng = np.random.default_rng(F + len(loss))
    rows = np.concatenate([[3, 1, 2, 4], rng.choice(np.setdiff1d(np.arange(n_src), [1, 2, 3, 4]), B - 4, replace=False)]).astype(np.int32)
    xd = _dev_csr(x_src)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    for act in so.ACTS:
        if loss == 'cross_entropy' and act != 'sigmoid':
            Z = rng.uniform(-0.2, 0.2, (B, F)).astype(np.float32)
            bv = rng.uniform(0.3, 0.7, F).astype(np.float32)
        else:
            Z = rng.normal(0, 1.5, (B, F)).astype(np.float32)
            bv = rng.normal(0, 0.3, F).astype(np.float32)
        w = (rng.random(B) * 2).astype(np.float32)
        w[5] = 0.0
        sum_w = float(np.sum(w.astype(np.float64)))
        stats = torch.zeros(16, dtype=torch.float64, device=DEV)
        stats[c.STAT['sum_w']] = sum_w
        ldz = F + 4
        Zd = torch.full((B, ldz), SENT, device=DEV)
        Zd[:, :F] = T(Z)
        rl = torch.full((B,), SENT, device=DEV)
        rows_t, bv_t, w_t = T(rows), T(bv), T(w)   # held until the launch: a freed block is handed to the next allocation
        c.call('dae_decode_loss_bwd', xd[0].data_ptr(), xd[1].data_ptr(), xd[2].data_ptr(), rows_t.data_ptr(), B, F, bv_t.data_ptr(),
               c.ACT[act], c.LOSS[loss], w_t.data_ptr(), stats.data_ptr(), Zd.data_ptr(), ldz, rl.data_ptr(), _st())
        z = Z.astype(np.float64) + bv.astype(np.float64)
        zs = np.abs(Z.astype(np.float64)) + np.abs(bv.astype(np.float64))
        dZ, s_dZ, lt, s_l = so.decode_loss(z, x_src[rows], w, sum_w, act, loss, zs)
        got = _np(Zd)
        _check('%s dZ' % act, got[:, :F], dZ, s_dZ, so.C_FP32)
        assert np.all(got[:, F:] == SENT)
        _check('%s row loss' % act, _np(rl), lt.sum(1), s_l.sum(1), so.C_FP32)
        if loss == 'cosine_proximity':
            assert np.all(got[0, :F] == 0.0) and float(rl[0]) == 0.0          # all-zero target row
        out = torch.full((F,), SENT, device=DEV)
        c.call('dae_colsum', Zd.data_ptr(), B, F, ldz, out.data_ptr(), _st())
        g = got[:, :F]
        _check('%s colsum' % act, _np(out), g.sum(0), np.abs(g).sum(0), so.C_FP32)


# ---------------------------------------------------------------------------------------------------------------------------------
# optimizer: dae_optimizer_step
# ---------------------------------------------------------------------------------------------------------------------------------
OPTS = ['gradient_descent', 'ada_grad', 'momentum', 'adam']


def _opt_call(theta, grad, s1, s2, n, opt, lr, mom, gscale, step, ctl=None, split=None):
    c = _cabi()
    wh, wl, F, H, lds = (None, None, 0, 0, 0) if split is None else split
    c.call('dae_optimizer_step', theta.data_ptr(), grad.data_ptr(), None if s1 is None else s1.data_ptr(),
           None if s2 is None else s2.data_ptr(), n, c.OPT[opt], lr, mom, gscale, step, None if ctl is None else ctl.data_ptr(),
           None if wh is None else wh.data_ptr(), None if wl is None else wl.data_ptr(), F, H, lds, _st())


@pytest.mark.parametrize('offset', [0, 1], ids=['aligned', 'offset4'])
@pytest.mark.parametrize('opt', OPTS)
def test_optimizer_five_steps(opt, offset):
    """Five steps of each rule against fp64, n % 4 != 0 (float4 bulk + scalar tail) and theta 4 bytes off its 16-byte alignment
    (the scalar kernel for everything)."""
    n = 4 * 2503 + 3
    rng = np.random.default_rng(OPTS.index(opt) * 2 + offset)
    theta0 = rng.normal(0, 1, n).astype(np.float32)
    grads = [rng.normal(0, 1, n).astype(np.float32) for _ in range(5)]
    buf = torch.zeros(n + 4, device=DEV)
    theta = buf[offset:offset + n]
    theta.copy_(torch.from_numpy(theta0))
    s1 = torch.full((n,), 0.1 if opt == 'ada_grad' else 0.0, device=DEV) if opt != 'gradient_descent' else None
    s2 = torch.zeros(n, device=DEV) if opt == 'adam' else None
    lr, mom, gscale = 0.05, 0.7, 0.6
    for t, g in enumerate(grads, 1):
        _opt_call(theta, torch.from_numpy(g).to(DEV), s1, s2, n, opt, lr, mom, gscale, t)
    want, _, _, scale = so.optimizer_steps(opt, theta0, [g.astype(np.float64) for g in grads], lr, mom, gscale,
                                           slot1=np.full(n, 0.1) if opt == 'ada_grad' else None)
    _check(opt, _np(theta), want, scale, so.C_FP32)


@pytest.mark.parametrize('F,H,ld', [(37, 51, 56), (40, 52, 64), (33, 7, 7)])
def test_optimizer_bf16_copy_of_w(F, H, ld):
    """The fused bf16 hi / lo copy of W equals the bf16 split of the updated theta bit for bit (H odd and ld_split > H: scalar
    path; H % 4 == 0: float4 path), its padding columns untouched, and the whole of theta -- W and the biases past F x H, which
    get no bf16 copy -- updated as fp64 Adam says."""
    n = F * H + H + F
    rng = np.random.default_rng(F * H)
    theta0 = rng.normal(0, 1, n).astype(np.float32)
    g0 = rng.normal(0, 1, n).astype(np.float32)
    theta = torch.from_numpy(theta0).to(DEV)
    g = torch.from_numpy(g0).to(DEV)
    s1, s2 = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    wh, wl = _bf16_sentinel(F + 1, ld), _bf16_sentinel(F + 1, ld)
    _opt_call(theta, g, s1, s2, n, 'adam', 0.01, 0.0, 1.0, 1, split=(wh, wl, F, H, ld))
    want, _, _, scale = so.optimizer_steps('adam', theta0, [g0], 0.01)
    got = _np(theta)
    _check('theta', got, want, scale, so.C_FP32)
    assert np.all(got[F * H:] != theta0[F * H:])          # the biases moved (Adam's first step moves every entry by ~lr)
    th = got.astype(np.float32)[:F * H].reshape(F, H)
    eh, el = so.bf16_split(th)
    hb, lb = _bits16(wh), _bits16(wl)
    assert np.array_equal(hb[:F, :H], eh) and np.array_equal(lb[:F, :H], el)
    assert np.all(hb[:F, H:] == BF16_SENT) and np.all(lb[:F, H:] == BF16_SENT) and np.all(hb[F:] == BF16_SENT)


def test_optimizer_adam_device_step_counter():
    """Adam with the step read from ctl[2] on the device gives the same bits as the host-side step argument, at t = 1, 2 and 7."""
    n = 4 * 1000 + 1
    rng = np.random.default_rng(11)
    th0 = torch.from_numpy(rng.normal(0, 1, n).astype(np.float32)).to(DEV)
    a, b = th0.clone(), th0.clone()
    sa1, sa2, sb1, sb2 = (torch.zeros(n, device=DEV) for _ in range(4))
    ctl = torch.zeros(4, dtype=torch.int64, device=DEV)
    for t in (1, 2, 7):
        g = torch.from_numpy(rng.normal(0, 1, n).astype(np.float32)).to(DEV)
        _opt_call(a, g, sa1, sa2, n, 'adam', 0.01, 0.0, 1.0, t)
        ctl[2] = t
        _opt_call(b, g, sb1, sb2, n, 'adam', 0.01, 0.0, 1.0, 0, ctl=ctl)
        torch.cuda.synchronize()
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), t
        assert torch.equal(sa2.view(torch.int32), sb2.view(torch.int32)), t


def test_optimizer_adagrad_step_is_correctly_rounded():
    """One Adagrad step from theta = 0, bit for bit against NumPy float32: theta = -(lr * g) / sqrt(0.1 + g * g).

    This deliberately pins the kernel's expression and its build without fast-math (fp32 sqrt and division correctly rounded), not
    only the TF-1.12 rule, which TF writes as var -= lr * grad * rsqrt(accum): the same value up to about 1 ulp.  A rewrite of that
    kind is numerically harmless and passes the fp64 bound of test_optimizer_five_steps, but it changes the trained parameters'
    bits, so it should be made on purpose, together with this test.  The fp64 bound cannot see a 1-ulp change; this check can.  The accumulator is accepted with or without a fused multiply-add."""
    n = 4 * 4096 + 2
    g = np.random.default_rng(12).normal(0, 1, n).astype(np.float32)
    theta = torch.zeros(n, device=DEV)
    s1 = torch.full((n,), 0.1, device=DEV)
    lr = np.float32(0.05)
    _opt_call(theta, torch.from_numpy(g).to(DEV), s1, None, n, 'ada_grad', float(lr), 0.0, 1.0, 1)
    got = theta.cpu().numpy()
    acc_fma = (g.astype(np.float64) * g.astype(np.float64) + np.float64(np.float32(0.1))).astype(np.float32)
    acc_sep = (g * g + np.float32(0.1)).astype(np.float32)
    ok = np.zeros(n, bool)
    for acc in (acc_fma, acc_sep):
        want = -((lr * g) / np.sqrt(acc))
        ok |= got.view(np.int32) == want.astype(np.float32).view(np.int32)
    assert ok.all(), int((~ok).sum())
