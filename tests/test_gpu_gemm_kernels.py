"""The general GEMMs (dae_gemm_bf16x3, dae_gemm_bf16x3_det, dae_gemm_sym_bf16x3(_det), dae_sgemm) through the C ABI against the
references of tests/gemm_kernel_oracle.py, element by element.

Every output is surrounded by sentinels: C has columns [n_store, ldc), a row past M and a guard row, and may start one float into
its buffer; special_out has a guard element at index M.  Operand memory past K (and past M / N) holds bf16 NaN, so only TMA's zero
fill can give the tile tails.  (a) runs every tile engine on exact operands and asserts bit equality; (b) checks the step's shapes
against the fp64 bound with row and column scales spread over 2^+-20; (c) checks every GEMM call of real training steps against
its own inputs; (d) covers dae_sgemm; (e) asserts which kernels the dispatch launched."""
import functools

import numpy as np
import pytest
import torch

import gemm_kernel_oracle as gk
from helpers import device_copy, xavier

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SENT = np.float32(-7.25)


def _call(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call(name, *args)


def _st():
    return torch.cuda.current_stream().cuda_stream


@functools.lru_cache(None)
def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _ld(n):
    return (n + 1 + 7) // 8 * 8     # at least one padding column


def _operand(hi, lo, mn):
    """bf16 bit arrays [rows x K] -> device hi / lo buffers, K-major [rows + 3 x ld >= K + 1] or MN-major [K + 3 x ld >= rows + 1],
    every element outside the logical matrix bf16 NaN."""
    out = []
    for bits in (hi, lo):
        b = bits.T if mn else bits
        buf = np.full((b.shape[0] + 3, _ld(b.shape[1])), gk.BF16_NAN, np.uint16)
        buf[:b.shape[0], :b.shape[1]] = b
        out.append(torch.from_numpy(buf.view(np.int16)).to(DEV))
    return out[0], out[1], out[0].shape[1]


class Out:
    """C [M x ldc] starting `off` floats into a sentinel-filled buffer of M + 2 rows, and special_out [M + 1]."""

    def __init__(self, M, ldc, n_store, off=0, c0=None, sp0=None):
        self.M, self.ldc, self.n_store, self.off = M, ldc, n_store, off
        host = np.full(off + (M + 2) * ldc + 4, SENT, np.float32)
        if c0 is not None:
            host[off:off + M * ldc].reshape(M, ldc)[:, :n_store] = c0[:, :n_store]
        self.buf = torch.from_numpy(host).to(DEV)
        sp = np.full(M + 1, SENT, np.float32)
        if sp0 is not None:
            sp[:M] = sp0
        self.sp = torch.from_numpy(sp).to(DEV)

    @property
    def ptr(self):
        return self.buf.data_ptr() + 4 * self.off

    def check(self, name, want, want_sp=None):
        host = self.buf.cpu().numpy()
        M, ldc, ns, off = self.M, self.ldc, self.n_store, self.off
        C = host[off:off + (M + 2) * ldc].reshape(M + 2, ldc)
        gk.check_exact(name + ' C', C[:M, :ns], want[:, :ns])
        rest = host.copy()
        rest[off:off + M * ldc].reshape(M, ldc)[:, :ns] = SENT
        bad = rest.view(np.uint32) != SENT.view(np.uint32)
        assert not bad.any(), '%s: %d sentinels overwritten, first flat index %s (C starts at %d, ldc %d)' % (
            name, int(bad.sum()), np.argwhere(bad)[:5].ravel().tolist(), off, ldc)
        sp = self.sp.cpu().numpy()
        if want_sp is not None:
            gk.check_exact(name + ' special', sp[:M], want_sp)
            assert sp[M].view(np.uint32) == SENT.view(np.uint32), '%s: special_out[M] overwritten' % name
        else:
            assert (sp.view(np.uint32) == SENT.view(np.uint32)).all(), '%s: special_out written' % name


class Config:
    """dae_gemm_config for the duration of a with-block."""

    def __init__(self, pair=False, lean=False):
        self.args = (1 if pair else -1, 1 if lean else 0)

    def __enter__(self):
        _call('dae_gemm_config', *self.args)

    def __exit__(self, *exc):
        _call('dae_gemm_config', -1, 0)


@functools.lru_cache(None)
def _det_ws():
    from dae_rnn_news_recommendation_b200 import _cabi
    return torch.empty(_cabi.query('dae_gemm_det_workspace') // 4, dtype=torch.float32, device=DEV)


def _gemm(det, M, N, K, alpha, A, a_mn, B, b_mn, out, n_store, special_col, k_splits, accumulate):
    (ah, al, lda), (bh, bl, ldb) = A, B
    args = (M, N, K, float(alpha), ah.data_ptr(), al.data_ptr(), lda, a_mn, bh.data_ptr(), bl.data_ptr(), ldb, b_mn, out.ptr, out.ldc,
            n_store, special_col, out.sp.data_ptr() if special_col >= 0 else None, k_splits, accumulate)
    if det:
        ws = _det_ws()
        ws.fill_(float('nan'))      # a slot the fixup reads but no segment wrote shows up as NaN
        _call('dae_gemm_bf16x3_det', *args, ws.data_ptr(), ws.numel() * 4, _st())
    else:
        _call('dae_gemm_bf16x3', *args, _st())
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------------
# (a) every engine, bit for bit
# ---------------------------------------------------------------------------------------------------------------------------
ENGINES = {   # name: (pair, lean, det, k_splits)
    'auto': (False, False, False, 1),
    'stream_k': (False, False, False, -1),
    'split2': (False, False, False, 2),
    'split7': (False, False, False, 7),
    'split_over_kblocks': (False, False, False, 1000),
    'pair': (True, False, False, 1),
    'pair_stream_k': (True, False, False, -1),
    'lean': (False, True, False, 1),
    'lean_stream_k': (False, True, False, -1),
    'det': (False, False, True, 1),
    'det_stream_k': (False, False, True, -1),
}
# ragged M, N, K; (1345, 833): 77 tiles of 128 x 128 against 154 of 128 x 64 (two waves): the auto pick takes 128 x 128
RAGGED = [(1, 1, 1), (65, 17, 31), (129, 65, 33), (301, 129, 63), (65, 501, 65), (129, 501, 700), (301, 258, 3000), (1345, 833, 129)]


def _layouts(N):
    """(n_store, special_col, ldc, off): all columns with ldc a multiple of 4; [C | special] with an odd ldc and C one float into its
    buffer; n_store < N without a special column (column n_store computed, not stored); a gap between n_store and special_col."""
    out = [(N, -1, (N + 3) // 4 * 4, 0)]
    if N >= 2:
        out.append((N - 1, N - 1, N if N % 2 else N + 1, 1))
        out.append((max(1, N - 20), -1, max(1, N - 20) + 5, 0))
    if N >= 3:
        out.append((N - 2, N - 1, N, 0))
    return out


@functools.lru_cache(None)
def _exact_case(M, N, K):
    rng = np.random.default_rng(M * 7919 + N * 31 + K)
    a = gk.exact_operands(rng, M, K)
    b = gk.exact_operands(rng, N, K)
    S = gk.pair_exact(*a, *b)
    return a, b, S, gk.exact_c0(rng, M, N)


def _want(S, alpha, c0):
    v = np.float32(alpha) * S.astype(np.float32)
    return v if c0 is None else (c0 + v).astype(np.float32)


def _run_exact(engine, M, N, K, a_mn, b_mn, acc, layouts=None):
    pair, lean, det, k_splits = ENGINES[engine]
    (a_hi, a_lo), (b_hi, b_lo), S, c0 = _exact_case(M, N, K)
    A, B = _operand(a_hi, a_lo, a_mn), _operand(b_hi, b_lo, b_mn)
    d = gk.dispatch(M, N, K, k_splits, _sms(), pair=pair, lean=lean, det=det, a_mn=a_mn, b_mn=b_mn)
    # a general alpha where each element has one writer that stores it once: exactly fl32(alpha S); otherwise a power of two
    alpha = (0.3 if not d['partial'] else 0.5) if not acc else (-2.0 if d['partial'] else -0.7)
    for n_store, special, ldc, off in (layouts or _layouts(N)):
        out = Out(M, ldc, n_store, off, c0 if acc else None, c0[:, special] if (acc and special >= 0) else None)
        with Config(pair, lean):
            _gemm(det, M, N, K, alpha, A, a_mn, B, b_mn, out, n_store, special, k_splits, acc)
        want = _want(S, alpha, c0 if acc else None)
        name = '%s %dx%dx%d maj %d%d acc %d layout %s' % (engine, M, N, K, a_mn, b_mn, acc, (n_store, special, ldc, off))
        out.check(name, want, want[:, special] if special >= 0 else None)
    return d


@pytest.mark.parametrize('acc', [0, 1])
@pytest.mark.parametrize('a_mn,b_mn', [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize('engine', list(ENGINES))
def test_every_engine_bit_exact(engine, a_mn, b_mn, acc):
    for M, N, K in RAGGED:
        _run_exact(engine, M, N, K, a_mn, b_mn, acc)


def test_engine_shapes_reach_their_engines():
    """The dispatch restatement says the ragged table reaches each tile engine, and where the edge cases it exists for occur."""
    sms = _sms()
    seen = set()
    for engine, (pair, lean, det, k) in ENGINES.items():
        for M, N, K in RAGGED:
            bn, stages, pr, _, bk = gk.dispatch(M, N, K, k, sms, pair=pair, lean=lean, det=det)['kernel']
            seen.add((bn, stages, pr, bk))
    assert {(128, 2, 0, 64), (64, 3, 0, 64), (128, 4, 0, 32), (128, 2, 1, 64), (64, 2, 0, 64)} <= seen
    # an odd number of 128-row tiles for the pairs, stream-K tiles cut between CTAs, k_splits above the k-blocks
    assert any(-(-M // 128) % 2 == 1 and M > 128 for M, _, _ in RAGGED)
    assert any(gk.sk_split_tiles(gk.dispatch(M, N, K, -1, sms)) for M, N, K in RAGGED)
    assert gk.dispatch(129, 501, 700, 1000, sms)['k_splits'] == 11


# uniform split-K: 8 k-blocks in 7 requested splits become 4; with more work items than SMs some CTA's second item is one the
# unrounded 7 would have left empty (a stale accumulator)
ROUNDING = [(640, 1281, 449), (1000, 700, 512)]


@pytest.mark.parametrize('a_mn,b_mn', [(0, 0), (1, 1)])
def test_split_k_rounding_leaves_no_empty_split(a_mn, b_mn):
    for M, N, K in ROUNDING:
        d = gk.dispatch(M, N, K, 7, _sms(), a_mn=a_mn, b_mn=b_mn)
        assert d['k_splits'] == 4 and d['tiles'] * 7 > _sms()
        for acc in (0, 1):
            _run_exact('split7', M, N, K, a_mn, b_mn, acc, layouts=[(N, -1, N, 0)])


# deterministic stream-K: shapes with a CTA whose range starts at a tile's first k-block and ends inside it (slot 0 with u_c == T0),
# and CTAs with two partial segments (slots 0 and 1)
DET_SK = [(1000, 1001, 33), (800, 500, 2000), (300, 700, 2000), (129, 501, 700), (10000, 501, 64)]


@pytest.mark.parametrize('a_mn,b_mn', [(0, 1), (1, 1), (0, 0)])
def test_det_stream_k_workspace_slots(a_mn, b_mn):
    sms = _sms()
    ds = [gk.dispatch(M, N, K, -1, sms, det=True) for M, N, K in DET_SK]
    assert all(d['fixup'] for d in ds)
    assert any(gk.sk_aligned_partial(d) for d in ds) and any(gk.sk_two_partials(d) for d in ds)
    for M, N, K in DET_SK:
        for acc in (0, 1):
            _run_exact('det_stream_k', M, N, K, a_mn, b_mn, acc, layouts=[(N - 1, N - 1, N + 1, 1)])


def test_row_views():
    """dE2[r0:] style outputs and E[r0:] style operands: pointers into the middle of larger buffers."""
    M, N, K, r0 = 700, 300, 256, 256
    (a_hi, a_lo), (b_hi, b_lo), S, c0 = _exact_case(M, N, K)
    A, B = _operand(a_hi, a_lo, 0), _operand(b_hi, b_lo, 1)
    n = M - r0
    Ablk = (A[0][r0:], A[1][r0:], A[2])
    for engine in ('auto', 'stream_k', 'det'):
        pair, lean, det, k = ENGINES[engine]
        out = Out(M, N, N, 0, c0)
        view = Out.__new__(Out)
        view.M, view.ldc, view.n_store, view.off, view.buf, view.sp = n, N, N, r0 * N, out.buf, out.sp
        _gemm(det, n, N, K, 1.0, Ablk, 0, B, 1, view, N, -1, k, 1)
        want = c0.copy()
        want[r0:] = _want(S[r0:], 1.0, c0[r0:])
        out.check('row view ' + engine, want)


@functools.lru_cache(None)
def _sym_case(M, N):
    rng = np.random.default_rng(M * 13 + N)
    g = gk.exact_operands(rng, M, 2 * M)
    g = (g[0][:, :M], g[1][:, :M])
    bt = gk.exact_operands(rng, N, 2 * M)
    bt = (bt[0][:, :M], bt[1][:, :M])                      # B^T [N x M]
    S = gk.pair_exact(g[0], g[1], *bt) + gk.pair_exact(g[0].T, g[1].T, *bt)
    return g, bt, S, gk.exact_c0(rng, M, N)


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('M,N', [(1, 1), (65, 17), (129, 65), (301, 129), (800, 500)])
def test_sym_bit_exact(M, N, det):
    (g_hi, g_lo), (bt_hi, bt_lo), S, c0 = _sym_case(M, N)
    G = _operand(g_hi, g_lo, 0)
    Bm = _operand(bt_hi, bt_lo, 1)       # stored [M x ldb], n contiguous
    for acc, alpha in ((0, 0.5), (1, -2.0)):
        out = Out(M, N + 3, N, 1, c0 if acc else None)
        args = (M, N, alpha, G[0].data_ptr(), G[1].data_ptr(), G[2], Bm[0].data_ptr(), Bm[1].data_ptr(), Bm[2], out.ptr, out.ldc, acc)
        if det:
            ws = _det_ws()
            ws.fill_(float('nan'))
            _call('dae_gemm_sym_bf16x3_det', *args, ws.data_ptr(), ws.numel() * 4, _st())
        else:
            _call('dae_gemm_sym_bf16x3', *args, _st())
        torch.cuda.synchronize()
        out.check('sym %dx%d det %d acc %d' % (M, N, det, acc), _want(S, alpha, c0 if acc else None))


# ---------------------------------------------------------------------------------------------------------------------------
# (b) the step's shapes against the fp64 bound, operands scaled over 2^+-20
# ---------------------------------------------------------------------------------------------------------------------------
WORST = {}


def _scaled_pair(rows, cols, seed, spread_rows, spread_cols):
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = 2.0 ** torch.randint(-spread_rows, spread_rows + 1, (rows,), device=DEV, generator=g).float()
    c = 2.0 ** torch.randint(-spread_cols, spread_cols + 1, (cols,), device=DEV, generator=g).float()
    x = torch.randn(rows, cols, device=DEV, generator=g) * r[:, None] * c[None, :]
    hi = x.bfloat16()
    lo = (x - hi.float()).bfloat16()
    return hi, lo


def _stored(hi, lo, mn, ld_extra=8):
    """[rows x K] pair -> device buffers in the given majorness, padding NaN."""
    out = []
    for t in (hi, lo):
        t = t.t() if mn else t
        buf = torch.full((t.shape[0] + 1, t.shape[1] + ld_extra - t.shape[1] % 8), float('nan'), dtype=torch.bfloat16, device=DEV)
        buf[:t.shape[0], :t.shape[1]] = t
        out.append(buf)
    return out[0], out[1], out[0].shape[1]


def _bound_check(name, got, A, B, K, alpha, c0=None):
    Ad, Bd = A.double(), B.double()
    want = alpha * (Ad @ Bd.t())
    bound = gk.pair_c(K) * abs(alpha) * (Ad.abs() @ Bd.abs().t())
    if c0 is not None:
        want = want + c0.double()
        bound = bound + gk.U * (c0.double().abs() + want.abs())
    err = (got.double() - want).abs()
    ratio = float((err / (bound + 1e-300)).max())
    WORST[name] = max(WORST.get(name, 0.0), ratio)
    assert bool((err <= bound).all()), '%s: worst err / bound %.3g' % (name, ratio)


# (name, M, N, K, a_mn, b_mn, n_store, special): dE = dZ.W, [dW | dbv] = dZ^T.[E | 1] at C2 (B 800, F 10 000, H 500), C4 (F 50 000,
# H 1 000) and C5 (2 400 stacked rows)
STEP_SHAPES = [
    ('C2 dE', 800, 500, 10000, 0, 1, 500, -1), ('C2 dW', 10000, 501, 800, 1, 1, 500, 500),
    ('C4 dE', 800, 1000, 50000, 0, 1, 1000, -1), ('C4 dW', 50000, 1001, 800, 1, 1, 1000, 1000),
    ('C5 dE', 2400, 500, 10000, 0, 1, 500, -1), ('C5 dW', 10000, 501, 2400, 1, 1, 500, 500),
]


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('shape', STEP_SHAPES, ids=[s[0] for s in STEP_SHAPES])
def test_step_shapes_within_fp64_bound(shape, det):
    name, M, N, K, a_mn, b_mn, n_store, special = shape
    ahl = _scaled_pair(M, K, M + K, 20, 20)
    bhl = _scaled_pair(N, K, N + K + 1, 20, 20)
    A, B = _stored(*ahl, a_mn), _stored(*bhl, b_mn)
    Ap = ahl[0].double() + ahl[1].double()
    Bp = bhl[0].double() + bhl[1].double()
    C = torch.full((M, n_store), float('nan'), device=DEV)
    sp = torch.full((M,), float('nan'), device=DEV)
    args = (M, N, K, 1.0, A[0].data_ptr(), A[1].data_ptr(), A[2], a_mn, B[0].data_ptr(), B[1].data_ptr(), B[2], b_mn, C.data_ptr(), n_store,
            n_store, special, sp.data_ptr() if special >= 0 else None, -1, 0)
    if det:
        ws = _det_ws()
        _call('dae_gemm_bf16x3_det', *args, ws.data_ptr(), ws.numel() * 4, _st())
    else:
        _call('dae_gemm_bf16x3', *args, _st())
    torch.cuda.synchronize()
    full = torch.cat([C, sp[:, None]], 1) if special >= 0 else C
    _bound_check('%s%s' % (name, ' det' if det else ''), full, Ap, Bp, K, 1.0)
    del Ap, Bp, full


# ---------------------------------------------------------------------------------------------------------------------------
# (c) every GEMM call of real training steps, against the inputs it was given
# ---------------------------------------------------------------------------------------------------------------------------
GEMM_EXPORTS = ('dae_gemm_bf16x3', 'dae_gemm_bf16x3_det', 'dae_gemm_sym_bf16x3', 'dae_gemm_sym_bf16x3_det', 'dae_sgemm')


def _pair_dev(p_hi, p_lo, rows, ld):
    hi = device_copy(p_hi, (rows, ld), '<i2').view(torch.bfloat16).double()
    lo = device_copy(p_lo, (rows, ld), '<i2').view(torch.bfloat16).double()
    return hi + lo


class GemmRecorder:
    """Stands in for engine.call: every GEMM export call runs between two device synchronisations, and its output is checked
    against the fp64 reference of the inputs (and the C it accumulated onto) it was given."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __call__(self, name, *a):
        if name not in GEMM_EXPORTS:
            return self.real(name, *a)
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('GemmRecorder synchronises the device around every GEMM: it cannot run under stream capture')
        torch.cuda.synchronize()
        if name == 'dae_sgemm':
            self._sgemm(name, a)
        elif name.startswith('dae_gemm_sym'):
            self._sym(name, a)
        else:
            self._gemm(name, a)
        self.calls.append((name, a[:3]))

    def _gemm(self, name, a):
        M, N, K, alpha = a[0], a[1], a[2], a[3]
        a_mn, b_mn, ldc, n_store, special_col, sp, acc = a[7], a[11], a[13], a[14], a[15], a[16], a[18]
        ns = N if (n_store <= 0 or n_store > N) else n_store
        A = _pair_dev(a[4], a[5], K if a_mn else M, a[6])
        A = (A.t() if a_mn else A)[:M, :K]
        B = _pair_dev(a[8], a[9], K if b_mn else N, a[10])
        B = (B.t() if b_mn else B)[:N, :K]
        c0 = device_copy(a[12], (M, ldc), '<f4')[:, :ns] if acc else None
        s0 = device_copy(sp, (M,), '<f4') if (acc and sp) else None
        self.real(name, *a)
        torch.cuda.synchronize()
        C = device_copy(a[12], (M, ldc), '<f4')[:, :ns]
        cols = list(range(ns))
        if sp:
            C = torch.cat([C, device_copy(sp, (M,), '<f4')[:, None]], 1)
            cols.append(special_col)
            if acc:
                c0 = torch.cat([c0, s0[:, None]], 1)
        _bound_check('step %s %dx%dx%d' % (name, M, N, K), C, A, B[cols], K, float(np.float32(alpha)), c0)

    def _sym(self, name, a):
        M, N, alpha, ldg, ldb, ldc, acc = a[0], a[1], a[2], a[5], a[8], a[10], a[11]
        G = _pair_dev(a[3], a[4], M, ldg)[:, :M]
        Bm = _pair_dev(a[6], a[7], M, ldb)[:, :N]
        c0 = device_copy(a[9], (M, ldc), '<f4')[:, :N] if acc else None
        self.real(name, *a)
        torch.cuda.synchronize()
        C = device_copy(a[9], (M, ldc), '<f4')[:, :N]
        _bound_check('step %s %dx%d' % (name, M, N), C, torch.cat([G, G.t()], 1), torch.cat([Bm, Bm], 0).t(), 2 * M,
                     float(np.float32(alpha)), c0)

    def _sgemm(self, name, a):
        M, N, K, alpha, sam, sak, sbn, sbk, beta, ldc = a[0], a[1], a[2], a[3], a[5], a[6], a[8], a[9], a[10], a[12]
        A = device_copy(a[4], ((M - 1) * sam + (K - 1) * sak + 1,), '<f4').as_strided((M, K), (sam, sak)).double()
        B = device_copy(a[7], ((N - 1) * sbn + (K - 1) * sbk + 1,), '<f4').as_strided((N, K), (sbn, sbk)).double()
        c0 = device_copy(a[11], (M, ldc), '<f4')[:, :N].double() if beta != 0.0 else None
        self.real(name, *a)
        torch.cuda.synchronize()
        C = device_copy(a[11], (M, ldc), '<f4')[:, :N].double()
        _sgemm_check('step %s %dx%dx%d' % (name, M, N, K), C, A, B, alpha, beta, c0)


def _sgemm_check(name, C, A, B, alpha, beta, c0):
    M, K = A.shape
    a, b = float(np.float32(alpha)), float(np.float32(beta))
    want = a * (A @ B.t())
    scale = abs(a) * (A.abs() @ B.abs().t())
    if b != 0.0:
        want = want + b * c0
        scale = scale + abs(b) * c0.abs()
    bound = gk.sgemm_c(M, B.shape[0], K, _sms()) * scale + 1e-37
    err = (C - want).abs()
    ratio = float((err / bound).max())
    WORST[name] = max(WORST.get(name, 0.0), ratio)
    assert bool((err <= bound).all()), '%s: worst err / bound %.3g' % (name, ratio)


def _engine(strategy, det=False, gemm='tc', block=None, loss='cross_entropy', F=10000, H=500, B=800):
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    import scipy.sparse as sp
    n = 3 * B if strategy == 'explicit' else B
    x = make_sparse(n, F, 100, 'tfidf', seed=1)
    if strategy == 'explicit':
        x = sp.vstack([x[:B], x[:B], x[B:2 * B]]).tocsr()
    kw = dict(triplet_strategy=strategy, gemm=gemm, device=DEV, deterministic=det, loss_func=loss, dec_act_func='sigmoid',
              enc_act_func='sigmoid', alpha=1.0)
    if block:
        kw['mining_block_rows'] = block
    eng = TrainEngine(F, H, **kw)
    eng.set_parameters(xavier(F, H, 2) * 3)
    labels = None if strategy == 'explicit' else torch.from_numpy(make_labels(n, 4, seed=1)).to(DEV)
    eng.set_data(DeviceCSR(x, eng.device), None, labels)
    eng.corrupt_masking(0.3, seed=5, epoch=0)
    return eng


# (strategy, deterministic, gemm, mining_block_rows, loss)
STEP_CONFIGS = [(s, d, 'tc', None, 'cross_entropy') for s in ('none', 'batch_all', 'batch_hard', 'explicit') for d in (False, True)]
STEP_CONFIGS += [('batch_all', False, 'tc', 256, 'cross_entropy'), ('batch_hard', False, 'tc', 256, 'cross_entropy'),
                 ('batch_all', False, 'tc', None, 'cosine_proximity'), ('batch_all', False, 'ffma', None, 'cross_entropy'),
                 ('explicit', False, 'ffma', None, 'cross_entropy')]


def _expected_tags(strategy, det, gemm, block, loss):
    if gemm == 'ffma':
        t = {('dae_sgemm', 'gemm_decode_fwd'), ('dae_sgemm', 'gemm_decode_dW'), ('dae_sgemm', 'gemm_decode_dE')}
        if strategy in ('batch_all', 'batch_hard'):
            t |= {('dae_sgemm', 'gemm_gram'), ('dae_sgemm', 'gemm_dE_tri')}
        return t
    big = 'dae_gemm_bf16x3_det' if det else 'dae_gemm_bf16x3'
    t = {(big, 'gemm_decode_dW'), (big, 'gemm_decode_dE')}
    if loss == 'cosine_proximity':
        t.add(('dae_gemm_bf16x3', 'gemm_decode_fwd'))
    if strategy in ('batch_all', 'batch_hard'):
        t.add(('dae_gemm_bf16x3', 'gemm_gram'))
        if strategy == 'batch_all' and block is None:
            t.add(('dae_gemm_sym_bf16x3_det' if det else 'dae_gemm_sym_bf16x3', 'gemm_dE_tri'))
        else:
            t.add(('dae_gemm_bf16x3', 'gemm_dE_tri'))
    return t


@pytest.mark.parametrize('fork', [True, False])
@pytest.mark.parametrize('cfg', STEP_CONFIGS, ids=['-'.join(str(v) for v in c) for c in STEP_CONFIGS])
def test_every_gemm_of_a_training_step(cfg, fork, monkeypatch):
    from dae_rnn_news_recommendation_b200 import engine as engine_mod
    strategy, det, gemm, block, loss = cfg
    eng = _engine(strategy, det, gemm, block, loss)
    eng.fork_branches = fork
    rec = GemmRecorder(engine_mod.call)
    monkeypatch.setattr(engine_mod, 'call', rec)
    tags = []
    real_k = eng._k

    def k(name, *a, **kw):
        if name in GEMM_EXPORTS:
            tags.append((name, kw.get('tag')))
        return real_k(name, *a, **kw)

    eng._k = k
    for s in range(2):     # the second step runs on the updated parameters and the refreshed W split
        if strategy == 'explicit':
            eng.step_explicit(None, 0, 800, 800)
        else:
            eng.step(None, 0, 800)
        torch.cuda.synchronize()
        assert set(tags) == _expected_tags(*cfg), sorted(set(tags))
        tags.clear()
    assert rec.calls


def test_recorder_refuses_stream_capture(monkeypatch):
    seen = []
    rec = GemmRecorder(lambda *a: seen.append(a[0]))
    monkeypatch.setattr(torch.cuda, 'is_current_stream_capturing', lambda: True)
    for name in GEMM_EXPORTS:
        with pytest.raises(RuntimeError, match='stream capture'):
            rec(name, 1, 1, 1, 1.0, 0, 1, 1, 0, 1, 1, 0.0, 0, 1, None)
    rec('dae_split_bf16')       # anything else goes straight through
    assert seen == ['dae_split_bf16'] and rec.calls == []


# ---------------------------------------------------------------------------------------------------------------------------
# (d) dae_sgemm
# ---------------------------------------------------------------------------------------------------------------------------
SGEMM_STRIDES = ['nt', 'nn', 'tn', 'tt']   # A row-major or transposed x B row-major or transposed (stride swaps)


@pytest.mark.parametrize('beta', [0.0, 0.75])
@pytest.mark.parametrize('strides', SGEMM_STRIDES)
@pytest.mark.parametrize('M,N,K', [(800, 500, 10000), (1, 17, 300), (129, 65, 255), (301, 1001, 33), (1000, 700, 64), (65, 129, 4000)])
def test_sgemm(M, N, K, strides, beta):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    r = 2.0 ** torch.randint(-20, 21, (M,), device=DEV, generator=g).float()
    A = torch.randn(M, K, device=DEV, generator=g) * r[:, None]
    B = torch.randn(N, K, device=DEV, generator=g)
    Ab = A if strides[0] == 'n' else A.t().contiguous()
    Bb = B if strides[1] == 'n' else B.t().contiguous()
    sam, sak = (K, 1) if strides[0] == 'n' else (1, M)
    sbn, sbk = (K, 1) if strides[1] == 'n' else (1, N)
    ldc = N + 3
    C = torch.full((M + 1, ldc), float('nan') if beta == 0.0 else 0.0, device=DEV)
    if beta != 0.0:
        C[:M, :N] = torch.randn(M, N, device=DEV, generator=g)
    C[:, N:] = float(SENT)
    C[M] = float(SENT)
    c0 = C[:M, :N].double().clone()
    _call('dae_sgemm', M, N, K, 1.5, Ab.data_ptr(), sam, sak, Bb.data_ptr(), sbn, sbk, beta, C.data_ptr(), ldc, _st())
    torch.cuda.synchronize()
    splits, _ = gk.sgemm_splits(M, N, K, _sms())
    _sgemm_check('sgemm %s splits %d' % (strides, splits), C[:M, :N].double(), A.double(), B.double(), 1.5, beta,
                 c0 if beta != 0.0 else None)
    assert bool((C[:, N:] == float(SENT)).all()) and bool((C[M] == float(SENT)).all())


def test_sgemm_table_reaches_both_branches():
    sms = _sms()
    br = {gk.sgemm_splits(M, N, K, sms)[0] > 1 for M, N, K in [(800, 500, 10000), (1, 17, 300), (129, 65, 255), (65, 129, 4000)]}
    assert br == {True, False}


# ---------------------------------------------------------------------------------------------------------------------------
# (e) which engine ran
# ---------------------------------------------------------------------------------------------------------------------------
PROFILE_TABLE = [   # (engine, M, N, K, a_mn, b_mn)
    ('auto', 1345, 833, 129, 0, 0), ('auto', 800, 800, 500, 0, 0), ('stream_k', 800, 500, 10000, 0, 1),
    ('stream_k', 10000, 501, 800, 1, 1), ('split7', 300, 200, 4000, 1, 0), ('pair', 301, 258, 64, 0, 0),
    ('lean', 301, 258, 64, 0, 1), ('det', 800, 800, 500, 0, 0), ('det_stream_k', 800, 500, 10000, 0, 1),
]


def test_profiler_sees_the_predicted_kernels():
    from torch.profiler import ProfilerActivity, profile
    launched, predicted = [], []
    for engine, M, N, K, a_mn, b_mn in PROFILE_TABLE:
        pair, lean, det, k = ENGINES[engine]
        d = gk.dispatch(M, N, K, k, _sms(), pair=pair, lean=lean, det=det, a_mn=a_mn, b_mn=b_mn)
        (a_hi, a_lo), (b_hi, b_lo) = gk.exact_operands(np.random.default_rng(0), M, K), gk.exact_operands(np.random.default_rng(1), N, K)
        A, B = _operand(a_hi, a_lo, a_mn), _operand(b_hi, b_lo, b_mn)
        out = Out(M, N, N)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with Config(pair, lean):
                _gemm(det, M, N, K, 0.5, A, a_mn, B, b_mn, out, N, -1, k, 0)
        names = [e.name for e in prof.events() if e.device_type.name == 'CUDA']
        got = [gk.kernel_of(n) for n in names if gk.kernel_of(n)]
        fix = [n for n in names if gk.FIXUP_RE.search(n)]
        launched.append((engine, got, len(fix)))
        predicted.append((engine, [d['kernel']], 1 if d['fixup'] else 0))
    print('\nlaunched:', launched)
    assert launched == predicted


def test_zz_report_worst_ratios():
    """Prints the worst err / bound per shape and engine seen by this module's bound checks (run last)."""
    for k in sorted(WORST):
        print('%-50s %.3f' % (k, WORST[k]))
