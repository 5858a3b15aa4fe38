"""CPU checks of tests/gemm_kernel_oracle.py (the exact operands really are exact, the bound covers a float32 emulation of the
kernel's arithmetic, the dispatch restatement gives the tile counts the engine states) and the GEMM exports' argument checks through
the C ABI, which need no GPU."""
import numpy as np
import pytest

import gemm_kernel_oracle as gk
from mining_kernel_oracle import bf16_split


@pytest.mark.parametrize('K', [1, 31, 33, 65, 800, 4000, 10000])
def test_exact_operands_sum_exactly_in_any_order(K):
    rng = np.random.default_rng(K)
    a_hi, a_lo = gk.exact_operands(rng, 24, K)
    b_hi, b_lo = gk.exact_operands(rng, 1, K)
    want = gk.pair_exact(a_hi, a_lo, b_hi, b_lo)[:, 0]
    ah, al, bh, bl = (gk.bf16_value(x) for x in (a_hi, a_lo, b_hi, b_lo))
    terms = np.concatenate([ah * bh, ah * bl, al * bh], axis=1)      # every product is exact in fp64 and in fp32
    assert np.array_equal(terms.astype(np.float32).astype(np.float64), terms)
    assert float(np.abs(terms).sum(1).max()) <= 2.0 ** 15
    for order, got in zip(('forward', 'reverse', 'blocked'), gk.fl32_sum_orders(terms)):
        assert np.array_equal(got.astype(np.float64), want), order
    # the kernel's own grouping (three products per 16-deep step) is one more order
    assert np.array_equal(gk.emulate_bf16x3(a_hi, a_lo, b_hi, b_lo)[:, 0].astype(np.float64), want)
    # alpha a power of two and C0 on the grid keep C0 + alpha S exact
    c0 = gk.exact_c0(rng, 24, 1)[:, 0].astype(np.float64)
    for alpha in (0.5, -2.0, 0.25):
        v = c0 + alpha * want
        assert np.array_equal(v.astype(np.float32).astype(np.float64), v)


def test_exact_h_keeps_partial_sums_below_2pow15():
    for K in (1, 16, 64, 500, 800, 4000, 10000, 10922):
        h = gk.exact_h(K)
        assert K * (h * h + 2 * h) <= 2 ** 15 and h <= 64
    with pytest.raises(AssertionError):
        gk.exact_h(11000)


@pytest.mark.parametrize('M,N,K', [(32, 40, 16), (17, 9, 700), (8, 33, 2000)])
def test_bf16x3_emulation_within_half_the_bound(M, N, K):
    rng = np.random.default_rng(M * N + K)
    A = gk.scaled_operand(rng, M, K, 20, 0)
    B = gk.scaled_operand(rng, N, K, 20, 0)
    # spread over k as well: a few columns of each operand dominate the rest by 2^20
    A[:, ::7] *= np.float32(2.0 ** 10)
    B[:, 3::11] *= np.float32(2.0 ** -10)
    (a_hi, a_lo), (b_hi, b_lo) = bf16_split(A), bf16_split(B)
    want, bound = gk.pair_bound(a_hi, a_lo, b_hi, b_lo, K)
    got = gk.emulate_bf16x3(a_hi, a_lo, b_hi, b_lo)
    assert gk.worst_ratio(got, want, bound) <= 0.5
    # against the fp32 values themselves the representation term comes back: gemm_c
    import torch
    w2, b2 = gk.gemm(torch.from_numpy(A), torch.from_numpy(B))
    assert gk.worst_ratio(got, w2, b2) <= 0.5
    assert gk.pair_c(K) < gk.gemm_c(K)


def test_dispatch_matches_the_step_shapes_on_132_sms():
    # C2 (F = 10 000, H = 500, B = 800): dE = dZ.W (28 tiles) and [dW | dbv] = dZ^T.[E | 1] (316 tiles), both stream-K
    dE = gk.dispatch(800, 500, 10000, -1, 132, a_mn=0, b_mn=1)
    assert dE['tiles'] == 28 and dE['stream_k'] and dE['kernel'] == (128, 4, 0, 2, 32)
    dW = gk.dispatch(10000, 501, 800, -1, 132, a_mn=1, b_mn=1)
    assert dW['tiles'] == 316 and dW['stream_k'] and dW['kernel'] == (128, 4, 0, 3, 32)
    assert gk.sk_split_tiles(dE) and gk.sk_split_tiles(dW)
    # the C2 Gram: 49 tiles at 128 x 128 and 91 at 128 x 64, one wave either way: 128 x 64 with the 3-stage ring
    gram = gk.dispatch(800, 800, 500, 1, 132)
    assert gram['kernel'] == (64, 3, 0, 0, 64) and gram['tiles'] == 91
    assert gk.dispatch(800, 800, 500, 1, 132, lean=True)['kernel'] == (64, 2, 0, 0, 64)
    assert gk.dispatch(800, 800, 500, 1, 132, pair=True)['kernel'][:3] == (128, 2, 1)
    # the deterministic twin: the same stream-K choice plus the fixup
    d = gk.dispatch(800, 500, 10000, -1, 132, det=True, a_mn=0, b_mn=1)
    assert d['kernel'] == dE['kernel'] and d['n_cta'] == dE['n_cta'] and d['fixup']
    assert not gk.dispatch(800, 500, 10000, 1, 132, det=True)['fixup']
    # whole waves: 132 tiles of 128 x 128 are not stream-K
    assert not gk.dispatch(128 * 12, 128 * 11, 640, -1, 132)['stream_k']


def test_dispatch_split_k_rounding():
    # 8 k-blocks in 7 splits would leave 3 empty: per = 2 -> 4 splits; more splits than k-blocks clamp to the k-blocks
    assert gk.dispatch(300, 200, 512, 7)['k_splits'] == 4
    assert gk.dispatch(300, 200, 449, 7)['k_splits'] == 4
    assert gk.dispatch(300, 200, 100, 9)['k_splits'] == 2
    assert gk.dispatch(300, 200, 4000, 7)['k_splits'] == 7
    assert gk.dispatch(300, 200, 4000, 0)['k_splits'] == 1


def test_stream_k_cuts():
    d = gk.dispatch(1000, 1001, 33, -1, 132)
    u = gk.sk_cuts(d)
    assert u[0] == 0 and u[-1] == d['tiles'] * d['kb'] and all(b >= a for a, b in zip(u, u[1:]))


def test_sgemm_splits():
    assert gk.sgemm_splits(800, 500, 10000, 132)[0] > 1          # 28 tiles, deep K: split-K
    assert gk.sgemm_splits(800, 500, 200, 132) == (1, 208)       # K < 256: one pass (the chunk is rounded up to 16)
    assert gk.sgemm_splits(10000, 500, 800, 132)[0] == 1         # 316 tiles fill the SMs
    s, kc = gk.sgemm_splits(100, 100, 1000, 132)
    assert (s - 1) * kc < 1000 <= s * kc


@pytest.mark.parametrize('M,N,K,beta', [(3, 5, 300, 0.0), (2, 7, 1000, 0.75), (4, 3, 40, -1.5)])
def test_sgemm_bound_covers_a_float32_emulation(M, N, K, beta):
    """dae_sgemm restated in float32: an FMA chain per k chunk, alpha times it, then beta C or (split-K) one add per split."""
    rng = np.random.default_rng(K)
    A = (rng.standard_normal((M, K)) * np.ldexp(1.0, rng.integers(-20, 21, (M, 1)))).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    alpha = np.float32(1.5)
    splits, kchunk = gk.sgemm_splits(M, N, K, 132)
    parts = []
    for s in range(splits):
        acc = np.zeros((M, N), np.float32)
        for k in range(s * kchunk, min(K, (s + 1) * kchunk)):
            acc = (acc.astype(np.float64) + A[:, k:k + 1].astype(np.float64) * B[:, k].astype(np.float64)).astype(np.float32)
        parts.append((alpha * acc).astype(np.float32))
    if splits == 1:
        got = parts[0] + (np.float32(beta) * C0 if beta != 0.0 else np.float32(0))
    else:
        got = (np.float32(beta) * C0).astype(np.float32)
        for p in parts:
            got = (got + p).astype(np.float32)
    want, bound = gk.sgemm_ref(A, B, alpha, beta, C0, 132)
    assert gk.worst_ratio(got, want, bound) <= 0.5


def test_kernel_name_parse():
    assert gk.kernel_of('void dae::gemm_bf16x3_kernel<128, 4, 0, 2, 32>(CUtensorMap, CUtensorMap)') == (128, 4, 0, 2, 32)
    assert gk.kernel_of('void dae::sk_fixup_kernel<128>(dae::GemmParams, int, int, int, int)') is None


# ---------------------------------------------------------------------------------------------------------------------------
# the C ABI without a GPU: the output contract of dae_gemm_bf16x3 / _det is checked before any device work
# ---------------------------------------------------------------------------------------------------------------------------
def _gemm_args(M, N, K, ldc, n_store, special_col, special_out):
    return (M, N, K, 1.0, 16, 32, 64, 0, 48, 64, 64, 0, 80, ldc, n_store, special_col, special_out, 1, 0)


BAD_OUTPUTS = [
    ((100, 501, 64, 499, 500, 500, 96), 'ldc'),             # ldc below n_store
    ((100, 501, 64, 400, 0, -1, None), 'ldc'),              # n_store 0 means N: ldc must cover N
    ((100, 501, 64, 500, 500, 499, 96), 'special_col'),     # the special column inside the stored ones
    ((100, 501, 64, 500, 500, 501, 96), 'special_col'),     # the special column past N
    ((100, 501, 64, 501, 0, 500, 96), 'special_col'),       # n_store = N leaves no room for it
    ((100, 501, 64, 500, 500, -1, 96), 'special_col'),
]


@pytest.mark.parametrize('args,what', BAD_OUTPUTS)
@pytest.mark.parametrize('det', [False, True])
def test_gemm_output_contract_rejected_before_device_work(args, what, det):
    from dae_rnn_news_recommendation_b200 import _cabi
    name = 'dae_gemm_bf16x3_det' if det else 'dae_gemm_bf16x3'
    a = _gemm_args(*args)
    a = a + ((112, 1 << 30, None) if det else (None,))
    with pytest.raises(_cabi.DaeError, match='%s: .*%s' % (name, what)):
        _cabi.call(name, *a)


# the argument checks of dae_decode_fused_bf16x3 / _det and dae_gemm_sym_bf16x3 / _det, each under the export's own name; the
# pointers are never dereferenced, since every case is rejected before any device work
def _decode_args(**bad):
    a = dict(Brows=100, F=500, K=64, e_hi=16, e_lo=32, lde=64, w_hi=48, w_lo=64, ldw=64, indptr=80, indices=96, values=112, rows=None,
             bv=128, dec_act=1, loss_func=0, weight=None, stats=144, dz_hi=160, dz_lo=176, ld_dz=512, row_loss_part=192, tile_ptr=208,
             prepared=1, stream=None)
    a.update(bad)
    return tuple(a.values())


BAD_DECODE = [
    (dict(e_hi=None), 'null pointer'),
    (dict(w_lo=None), 'null pointer'),
    (dict(indices=None), 'null pointer'),
    (dict(stats=None), 'null pointer'),
    (dict(dz_lo=None), 'null pointer'),
    (dict(row_loss_part=None), 'null pointer'),
    (dict(tile_ptr=None), 'null pointer'),
    (dict(loss_func=2), 'cosine loss uses the unfused path'),     # DAE_LOSS_COSINE
    (dict(loss_func=7), 'cosine loss uses the unfused path'),
    (dict(ld_dz=520), 'bad leading dimensions'),                   # covers F, not a multiple of 32
    (dict(ld_dz=480), 'bad leading dimensions'),                   # a multiple of 32 below F
    (dict(lde=60), 'bad leading dimensions'),
    (dict(ldw=68), 'bad leading dimensions'),
]


@pytest.mark.parametrize('bad,what', BAD_DECODE)
@pytest.mark.parametrize('det', [False, True])
def test_decode_fused_arguments_rejected_before_device_work(bad, what, det):
    from dae_rnn_news_recommendation_b200 import _cabi
    name = 'dae_decode_fused_bf16x3_det' if det else 'dae_decode_fused_bf16x3'
    with pytest.raises(_cabi.DaeError, match=r'%s failed \(-1\): %s: .*%s' % (name, name, what)):
        _cabi.call(name, *_decode_args(**bad))


def _sym_args(det, **bad):
    a = dict(M=100, N=500, alpha=1.0, g_hi=16, g_lo=32, ldg=104, b_hi=48, b_lo=64, ldb=504, C=80, ldc=500, accumulate=0)
    if det:
        a.update(workspace=96, workspace_bytes=1 << 40)
    a['stream'] = None
    a.update(bad)
    return tuple(a.values())


BAD_SYM = [
    (dict(g_hi=None), 'bad arguments'),
    (dict(b_lo=None), 'bad arguments'),
    (dict(C=None), 'bad arguments'),
    (dict(M=0), 'bad arguments'),
    (dict(ldg=100), 'multiples of 8 and cover'),       # covers M, not a multiple of 8
    (dict(ldg=96), 'multiples of 8 and cover'),        # below M
    (dict(ldb=502), 'multiples of 8 and cover'),
    (dict(ldb=496), 'multiples of 8 and cover'),       # below N
    (dict(g_lo=40), '16-byte aligned'),
    (dict(b_hi=56), '16-byte aligned'),
]
BAD_SYM_DET = [
    (dict(workspace_bytes=1), 'workspace of 1 bytes, need'),
    (dict(workspace=None), 'workspace of .* bytes, need'),
]


@pytest.mark.parametrize('bad,what,det', [(b, w, d) for b, w in BAD_SYM for d in (False, True)] + [(b, w, True) for b, w in BAD_SYM_DET])
def test_gemm_sym_arguments_rejected_before_device_work(bad, what, det):
    from dae_rnn_news_recommendation_b200 import _cabi
    name = 'dae_gemm_sym_bf16x3_det' if det else 'dae_gemm_sym_bf16x3'
    with pytest.raises(_cabi.DaeError, match=r'%s failed \(-1\): %s: .*%s' % (name, name, what)):
        _cabi.call(name, *_sym_args(det, **bad))
