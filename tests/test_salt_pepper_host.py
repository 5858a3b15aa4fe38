"""Host-side parts of the device salt-and-pepper noise (dae_salt_pepper_csr): utils.salt_and_pepper_draws plus the oracle's application
of the draws reproduce utils.salt_and_pepper_noise array for array, the oracle's Philox matches Random123's known answers, the capacity
bound holds, and the export checks its arguments before any CUDA call."""
import numpy as np
import pytest

from salt_pepper_oracle import apply_draws, capacity, cases, philox4x32_10, philox_draws, value_range

FAKE = 1 << 20   # 16-byte aligned non-null stand-in for a device pointer: every call below fails validation before using it


def test_philox_known_answers():
    c = philox4x32_10((0, 0, 0, 0), (0, 0))
    assert [int(x) for x in c] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    c = philox4x32_10((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0))
    assert [int(x) for x in c] == [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def test_philox_draw_layout():
    """Draw j of row r: words (c0, c1) of counter (j // 2, r, epoch) when j is even, (c2, c3) when odd."""
    F, v, seed, epoch = 1000, 7, (5 << 32) | 3, (2 << 32) | 9
    d = philox_draws([4, 11], F, v, seed, epoch)
    for k, r in enumerate([4, 11]):
        for j in range(v):
            c = philox4x32_10((j // 2, r, epoch & 0xFFFFFFFF, epoch >> 32), (seed & 0xFFFFFFFF, seed >> 32))
            a, b = (c[0], c[1]) if j % 2 == 0 else (c[2], c[3])
            assert int(d[k, j]) & 0x7FFFFFFF == (int(a) * F) >> 32
            assert int(d[k, j]) >> 31 == int(b) >> 31


@pytest.mark.parametrize('name,X,v', cases(), ids=[c[0] for c in cases()])
def test_draws_and_oracle_equal_host_function(name, X, v):
    from dae_rnn_news_recommendation_b200.autoencoder import utils
    np.random.seed(1234)
    want = utils.salt_and_pepper_noise(X, v)
    np.random.seed(1234)
    draws = utils.salt_and_pepper_draws(X, v)
    assert draws.dtype == np.uint32 and draws.shape == (X.shape[0], v)
    after = np.random.random()                                   # the draws consumed exactly the host function's share of the stream
    np.random.seed(1234)
    utils.salt_and_pepper_noise(X, v)
    assert np.random.random() == after
    lo, hi = value_range(X)
    if name.startswith('full'):
        assert lo != 0 and hi != 0
    ip, ix, dat = apply_draws(X, draws, lo, hi)
    assert want.has_sorted_indices
    np.testing.assert_array_equal(ip, want.indptr)
    np.testing.assert_array_equal(ix, want.indices)
    np.testing.assert_array_equal(dat, want.data.astype(np.float32))
    per_row = np.diff(ip)
    assert (per_row <= np.minimum(np.diff(X.indptr) + v, X.shape[1])).all()
    assert ip[-1] <= capacity(X, v)
    if name == 'small_F_large_v':   # repeated columns with opposite coins: the last draw decides
        cols, coin = draws & 0x7FFFFFFF, draws >> 31
        assert any(len(set(coin[r][cols[r] == m])) == 2 for r in range(X.shape[0]) for m in range(X.shape[1]))


def test_explicit_zeros_survive_untouched():
    """An explicit stored zero no draw touches stays stored, as tolil / tocsr keep it."""
    from dae_rnn_news_recommendation_b200.autoencoder import utils
    name, X, v = [c for c in cases() if c[0] == 'explicit_zeros_empty_rows'][0]
    np.random.seed(5)
    draws = utils.salt_and_pepper_draws(X, v)
    lo, hi = value_range(X)
    ip, ix, dat = apply_draws(X, draws, lo, hi)
    kept_zero = 0
    for r in range(X.shape[0]):
        touched = set((draws[r] & 0x7FFFFFFF).tolist())
        for e in range(X.indptr[r], X.indptr[r + 1]):
            if X.data[e] == 0 and X.indices[e] not in touched:
                assert X.indices[e] in ix[ip[r]:ip[r + 1]]
                kept_zero += 1
    assert kept_zero > 0


def _call(indptr=FAKE, indices=FAKE, values=FAKE, row0=0, n=10, F=100, v=30, draws=None, out_ptr=FAKE, out_ind=FAKE, out_val=FAKE, cap=1000,
          overflow=FAKE, ws=FAKE, ws_bytes=1 << 20):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_salt_pepper_csr', indptr, indices, values, row0, n, F, v, 0.0, 1.0, draws, 0, 0, out_ptr, out_ind, out_val, cap, overflow,
               ws, ws_bytes, None)


def test_export_argument_checks():
    from dae_rnn_news_recommendation_b200 import _cabi
    for kw in (dict(indptr=None), dict(indices=None), dict(values=None), dict(out_ptr=None), dict(out_ind=None), dict(out_val=None),
               dict(overflow=None)):
        with pytest.raises(_cabi.DaeError, match='null pointer'):
            _call(**kw)
    for kw, msg in ((dict(row0=-1), 'bad rows'), (dict(n=-1), 'bad rows'), (dict(F=0), 'F = 0'), (dict(F=1 << 30), 'F = '),
                    (dict(v=-1), 'v = -1'), (dict(v=1 << 30), 'v = '), (dict(cap=-1), 'negative cap'), (dict(ws=None), 'workspace'),
                    (dict(ws_bytes=8), 'workspace')):
        with pytest.raises(_cabi.DaeError, match=msg):
            _call(**kw)
    need = _cabi.query('dae_salt_pepper_workspace', 10, ctype=__import__('ctypes').c_size_t)
    assert need >= 2 * 10 * 8
    with pytest.raises(_cabi.DaeError, match='workspace'):
        _call(ws_bytes=need - 1)
    with pytest.raises(_cabi.DaeError, match='dae_salt_pepper_workspace'):
        _cabi.query('dae_salt_pepper_workspace', -1, ctype=__import__('ctypes').c_size_t)


def test_value_range_is_global_with_implicit_zeros():
    import scipy.sparse as sp
    X = sp.csr_matrix(np.array([[0.5, 0.0], [0.7, 0.9]]))
    assert value_range(X) == (0.0, 0.9)
    X = sp.csr_matrix(np.array([[0.5, 0.6], [0.7, 0.9]]))
    assert value_range(X) == (0.5, 0.9)
