"""Near-duplicate pairs without a GPU: duplicate_groups and pair_label_agreement against brute force, and the argument checks of
similar_pairs and of dae_similarity_pairs_bf16x3 / dae_csr_similarity_pairs, which all fail before any CUDA call."""
import ctypes
import itertools
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FAKE = 1 << 20   # 16-byte aligned non-null stand-in for a device pointer: every call below fails validation before using it


def _groups_brute(i, j, n):
    """Union-find, each row labelled by the smallest row of its component."""
    parent = list(range(n))

    def find(a):
        while parent[a] != a:
            a = parent[a]
        return a
    for a, b in zip(i, j):
        ra, rb = find(int(a)), find(int(b))
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    return np.array([find(a) for a in range(n)], dtype=np.int32)


@pytest.mark.parametrize('case', ['chain', 'star', 'singletons', 'duplicate_edges', 'empty', 'random'])
def test_duplicate_groups(case):
    from dae_rnn_news_recommendation_b200.helpers import duplicate_groups
    n = 12
    if case == 'chain':        # 9 - 7 - 5 - 3 - 1: one group labelled 1
        i, j = [9, 7, 5, 3], [7, 5, 3, 1]
    elif case == 'star':       # centre 6 with leaves 2, 8, 11; a separate pair (10, 4)
        i, j = [6, 8, 11, 10], [2, 6, 6, 4]
    elif case == 'singletons':
        i, j = [5], [4]
    elif case == 'duplicate_edges':
        i, j = [3, 3, 3, 2, 2], [1, 1, 1, 1, 1]
    elif case == 'empty':
        i, j = [], []
    else:
        rng = np.random.default_rng(3)
        i, j = rng.integers(0, n, 9), rng.integers(0, n, 9)
    i, j = np.asarray(i, dtype=np.int32), np.asarray(j, dtype=np.int32)
    got = duplicate_groups(i, j, n)
    assert got.dtype == np.int32 and got.shape == (n,)
    assert np.array_equal(got, _groups_brute(i, j, n))
    if case == 'chain':
        assert set(got[[1, 3, 5, 7, 9]]) == {1} and all(got[r] == r for r in (0, 2, 4, 6, 8, 10, 11))
    if case == 'star':
        assert set(got[[2, 6, 8, 11]]) == {2} and got[10] == got[4] == 4


def test_duplicate_groups_rejects_bad_indices():
    from dae_rnn_news_recommendation_b200.helpers import duplicate_groups
    with pytest.raises(ValueError, match='outside'):
        duplicate_groups([5], [0], 5)
    with pytest.raises(ValueError, match='outside'):
        duplicate_groups([1], [-1], 5)
    with pytest.raises(ValueError):
        duplicate_groups([1, 2], [0], 5)
    assert duplicate_groups([], [], 0).shape == (0,)


def _agreement_brute(i, j, ql, cl, self_mode):
    use = [(a, b) for a, b in zip(i, j) if ql[a] != -1 and cl[b] != -1]
    same = sum(ql[a] == cl[b] for a, b in use)
    if self_mode:
        total = sum(ql[a] == ql[b] for a, b in itertools.combinations(range(len(ql)), 2) if ql[a] != -1)
    else:
        total = sum(ql[a] == cl[b] for a in range(len(ql)) for b in range(len(cl)) if ql[a] != -1)
    return len(use), (same / len(use) if use else float('nan')), (same / total if total else float('nan'))


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_pair_label_agreement_self(seed):
    from dae_rnn_news_recommendation_b200.helpers import pair_label_agreement
    rng = np.random.default_rng(seed)
    n = 40
    lab = rng.integers(-1, 5, n)
    pairs = [(a, b) for a in range(n) for b in range(a) if rng.random() < 0.1]
    i, j = np.array([p[0] for p in pairs]), np.array([p[1] for p in pairs])
    got = pair_label_agreement(i, j, lab)
    want = _agreement_brute(i, j, lab, lab, True)
    assert got['pairs'] == want[0]
    assert got['precision'] == pytest.approx(want[1]) and got['recall'] == pytest.approx(want[2])


@pytest.mark.parametrize('seed', [0, 1])
def test_pair_label_agreement_corpus(seed):
    from dae_rnn_news_recommendation_b200.helpers import pair_label_agreement
    rng = np.random.default_rng(seed)
    ql, cl = rng.integers(-1, 4, 15), rng.integers(-1, 6, 30)
    i, j = rng.integers(0, 15, 60), rng.integers(0, 30, 60)
    got = pair_label_agreement(i, j, ql, cl)
    want = _agreement_brute(i, j, ql, cl, False)
    assert got['pairs'] == want[0]
    assert got['precision'] == pytest.approx(want[1]) and got['recall'] == pytest.approx(want[2])


def test_pair_label_agreement_empty():
    from dae_rnn_news_recommendation_b200.helpers import pair_label_agreement
    got = pair_label_agreement(np.zeros(0, np.int32), np.zeros(0, np.int32), [0, 0, 1])
    assert got['pairs'] == 0 and np.isnan(got['precision']) and got['recall'] == 0.0
    got = pair_label_agreement([1], [0], [-1, -1])
    assert got['pairs'] == 0 and np.isnan(got['precision']) and np.isnan(got['recall'])


def test_similar_pairs_rejects_before_touching_the_device():
    from dae_rnn_news_recommendation_b200.helpers import similar_pairs
    x = sp.random(20, 30, density=0.2, format='csr', dtype=np.float32, random_state=0)
    d = np.ones((20, 30), dtype=np.float32)
    with pytest.raises(ValueError, match='both sparse or both dense'):
        similar_pairs(x, 0.5, corpus=d)
    with pytest.raises(ValueError, match='both sparse or both dense'):
        similar_pairs(d, 0.5, corpus=x)
    for t in (float('nan'), float('inf'), -float('inf'), 1e39):
        with pytest.raises(ValueError, match='not finite'):
            similar_pairs(d, t)
    with pytest.raises(ValueError, match='not a number'):
        similar_pairs(d, 'high')
    for t in (0.0, -0.5, 1e-46):   # 1e-46 rounds to 0 in float32
        with pytest.raises(ValueError, match='> 0 on sparse input'):
            similar_pairs(x, t)
    with pytest.raises(ValueError, match='metric'):
        similar_pairs(d, 0.5, metric='euclidean')
    with pytest.raises(ValueError, match='max_pairs'):
        similar_pairs(d, 0.5, max_pairs=-1)


def _dense_pairs(n_q=300, n_c=500, dim=64, ldq=64, ldc=64, self_mode=0, tau=0.5, count=FAKE, cap=10, out=FAKE, q=FAKE, c=FAKE):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_similarity_pairs_bf16x3', n_q, n_c, dim, q, q, ldq, c, c, ldc, self_mode, tau, count, cap, out, out, out, None)


def test_dense_export_checks_arguments():
    from dae_rnn_news_recommendation_b200 import _cabi
    bad = [(dict(q=None), 'null pointer'), (dict(count=None), 'null pointer'), (dict(cap=-1), 'capacity'),
           (dict(out=None), 'null output'), (dict(n_q=0), 'bad sizes'), (dict(dim=0), 'bad sizes'),
           (dict(self_mode=1), 'self mode'), (dict(self_mode=1, n_c=300, c=FAKE + 4096), 'self mode'),
           (dict(tau=float('nan')), 'not finite'), (dict(tau=float('inf')), 'not finite'),
           (dict(ldq=60, dim=60), 'multiples of 8'), (dict(ldc=32), 'cover dim'), (dict(q=FAKE + 8), 'aligned'),
           (dict(count=FAKE + 4), 'aligned'), (dict(out=FAKE + 2), 'aligned')]
    for kw, msg in bad:
        with pytest.raises(_cabi.DaeError, match=msg):
            _dense_pairs(**kw)
    with pytest.raises(_cabi.DaeError, match='aligned'):   # capacity 0 counts only: null outputs pass, misaligned ones do not
        _dense_pairs(cap=0, out=FAKE + 2)


def _sparse_pairs(n_q=300, n_c=500, fq=64, fc=64, q_nnz=100, c_nnz=100, self_mode=0, tau=0.5, ws_bytes=1 << 30, count=FAKE, cap=10,
                  out=FAKE, q=FAKE, c=FAKE, ws=FAKE):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_csr_similarity_pairs', q, q, q, n_q, q_nnz, fq, c, c, c, n_c, c_nnz, fc, self_mode, tau, ws, ws_bytes, count, cap,
               out, out, out, None)


def test_sparse_export_checks_arguments():
    from dae_rnn_news_recommendation_b200 import _cabi
    bad = [(dict(q=None), 'null pointer'), (dict(ws=None), 'null pointer'), (dict(count=None), 'null pointer'),
           (dict(cap=-1), 'capacity'), (dict(out=None), 'null output'), (dict(n_c=0), 'bad sizes'), (dict(c_nnz=-1), 'bad sizes'),
           (dict(fq=65), 'features'), (dict(self_mode=1), 'self mode'), (dict(self_mode=1, n_c=300, c=FAKE + 4096), 'self mode'),
           (dict(tau=0.0), '> 0'), (dict(tau=-1.0), '> 0'), (dict(tau=float('nan')), '> 0'), (dict(tau=float('inf')), '> 0'),
           (dict(ws=FAKE + 8), 'aligned'), (dict(count=FAKE + 4), 'aligned'), (dict(ws_bytes=100), 'workspace of 100 bytes')]
    for kw, msg in bad:
        with pytest.raises(_cabi.DaeError, match=msg):
            _sparse_pairs(**kw)


def test_sparse_workspace_size():
    from dae_rnn_news_recommendation_b200 import _cabi
    out = (ctypes.c_int64 * 1)()
    _cabi.call('dae_csr_similarity_pairs_workspace', 300, 5000, 1000, 64, ctypes.addressof(out))
    want = (3 * 64 + 1) * 4 + 4 + 8 * 1000   # buckets of 3 ranges x 64 columns + 1, one scan tile, 8 B postings; no lists
    assert want <= out[0] <= want + 3 * 15
    with pytest.raises(_cabi.DaeError, match='bad arguments'):
        _cabi.call('dae_csr_similarity_pairs_workspace', 300, 0, 1000, 64, ctypes.addressof(out))


def test_dedup_flags():
    import main_autoencoder as cli
    F = cli.build_parser().parse_args([])
    assert F.dedup_threshold == 0.0 and F.dedup_input is False
    F = cli.check_flags(cli.build_parser().parse_args(['--dedup_threshold', '0.9', '--dedup_input']))
    assert F.dedup_threshold == 0.9 and F.dedup_input
    with pytest.raises(AssertionError, match='--dedup_input'):
        cli.check_flags(cli.build_parser().parse_args(['--dedup_input']))
    with pytest.raises(AssertionError):
        cli.check_flags(cli.build_parser().parse_args(['--dedup_threshold', '-1']))


def test_pairs_sort_checks_arguments():
    from dae_rnn_news_recommendation_b200 import _cabi
    which = (ctypes.c_int32 * 1)()
    w = ctypes.addressof(which)
    bad = [((10, 5, 40, None, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE, 1 << 20, w), 'null pointer'),
           ((10, 5, 40, FAKE, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE, 1 << 20, None), 'null pointer'),
           ((-1, 5, 40, FAKE, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE, 1 << 20, w), 'bad sizes'),
           ((1 << 31, 5, 40, FAKE, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE, 1 << 20, w), 'bad sizes'),
           ((10, 0, 40, FAKE, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE, 1 << 20, w), 'bad sizes'),
           ((10, 5, 65, FAKE, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE, 1 << 20, w), 'bad sizes'),
           ((10, 5, 40, FAKE, FAKE, FAKE + 8192, FAKE + 12288, FAKE, 1 << 20, w), 'distinct'),
           ((10, 5, 40, FAKE + 4, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE, 1 << 20, w), 'aligned')]
    for args, msg in bad:
        with pytest.raises(_cabi.DaeError, match=msg):
            _cabi.call('dae_pairs_sort', *args, None)
    out = (ctypes.c_int64 * 1)()
    with pytest.raises(_cabi.DaeError, match='bad arguments'):
        _cabi.call('dae_pairs_sort_workspace', 10, 0, ctypes.addressof(out))
