"""Host half of the histogram AUROC (helpers.auroc_from_histograms, score_bins, grid_range), the argument checks of the pair-histogram
entry points before any CUDA call, and the --eval_all_rows flag."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import eval_oracle  # noqa: E402

FAKE = 1 << 20   # 16-byte aligned non-null stand-in for a device pointer: every call below fails validation before using it


def host_histograms(scores, labels, M, bins):
    """hist [2, bins] and fp64 sums [2] of the strict lower triangle of a square score matrix, as the kernels count them."""
    rel, unrel = eval_oracle.related_unrelated(labels, np.asarray(scores, dtype=np.float32))
    from dae_rnn_news_recommendation_b200.helpers import score_bins
    hist = np.stack([np.bincount(score_bins(g, M, bins), minlength=bins) for g in (rel, unrel)]).astype(np.int64)
    return hist, np.array([rel.astype(np.float64).sum(), unrel.astype(np.float64).sum()]), rel, unrel


def _sym(n, values):
    s = np.zeros((n, n), np.float32)
    il = np.tril_indices(n, -1)
    s[il] = values
    return s + s.T


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_bin_centre_scores_give_the_exact_auroc_and_box_statistics(seed):
    from dae_rnn_news_recommendation_b200.helpers import auroc_from_histograms
    rng = np.random.default_rng(seed)
    n, bins, M = 300, 1 << 10, 1.0
    labels = rng.integers(-1, 5, n)
    w = 2 * M / bins
    b = np.clip(np.round(rng.normal(bins / 2, bins / 12, n * (n - 1) // 2)).astype(np.int64), 0, bins - 1)
    scores = _sym(n, (-M + (b + 0.5) * w).astype(np.float32))    # every score is the centre of its bin: the grid loses nothing
    hist, sums, rel, unrel = host_histograms(scores, labels, M, bins)
    out = auroc_from_histograms(hist, sums, M, bins)
    want, twice = eval_oracle.auroc(rel, unrel)
    assert out['twice_u'] == twice and out['auroc'] == want
    assert out['bin_width'] == w and 0.0 < out['auroc_error_bound'] < 0.5
    for grp, data in (('related', rel), ('unrelated', unrel)):
        ws = eval_oracle.box_stats(data)
        assert out[grp]['n'] == ws['n']
        for k in ('q1', 'median', 'q3', 'whisker_lo', 'whisker_hi', 'mean'):
            assert abs(out[grp][k] - ws[k]) <= 1e-12, (grp, k, out[grp][k], ws[k])


@pytest.mark.parametrize('bins', [1 << 10, 1 << 14, 1 << 21])
def test_random_scores_stay_within_the_bound(bins):
    from dae_rnn_news_recommendation_b200.helpers import auroc_from_histograms
    rng = np.random.default_rng(bins)
    n = 400
    labels = rng.integers(0, 3, n)
    v = (rng.normal(0.0, 0.2, n * (n - 1) // 2) + 0.05 * rng.random(n * (n - 1) // 2)).astype(np.float32)
    v[::7] = np.round(v[::7], 2)                                    # exact ties across the groups as well
    hist, sums, rel, unrel = host_histograms(_sym(n, v), labels, 1.0, bins)
    out = auroc_from_histograms(hist, sums, 1.0, bins)
    exact = eval_oracle.auroc(rel, unrel)[0]
    assert abs(out['auroc'] - exact) <= out['auroc_error_bound'] + 1e-15
    assert out['related']['n'] == len(rel) and out['unrelated']['n'] == len(unrel)
    assert abs(out['related']['mean'] - rel.astype(np.float64).mean()) < 1e-12
    for grp, data in (('related', rel), ('unrelated', unrel)):
        ws = eval_oracle.box_stats(data)
        for k in ('q1', 'median', 'q3'):
            assert abs(out[grp][k] - ws[k]) <= 2.0 / bins + 1e-7


def test_counts_near_1e11_give_an_exact_twice_u():
    from dae_rnn_news_recommendation_b200.helpers import auroc_from_histograms
    bins = 1 << 10
    hist = np.zeros((2, bins), np.int64)
    rng = np.random.default_rng(4)
    occ = rng.choice(bins, 40, replace=False)
    hist[0, occ[:25]] = 10 ** 11 + rng.integers(0, 10 ** 9, 25)
    hist[1, occ[15:]] = 3 * 10 ** 11 + rng.integers(0, 10 ** 9, 25)
    nr, nu = [int(x) for x in hist[0]], [int(x) for x in hist[1]]
    twice, below = 0, 0
    for b in range(bins):
        twice += nr[b] * (2 * below + nu[b])
        below += nu[b]
    out = auroc_from_histograms(hist, np.zeros(2), 1.0, bins)
    assert twice > 2 ** 64 and out['twice_u'] == twice
    r, u = sum(nr), sum(nu)
    assert out['auroc'] == twice / (2.0 * r * u)
    assert out['auroc_error_bound'] == sum(a * c for a, c in zip(nr, nu)) / (2.0 * r * u)


@pytest.mark.parametrize('labels', [[3, 3, 3, 3, 3], [0, 1, 2, 3, 4], [-1, -1, -1, -1, -1], [-1, -1, 0, -1, 1]])
def test_degenerate_groups_give_nan(labels):
    from dae_rnn_news_recommendation_b200.helpers import auroc_from_histograms
    hist, sums, rel, unrel = host_histograms(np.zeros((5, 5), np.float32), np.array(labels), 1.0, 1 << 10)
    out = auroc_from_histograms(hist, sums, 1.0, 1 << 10)
    assert np.isnan(out['auroc']) and np.isnan(out['auroc_error_bound']) and out['twice_u'] == 0
    assert out['related'].get('n') == len(rel) and out['unrelated'].get('n') == len(unrel)
    for grp in ('related', 'unrelated'):
        if out[grp]['n'] == 0:
            assert out[grp] == {'n': 0}


def test_bin_formula_is_monotone_and_clamps():
    from dae_rnn_news_recommendation_b200.helpers import score_bins
    rng = np.random.default_rng(5)
    for M, bins in ((1.0, 1 << 21), (1.0, 1 << 24), (4.0, 1 << 10), (2.0 ** -3, 1 << 16)):
        s = np.concatenate([rng.uniform(-1.2 * M, 1.2 * M, 200000), np.linspace(-M, M, bins + 1), [-np.inf, np.inf, 0.0, -0.0, M, -M]])
        s = np.sort(s.astype(np.float32))
        s = np.concatenate([s, np.nextafter(s, np.float32(np.inf)), np.nextafter(s, np.float32(-np.inf))])
        s = np.sort(s)
        b = score_bins(s, M, bins)
        assert (np.diff(b) >= 0).all()
        assert b.min() == 0 and b.max() == bins - 1
        assert score_bins(np.float32(0.0), M, bins) == bins // 2
        assert score_bins(np.float32(-M), M, bins) == 0 and score_bins(np.float32(M), M, bins) == bins - 1
    w = 2.0 / (1 << 10)                                               # bin edges and centres land where the contract says
    assert list(score_bins(np.float32([-1 + 3 * w, -1 + 3.5 * w, -1 + 4 * w - w / 64]), 1.0, 1 << 10)) == [3, 3, 3]


def test_grid_range():
    from dae_rnn_news_recommendation_b200.helpers import grid_range
    assert grid_range(123.0, 'cosine') == 1.0
    assert grid_range(1.0, 'linear kernel') == 1.0
    assert grid_range(1.0000004, 'linear kernel') == 1.0        # l2-normalised rows, rounded up by a few ulp
    assert grid_range(0.3, 'linear kernel') == 0.5
    assert grid_range(3.0, 'linear kernel') == 4.0 and grid_range(4.0, 'linear kernel') == 4.0
    assert grid_range(4.1, 'linear kernel') == 8.0
    assert grid_range(0.0, 'linear kernel') == 1.0


def test_python_rejects_before_touching_the_device():
    from dae_rnn_news_recommendation_b200.helpers import auroc_from_histograms, similarity_auroc
    x = np.zeros((10, 4), np.float32)
    for bins in (1000, 1 << 9, 1 << 25, 0, 2.0 ** 20):
        with pytest.raises(ValueError, match='bins'):
            similarity_auroc(x, np.zeros(10), bins=bins)
    with pytest.raises(ValueError, match='metric'):
        similarity_auroc(x, np.zeros(10), metric='euclidean')
    with pytest.raises(ValueError, match='labels'):
        similarity_auroc(x, np.zeros(9))
    with pytest.raises(ValueError, match='shape'):
        auroc_from_histograms(np.zeros((2, 1 << 11), np.int64), np.zeros(2), 1.0, 1 << 10)
    with pytest.raises(ValueError, match='bins'):
        auroc_from_histograms(np.zeros((2, 1000), np.int64), np.zeros(2), 1.0, 1000)


def _dense(n=300, dim=64, ld=64, x_ptr=FAKE, lab_ptr=FAKE, M=1.0, bins=1 << 20, hist_ptr=FAKE):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_similarity_pair_hist_bf16x3', n, dim, x_ptr, FAKE, ld, lab_ptr, M, bins, hist_ptr, FAKE, None)


def _sparse(n=300, nnz=100, f=64, ptr=FAKE, M=1.0, bins=1 << 20, ws_bytes=1 << 30, ws_ptr=FAKE):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_csr_similarity_pair_hist', ptr, FAKE, FAKE, n, nnz, f, FAKE, M, bins, ws_ptr, ws_bytes, FAKE, FAKE, None)


@pytest.mark.parametrize('call', [_dense, _sparse])
def test_entry_points_reject_bad_arguments(call):
    from dae_rnn_news_recommendation_b200 import _cabi
    for bins in (1000, 1 << 9, 1 << 25, 0, -1024):
        with pytest.raises(_cabi.DaeError, match='power of two'):
            call(bins=bins)
    for M in (0.75, 0.0, -1.0, float('inf'), float('nan'), 2.0 ** 70, 3.0):
        with pytest.raises(_cabi.DaeError, match='range M'):
            call(M=M)
    for n in (1, 0, -5):
        with pytest.raises(_cabi.DaeError, match='bad sizes'):
            call(n=n)
    with pytest.raises(_cabi.DaeError, match='null pointer'):
        call(**({'x_ptr': None} if call is _dense else {'ptr': None}))


def test_dense_entry_point_checks_layout():
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='leading dimension'):
        _dense(dim=64, ld=60)
    with pytest.raises(_cabi.DaeError, match='leading dimension'):
        _dense(dim=60, ld=60)
    with pytest.raises(_cabi.DaeError, match='aligned'):
        _dense(x_ptr=FAKE + 8)
    with pytest.raises(_cabi.DaeError, match='aligned'):
        _dense(hist_ptr=FAKE + 4)
    with pytest.raises(_cabi.DaeError, match='aligned'):
        _dense(lab_ptr=FAKE + 2)
    with pytest.raises(_cabi.DaeError, match='bad sizes'):
        _dense(dim=0)


def test_sparse_entry_point_checks_nnz_and_workspace():
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='bad sizes'):
        _sparse(nnz=2 ** 31)
    with pytest.raises(_cabi.DaeError, match='bad sizes'):
        _sparse(nnz=-1)
    with pytest.raises(_cabi.DaeError, match='aligned'):
        _sparse(ws_ptr=FAKE + 8)
    out = (ctypes.c_int64 * 1)()
    _cabi.call('dae_csr_similarity_pair_hist_workspace', 5000, 1000, 64, ctypes.addressof(out))
    want = (3 * 64 + 1) * 4 + 4 + 8 * 1000                       # buckets of 3 ranges x 64 columns + 1, one scan tile, postings
    assert want <= out[0] <= want + 3 * 15
    with pytest.raises(_cabi.DaeError, match='workspace'):
        _sparse(n=5000, nnz=1000, ws_bytes=out[0] - 1)
    for args in ((1, 1000, 64), (5000, 2 ** 31, 64), (5000, 1000, 0)):
        with pytest.raises(_cabi.DaeError, match='bad arguments'):
            _cabi.call('dae_csr_similarity_pair_hist_workspace', *args, ctypes.addressof(out))


def test_eval_all_rows_flag():
    import main_autoencoder as cli
    assert cli.build_parser().parse_args([]).eval_all_rows is False
    assert cli.check_flags(cli.build_parser().parse_args(['--eval_all_rows'])).eval_all_rows is True
