"""similarity_auroc / the pair-histogram kernels: bit-exact histograms against host oracles (dense integer scores, sparse float32
column-ordered scores), agreement with the sort path within the bound the contract gives, determinism, full-size runs with a memory
bound, and the --eval_all_rows CLI path."""
import os
import sys

import numpy as np
import pytest

from test_auroc_hist_host import host_histograms
from test_topk_sparse_host import f32_column_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _labels(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == 'single':
        return np.full(n, 7)
    if kind == 'many':
        return rng.integers(0, 300, n)
    lab = rng.integers(0, 5, n)
    lab[rng.random(n) < 0.2] = -1
    return lab


def _device_hist(data, labels, metric, bins):
    from dae_rnn_news_recommendation_b200.helpers import _pair_histograms
    hist, sums, M = _pair_histograms(data, labels, metric, bins)
    return hist.cpu().numpy(), sums.cpu().numpy(), M


def _grid_vs_sort_bound(h, hp):
    """|A(h) - A_sort| <= 1/2 sum|dh_rel| / R + 1/2 sum|dh_unrel| / U + bound(h'), h' the sort path's scores on the same grid."""
    r, u = int(hp[0].sum()), int(hp[1].sum())
    return 0.5 * np.abs(h[0] - hp[0]).sum() / r + 0.5 * np.abs(h[1] - hp[1]).sum() / u


@pytest.mark.parametrize('h', [16, 500])
@pytest.mark.parametrize('n', [2, 127, 128, 129, 1000, 3001])
def test_dense_integer_scores_bit_exact(n, h):
    """Small-integer rows: every bf16x3 score is an exact integer, so the histogram must equal the host binning exactly."""
    rng = np.random.default_rng(n * 1000 + h)
    x = rng.integers(-2, 3, (n, h)).astype(np.float32)
    s = (x.astype(np.int64) @ x.astype(np.int64).T).astype(np.float32)
    from dae_rnn_news_recommendation_b200.helpers import grid_range
    for kind in ('missing', 'single', 'many'):
        lab = _labels(kind, n, n + h)
        bins = 1 << 21 if kind == 'missing' else 1 << 12
        got, sums, M = _device_hist(x, lab, 'linear kernel', bins)
        assert M == grid_range(float((x.astype(np.float64) ** 2).sum(1).max()), 'linear kernel')
        want, want_sums, rel, unrel = host_histograms(s, lab, M, bins)
        assert np.array_equal(got, want), (kind, np.abs(got - want).sum())
        assert np.array_equal(sums, want_sums), (kind, sums, want_sums)   # integer scores: the fp64 sums are exact


def _tfidf_like(n, f, seed):
    from test_gpu_topk_sparse import _tfidf_like as make
    return make(n, f, seed)


@pytest.mark.parametrize('metric', ['linear kernel', 'cosine'])
def test_sparse_bit_exact_against_the_float32_oracle(metric):
    """4 500 rows (two full ranges of 2048 and a partial one): empty rows, a column in every row, negative values, exact ties."""
    from dae_rnn_news_recommendation_b200.helpers import _csr_operand
    x = _tfidf_like(4500, 700, 21)
    x.data[::5] = np.round(x.data[::5] * 4) / 4                 # ties
    x.eliminate_zeros()
    for kind in ('missing', 'single', 'many'):
        lab = _labels(kind, x.shape[0], 3)
        got, sums, M = _device_hist(x, lab, metric, 1 << 21)
        m = _csr_operand(x, metric)
        want, want_sums, rel, unrel = host_histograms(f32_column_oracle(m, m), lab, M, 1 << 21)
        assert np.array_equal(got, want), (kind, np.abs(got - want).sum())
        assert np.allclose(sums, want_sums, rtol=1e-9, atol=1e-9)
        assert got[0].sum() == len(rel) and got[1].sum() == len(unrel)


@pytest.mark.parametrize('label', ['category_publish_name', 'story'])
def test_sparse_uci_c1_binary_cosine(label):
    from helpers import load_uci_c1
    from dae_rnn_news_recommendation_b200.helpers import _csr_operand
    d = load_uci_c1()
    x, lab = d['train'], d['train_label_' + label]
    got, sums, M = _device_hist(x, lab, 'cosine', 1 << 21)
    m = _csr_operand(x, 'cosine')
    want, want_sums, _, _ = host_histograms(f32_column_oracle(m, m), lab, M, 1 << 21)
    assert np.array_equal(got, want)
    assert np.allclose(sums, want_sums, rtol=1e-9, atol=1e-6)


def _clustered(n, h, seed):
    rng = np.random.RandomState(seed)
    labels = rng.randint(0, 4, n)
    emb = (rng.randn(4, h)[labels] * 0.15 + rng.randn(n, h)).astype(np.float32)
    return emb, labels


def test_dense_against_the_sort_path():
    """8 000 clustered embeddings (as test_full_size_complement_property_and_json), cosine."""
    from dae_rnn_news_recommendation_b200.helpers import (auroc_from_histograms, pairwise_similarity, similarity_auroc,
                                                          visualize_pairwise_similarity)
    emb, labels = _clustered(8000, 500, 5)
    bins = 1 << 21
    sim = pairwise_similarity(emb, metric='cosine', to_host=False)
    a_sort = visualize_pairwise_similarity(labels, sim)
    hp, sums_p, _, _ = host_histograms(sim.cpu().numpy(), labels, 1.0, bins)
    del sim
    got = similarity_auroc(emb, labels, bins=bins)
    h, _, _ = _device_hist(emb, labels, 'cosine', bins)
    bound_p = auroc_from_histograms(hp, sums_p, 1.0, bins)['auroc_error_bound']
    assert abs(got['auroc'] - a_sort['auroc']) <= _grid_vs_sort_bound(h, hp) + bound_p
    assert got['auroc_error_bound'] < 1e-4
    w = got['bin_width']
    for grp in ('related', 'unrelated'):
        assert got[grp]['n'] == a_sort[grp]['n']
        for k in ('q1', 'median', 'q3', 'whisker_lo', 'whisker_hi', 'mean'):
            assert abs(got[grp][k] - a_sort[grp][k]) <= 2 * w + 1e-6, (grp, k, got[grp][k], a_sort[grp][k])


def test_two_calls_give_identical_histograms():
    emb, labels = _clustered(3000, 200, 6)
    a = _device_hist(emb, labels, 'cosine', 1 << 21)
    b = _device_hist(emb, labels, 'cosine', 1 << 21)
    assert np.array_equal(a[0], b[0])
    x = _tfidf_like(3000, 300, 7)
    a = _device_hist(x, labels, 'cosine', 1 << 21)
    b = _device_hist(x, labels, 'cosine', 1 << 21)
    assert np.array_equal(a[0], b[0])


def _group_sizes(labels):
    from dae_rnn_news_recommendation_b200.helpers import _group_sizes
    return _group_sizes(np.asarray(labels))


def test_full_size_dense_against_a_chunked_gemm_histogram():
    """100 000 x 500 cosine: totals, memory above the inputs, and the histogram of a chunked GEMM + torch.bucketize on the device."""
    import torch
    from dae_rnn_news_recommendation_b200 import helpers
    n, h, bins = 100000, 500, 1 << 21
    emb, labels = _clustered(n, h, 8)
    x = torch.from_numpy(emb).cuda()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    hist, sums, M = helpers._pair_histograms(x, labels, 'cosine', bins)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < 0.5 * 2 ** 30
    hist = hist.cpu().numpy()
    r, u = _group_sizes(labels)
    assert int(hist[0].sum()) == r and int(hist[1].sum()) == u
    # reference: S rows in chunks from dae_gemm_bf16x3, lower triangle binned by torch.bucketize on fl32(s + 1)
    hi, lo, _ = helpers._normalised_operands(x, 2)
    lab = torch.from_numpy(labels).cuda()
    edges = torch.arange(1, bins, dtype=torch.float32, device='cuda') * (2.0 / bins)
    ref = torch.zeros(2 * bins, dtype=torch.int64, device='cuda')
    chunk = 4096
    buf = torch.empty(chunk, n, dtype=torch.float32, device='cuda')
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        helpers._gemm_nt((hi[r0:r1], lo[r0:r1]), (hi, lo), r1 - r0, r1, h, buf)
        s = buf[:r1 - r0, :r1]
        keep = torch.arange(r1, device='cuda')[None, :] < torch.arange(r0, r1, device='cuda')[:, None]
        b = torch.bucketize(s[keep] + 1.0, edges, right=True)
        unrel = (lab[r0:r1, None] != lab[None, :r1])[keep].long()
        ref += torch.bincount(unrel * bins + b, minlength=2 * bins)
        del s, keep, b, unrel
    del buf
    hp = ref.view(2, bins).cpu().numpy()
    out = helpers.auroc_from_histograms(hist, sums.cpu().numpy(), M, bins)
    ref_out = helpers.auroc_from_histograms(hp, np.zeros(2), M, bins)
    assert abs(out['auroc'] - ref_out['auroc']) <= _grid_vs_sort_bound(hist, hp) + ref_out['auroc_error_bound']
    assert 0.5 < out['auroc'] < 1.0 and out['auroc_error_bound'] < 1e-4


def test_full_size_sparse_c2_like():
    """100 000 x 10 000 tf-idf (C2-like), linear kernel: totals and memory above the inputs."""
    import torch
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.synth import make_labels, make_sparse
    n = 100000
    x = make_sparse(n, 10000, mean_nnz=100, kind='tfidf', seed=10000)
    labels = make_labels(n, 4, seed=3)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    hist, sums, M = helpers._pair_histograms(x, labels, 'linear kernel', 1 << 21)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < 0.5 * 2 ** 30
    assert M == 1.0
    hist = hist.cpu().numpy()
    r, u = _group_sizes(labels)
    assert int(hist[0].sum()) == r and int(hist[1].sum()) == u
    out = helpers.auroc_from_histograms(hist, sums.cpu().numpy(), M, 1 << 21)
    assert 0.0 < out['auroc'] < 1.0 and out['related']['n'] == r


def test_cli_eval_all_rows(tmp_path):
    """evaluate(max_rows=500) with --eval_all_rows on the 1 200-row synthetic run: the 960 training rows take the histogram path,
    with the keys and JSON files of the sort path and AUROCs within the contract's distance of it."""
    import json
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.autoencoder import utils
    argv = ['--model_name', 'synevalall', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size',
            '200', '--seed', '3', '--eval_all_rows']
    model = cli.main(argv)
    F = cli.check_flags(cli.build_parser().parse_args(argv))
    trX, vlX, trL, vlL = cli.prepare_synthetic(F)
    enc = model.transform(utils.decay_noise(trX, F.corr_frac), name='article_encoded', save=False)
    enc_v = model.transform(utils.decay_noise(vlX, F.corr_frac), name='article_encoded_validate', save=False)
    sort_ev = cli.evaluate(F, model, trX, vlX, trL, vlL, enc, enc_v)
    ev = cli.evaluate(F, model, trX, vlX, trL, vlL, enc, enc_v, max_rows=500)
    assert set(ev) == set(sort_ev) == set(model.evaluation)
    for name, data in (('binary_count', trX), ('encoded', enc)):
        key = 'similarity_boxplot_%s(Category)' % name
        got = ev[key]
        assert 'auroc_error_bound' in got and got['title'] == key
        saved = json.load(open(model.plot_dir + key + '.json'))
        assert saved['auroc'] == got['auroc'] and saved['twice_u'] == got['twice_u']
        bins = 1 << 21
        h, _, _ = _device_hist(data, trL, 'cosine', bins)
        s = helpers.pairwise_similarity(data, metric='cosine')
        hp, sums_p, _, _ = host_histograms(s, trL, 1.0, bins)
        bound_p = helpers.auroc_from_histograms(hp, sums_p, 1.0, bins)['auroc_error_bound']
        assert abs(got['auroc'] - sort_ev[key]['auroc']) <= _grid_vs_sort_bound(h, hp) + bound_p
    idx, score = ev['nearest']
    want = helpers.top_k_similar(enc, k=1)
    assert np.array_equal(idx, want[0][:, 0]) and np.array_equal(score, want[1][:, 0])
    key_v = 'similarity_boxplot_encoded_validate(Category)'
    assert 'auroc_error_bound' not in ev[key_v] and ev[key_v]['auroc'] == sort_ev[key_v]['auroc']   # 240 rows: the sort path
