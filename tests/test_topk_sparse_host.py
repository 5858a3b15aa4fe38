"""Host-side parts of the sparse top-k (dae_csr_similarity_topk): argument checks before any CUDA call, the Python rejections, the
float32 column-ordered oracle the GPU tests compare with, and the --top_k_input flag."""
import ctypes
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FAKE = 1 << 20   # 16-byte aligned non-null stand-in for a device pointer: every call below fails validation before using it


def f32_column_oracle(q, c):
    """S = Q.C^T in float32 the way dae_csr_similarity_topk sums it: from 0, one rounded product per shared column, columns in
    increasing order.  q, c: scipy sparse with the values the kernel is given."""
    q = sp.csc_matrix(q, dtype=np.float32)
    c = sp.csc_matrix(c, dtype=np.float32)
    q.sum_duplicates(); c.sum_duplicates()
    q.sort_indices(); c.sort_indices()
    s = np.zeros((q.shape[0], c.shape[0]), np.float32)
    for f in range(q.shape[1]):
        a0, a1, b0, b1 = q.indptr[f], q.indptr[f + 1], c.indptr[f], c.indptr[f + 1]
        if a1 > a0 and b1 > b0:
            s[np.ix_(q.indices[a0:a1], c.indices[b0:b1])] += np.outer(q.data[a0:a1], c.data[b0:b1])
    return s


def _csr_topk(k=10, nq=300, nc=500, fq=64, fc=64, q_nnz=100, c_nnz=100, ws_bytes=1 << 30, splits=1, q_ptr=FAKE, c_ptr=FAKE):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_csr_similarity_topk', q_ptr, FAKE, FAKE, nq, q_nnz, fq, c_ptr, FAKE, FAKE, nc, c_nnz, fc, k, 0, 1, splits, FAKE,
               ws_bytes, FAKE, FAKE, None)


@pytest.mark.parametrize('k', [0, 33, -1])
def test_k_outside_the_limit_is_rejected(k):
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
        _csr_topk(k=k)
    out = (ctypes.c_int64 * 1)()
    with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
        _cabi.call('dae_csr_similarity_topk_workspace', 300, 500, 100, 64, k, 1, ctypes.addressof(out))


def test_short_workspace_is_rejected():
    from dae_rnn_news_recommendation_b200 import _cabi
    out = (ctypes.c_int64 * 1)()
    _cabi.call('dae_csr_similarity_topk_workspace', 300, 5000, 1000, 64, 10, 2, ctypes.addressof(out))
    # buckets: 3 ranges of 2048 rows x 64 columns + 1 (int32); one scan tile; postings 8 B per corpus entry; 2 partial lists of 10
    want = (3 * 64 + 1) * 4 + 4 + 8 * 1000 + 2 * (300 * 2 * 10 * 4)
    assert want <= out[0] <= want + 5 * 15
    with pytest.raises(_cabi.DaeError, match='workspace'):
        _csr_topk(nc=5000, c_nnz=1000, splits=2, ws_bytes=out[0] - 1)


def test_feature_mismatch_is_rejected():
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='features'):
        _csr_topk(fq=64, fc=65)


@pytest.mark.parametrize('field', ['nq', 'nc', 'fq', 'fc', 'q_nnz'])
def test_non_positive_sizes_are_rejected(field):
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='bad sizes'):
        _csr_topk(**{field: -1 if field == 'q_nnz' else 0})
    out = (ctypes.c_int64 * 1)()
    with pytest.raises(_cabi.DaeError, match='bad arguments'):
        _cabi.call('dae_csr_similarity_topk_workspace', 0, 500, 100, 64, 10, 1, ctypes.addressof(out))


def test_null_pointers_are_rejected():
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match='null pointer'):
        _csr_topk(q_ptr=None)
    with pytest.raises(_cabi.DaeError, match='null pointer'):
        _csr_topk(c_ptr=None)


def test_python_rejects_before_touching_the_device():
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200.helpers import top_k_similar
    x = sp.random(20, 30, density=0.2, format='csr', dtype=np.float32, random_state=0)
    with pytest.raises(ValueError, match='both sparse or both dense'):
        top_k_similar(x, k=5, corpus=x.toarray())
    with pytest.raises(ValueError, match='both sparse or both dense'):
        top_k_similar(x.toarray(), k=5, corpus=x)
    with pytest.raises(ValueError, match='columns'):
        top_k_similar(x, k=5, corpus=sp.random(20, 31, density=0.2, format='csr', dtype=np.float32, random_state=1))
    with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
        top_k_similar(x, k=33)


def test_cosine_operand_rows_are_unit_or_zero():
    from dae_rnn_news_recommendation_b200.helpers import _csr_operand
    x = sp.random(50, 40, density=0.1, format='csr', dtype=np.float32, random_state=2)
    x = sp.vstack([x, sp.csr_matrix((1, 40), dtype=np.float32)]).tocsr()
    m = _csr_operand(x, 'cosine')
    assert m.dtype == np.float32 and m.has_canonical_format
    n = np.sqrt(np.asarray(m.multiply(m).sum(1)).ravel())
    assert np.allclose(n[np.diff(x.indptr) > 0], 1.0, atol=1e-6) and n[-1] == 0.0
    assert _csr_operand(x, 'linear kernel').nnz == x.nnz


def test_f32_oracle_against_fp64():
    rng = np.random.default_rng(0)
    q = sp.random(40, 300, density=0.1, format='csr', dtype=np.float64, random_state=3)
    c = sp.random(70, 300, density=0.1, format='csr', dtype=np.float64, random_state=4)
    q.data = (rng.random(q.nnz) - 0.3).astype(np.float32)
    c.data = (rng.random(c.nnz) - 0.3).astype(np.float32)
    s32 = f32_column_oracle(q, c)
    s64 = (q.astype(np.float64) @ c.astype(np.float64).T).toarray()
    assert s32.dtype == np.float32
    assert np.abs(s32 - s64).max() < 1e-5
    # the summation order is the column order: a row pair sharing columns f1 < f2 < f3 gets ((0 + p1) + p2) + p3 in float32
    q1 = sp.csr_matrix((np.array([1.0, 1e-8, 1.0], np.float32), np.array([0, 1, 2]), np.array([0, 3])), shape=(1, 3))
    c1 = sp.csr_matrix((np.array([1.0, 1.0, -1.0], np.float32), np.array([0, 1, 2]), np.array([0, 3])), shape=(1, 3))
    assert f32_column_oracle(q1, c1)[0, 0] == np.float32(np.float32(np.float32(1.0) + np.float32(1e-8)) - np.float32(1.0))


def test_top_k_input_flag():
    import main_autoencoder as cli
    assert cli.build_parser().parse_args([]).top_k_input is False
    F = cli.check_flags(cli.build_parser().parse_args(['--top_k', '5', '--top_k_input']))
    assert F.top_k == 5 and F.top_k_input
    with pytest.raises(AssertionError, match='--top_k_input'):
        cli.check_flags(cli.build_parser().parse_args(['--top_k_input']))
