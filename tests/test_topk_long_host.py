"""Long top-k lists without a GPU: the new exports' argument checks, the helpers' validation before any device work, the CLI flags,
and the host oracle the GPU tests compare against."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp

from topk_groups_oracle import grouped_top_k


def _call(name, *args):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call(name, *args)


A = 1 << 12   # a fake, 16-byte aligned device address: every call here must fail before touching it


def _bound(**kw):
    a = dict(n_query=10, n_corpus=20, dim=8, q_hi=A, q_lo=A, ldq=8, c_hi=A, c_lo=A, ldc=8, k=100, diag_offset=0, exclude=0, splits=0,
             workspace=A, workspace_bytes=1 << 30, ex_indptr=None, ex_indices=None, ex_nnz=0, groups=None, tau=A, stream=None)
    a.update(kw)
    _call('dae_similarity_topk_bound_bf16x3', *a.values())


def _collect(**kw):
    a = dict(n_query=10, n_corpus=20, dim=8, q_hi=A, q_lo=A, ldq=8, c_hi=A, c_lo=A, ldc=8, diag_offset=0, exclude=0, tau=A,
             ex_indptr=None, ex_indices=None, ex_nnz=0, count=A, row_count=A, capacity=0, i_out=None, j_out=None, s_out=None,
             stream=None)
    a.update(kw)
    _call('dae_similarity_topk_collect_bf16x3', *a.values())


def _select(**kw):
    a = dict(n_query=10, n_pairs=5, i=A, j=A, s=A, k=100, groups=None, idx_out=A, val_out=A, stream=None)
    a.update(kw)
    _call('dae_similarity_topk_select', *a.values())


@pytest.mark.parametrize('fn, kw, msg', [
    (_bound, dict(q_hi=None), 'null pointer'), (_bound, dict(tau=None), 'null pointer'), (_bound, dict(ex_nnz=3), 'null pointer'),
    (_bound, dict(n_query=0), 'bad sizes'), (_bound, dict(dim=0), 'bad sizes'), (_bound, dict(k=0), '1 <= k <= 1024'),
    (_bound, dict(k=1025), '1 <= k <= 1024'), (_bound, dict(ldq=7), 'leading dimensions'), (_bound, dict(q_lo=A + 8), 'aligned'),
    (_bound, dict(tau=A + 2), 'aligned'), (_bound, dict(workspace_bytes=16), 'workspace of 16 bytes'),
    (_collect, dict(count=None), 'null pointer'), (_collect, dict(row_count=None), 'null pointer'),
    (_collect, dict(capacity=-1), 'capacity'), (_collect, dict(capacity=4), 'null output'), (_collect, dict(n_corpus=0), 'bad sizes'),
    (_collect, dict(ldc=12), 'leading dimensions'), (_collect, dict(count=A + 4), 'aligned'),
    (_select, dict(i=None), 'null pointer'), (_select, dict(val_out=None), 'null pointer'), (_select, dict(n_pairs=-1), 'bad sizes'),
    (_select, dict(n_query=0), 'bad sizes'), (_select, dict(k=0), '1 <= k <= 1024'), (_select, dict(k=1025), '1 <= k <= 1024'),
    (_select, dict(s=A + 2), 'aligned'),
])
def test_export_argument_checks(fn, kw, msg):
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError, match=msg):
        fn(**kw)


def test_bound_workspace_query():
    from dae_rnn_news_recommendation_b200 import _cabi
    need = (ctypes.c_int64 * 1)()
    for k in (0, 1025):
        with pytest.raises(_cabi.DaeError, match='1 <= k <= 1024'):
            _call('dae_similarity_topk_bound_workspace', 10, 20, k, 0, ctypes.addressof(need))
    with pytest.raises(_cabi.DaeError):
        _call('dae_similarity_topk_bound_workspace', 10, 20, 5, 0, None)


def test_helper_validation_before_device_work():
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200.helpers import recommend, top_k_similar
    x = np.zeros((4, 3), np.float32)
    for k in (0, 1025):
        with pytest.raises(_cabi.DaeError, match='1 <= k <= 1024'):
            top_k_similar(x, k=k, long_lists=True)
        with pytest.raises(_cabi.DaeError, match='1 <= k <= 1024'):
            recommend(sp.csr_matrix((2, 4)), x, k=k, long_lists=True)
    with pytest.raises(_cabi.DaeError, match='1 <= k <= 32'):
        top_k_similar(x, k=100)
    with pytest.raises(ValueError, match='at most 32'):
        top_k_similar(sp.csr_matrix(x), k=33, long_lists=True)
    for bad in (0, -5, 1.5, 'many', True):
        with pytest.raises(ValueError, match='max_candidates'):
            top_k_similar(x, k=100, long_lists=True, max_candidates=bad)
        with pytest.raises(ValueError, match='max_candidates'):
            recommend(sp.csr_matrix((2, 4)), x, k=100, long_lists=True, max_candidates=bad)


def test_cli_flags():
    import main_autoencoder as cli

    def check(*argv):
        return cli.check_flags(cli.build_parser().parse_args(list(argv)))
    assert check().long_lists is False
    with pytest.raises(AssertionError):
        check('--top_k', '100')
    F = check('--top_k', '100', '--long_lists')
    assert F.top_k == 100 and F.long_lists
    assert check('--top_k', '1024', '--long_lists').top_k == 1024
    with pytest.raises(AssertionError):
        check('--top_k', '1025', '--long_lists')
    with pytest.raises(ValueError, match='32'):
        check('--top_k', '100', '--long_lists', '--top_k_input')
    assert check('--top_k', '32', '--long_lists', '--top_k_input').top_k_input


def test_oracle_by_hand():
    s = np.array([[3.0, 1.0, 3.0, -0.0, 0.0, 2.0],
                  [1.0, 1.0, 1.0, 1.0, 1.0, 1.0]])
    idx, val = grouped_top_k(s, np.arange(6), 5)
    assert idx.tolist() == [[0, 2, 5, 1, 3], [0, 1, 2, 3, 4]]          # ties by index; -0.0 ties with +0.0
    assert val[0].tolist() == [3.0, 3.0, 2.0, 1.0, 0.0]
    idx, val = grouped_top_k(s, np.array([0, 1, 0, 2, 2, 1]), 5)       # one entry per group, then padding
    assert idx.tolist() == [[0, 5, 3, -1, -1], [0, 1, 3, -1, -1]]
    assert val[0].tolist()[:3] == [3.0, 2.0, 0.0] and np.isneginf(val[:, 3:]).all()
    allowed = np.ones_like(s, bool)
    allowed[0, [0, 2]] = False
    allowed[1] = False
    idx, val = grouped_top_k(s, np.arange(6), 8, allowed)
    assert idx.tolist() == [[5, 1, 3, 4, -1, -1, -1, -1], [-1] * 8] and np.isneginf(val[1]).all()
