"""Host side of the GRU user encoder: packing, sequences_from_csr, the negative mapping, state dicts, the fp64 oracle against
torch.nn.GRU, make_sequences and input validation.  No GPU needed."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from user_gru_oracle import NAMES, gru_states  # noqa: E402

from dae_rnn_news_recommendation_b200.user_model import Packed, UserGRU, check_sequences, negatives_from_draws  # noqa: E402


def _seqs(lens, n_items=50, seed=0):
    rng = np.random.default_rng(seed)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return indptr, rng.integers(0, n_items, int(indptr[-1])).astype(np.int32)


def test_packing_order_counts_truncation():
    lens = [3, 0, 1, 7, 2, 7, 5]
    indptr, items = _seqs(lens)
    pk = Packed(indptr, items, np.arange(len(lens)), max_len=5)
    assert list(pk.order) == [3, 5, 6, 0, 4, 2]            # by truncated length desc, stable; the empty user left out
    assert list(pk.L) == [5, 5, 5, 3, 2, 1]
    assert list(pk.n) == [6, 5, 4, 3, 3]
    assert list(pk.off) == [0, 6, 11, 15, 18, 21] and pk.P == 21
    assert pk.terms == 4 + 4 + 4 + 2 + 1
    for i, u in enumerate(pk.order):
        s = items[indptr[u]:indptr[u + 1]][-5:]             # the last max_len reads
        for t in range(len(s)):
            p = pk.position(i, t)
            assert pk.items[p] == s[t]
            assert pk.nxt[p] == (s[t + 1] if t + 1 < len(s) else -1)
    assert (pk.n[1:] <= pk.n[:-1]).all()


def test_packing_short_users():
    indptr, items = _seqs([0, 1, 0])
    pk = Packed(indptr, items, np.arange(3), max_len=50)
    assert pk.B == 1 and pk.P == 1 and pk.terms == 0 and list(pk.nxt) == [-1]
    pk = Packed(indptr, items, [0, 2], max_len=50)
    assert pk.B == 0 and pk.P == 0


def test_sequences_from_csr():
    from dae_rnn_news_recommendation_b200.helpers import sequences_from_csr
    m = sp.csr_matrix((np.array([5., 1., 3., 0., 2., 2.]), (np.array([0, 0, 0, 2, 2, 2]), np.array([4, 7, 1, 9, 3, 0]))), shape=(3, 10))
    indptr, items = sequences_from_csr(m)
    assert list(indptr) == [0, 3, 3, 6]
    assert list(items) == [7, 1, 4, 9, 0, 3]               # by time; explicit 0 is a read; tie at 2 by column
    with pytest.raises(ValueError):
        sequences_from_csr(np.zeros((2, 2)))


def test_negative_mapping():
    n = 7
    c = (np.arange(1 << 16, dtype=np.uint64) * np.uint64(65537)) & np.uint64(0xFFFFFFFF)   # an even spread of 32-bit draws
    for pos in range(n):
        neg = negatives_from_draws(np.full(c.size, pos), c, n)
        assert (neg != pos).all() and neg.min() >= 0 and neg.max() < n
        cnt = np.bincount(neg, minlength=n)
        assert cnt[pos] == 0
        others = np.delete(cnt, pos)
        assert others.max() - others.min() <= 1 + c.size // (1 << 12)
    # extreme draws: c = 0 gives pos + 1, c = 2^32 - 1 gives pos - 1 (mod n)
    assert negatives_from_draws([3], [0], n)[0] == 4
    assert negatives_from_draws([3], [0xFFFFFFFF], n)[0] == 2


def test_state_dict_names_and_torch_round_trip():
    m = UserGRU(6, device='cpu')
    sd = m.state_dict()
    g = torch.nn.GRU(6, 6)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in g.state_dict().items()}
    g.load_state_dict(sd)
    m2 = UserGRU(6, seed=5, device='cpu')
    m2.load_state_dict(g.state_dict())
    for k in NAMES:
        assert torch.equal(m2.state_dict()[k], sd[k])


def test_save_load(tmp_path):
    m = UserGRU(5, max_len=7, seed=3, device='cpu')
    m.save(tmp_path / 'u.npz')
    m2 = UserGRU.load(tmp_path / 'u.npz', device='cpu')
    assert m2.dim == 5 and m2.max_len == 7
    for k in NAMES:
        assert torch.equal(m2.state_dict()[k], m.state_dict()[k])


def test_oracle_forward_matches_torch_gru_padded():
    rng = np.random.default_rng(1)
    H, N = 9, 30
    emb = rng.standard_normal((N, H))
    g = torch.nn.GRU(H, H, batch_first=True).double()
    params = {k: v.detach().clone() for k, v in g.state_dict().items()}
    seqs = [rng.integers(0, N, L) for L in (6, 1, 3, 6)]
    hs = gru_states(params, seqs, emb)
    x = torch.zeros(len(seqs), 6, H, dtype=torch.float64)
    for u, s in enumerate(seqs):
        x[u, :len(s)] = torch.as_tensor(emb[s])
    with torch.no_grad():
        y, _ = g(x)
    for u, s in enumerate(seqs):
        np.testing.assert_allclose(hs[u].detach().numpy(), y[u, :len(s)].numpy(), rtol=1e-12, atol=1e-12)


def test_make_sequences():
    from dae_rnn_news_recommendation_b200.synth import make_sequences
    labels = np.repeat(np.arange(6), 100)
    labels[:10] = -1
    indptr, items, targets = make_sequences(2000, labels, mean_len=20, session_len=5, seed=3)
    lens = np.diff(indptr)
    assert lens.min() >= 1 and abs(lens.mean() - 20) < 2
    assert (labels[items] >= 0).all()
    per_user = [np.unique(labels[items[indptr[u]:indptr[u + 1]]]).size for u in range(2000)]
    assert max(per_user) <= 3
    # consecutive reads share a class far more often than independent draws from 2-3 classes would
    same = (labels[items[1:]] == labels[items[:-1]])[np.diff(np.repeat(np.arange(2000), lens)) == 0].mean()
    assert same > 0.75
    ok = targets >= 0
    assert ok.mean() > 0.95
    for u in np.flatnonzero(ok)[:200]:
        s = items[indptr[u]:indptr[u + 1]]
        assert targets[u] not in s
    last = np.array([labels[items[indptr[u + 1] - 1]] for u in range(2000)])
    assert (labels[targets[ok]] == last[ok]).mean() > 0.7
    again = make_sequences(2000, labels, seed=3)
    assert all(np.array_equal(a, b) for a, b in zip(again, (indptr, items, targets)))


def test_input_validation():
    with pytest.raises(ValueError, match='indptr'):
        check_sequences((np.array([0, 3, 2]), np.zeros(2, np.int32)), 10, 'f')
    with pytest.raises(ValueError, match='indptr'):
        check_sequences((np.array([1, 2]), np.zeros(2, np.int32)), 10, 'f')
    with pytest.raises(ValueError, match='outside'):
        check_sequences((np.array([0, 2]), np.array([0, 10])), 10, 'f')
    with pytest.raises(ValueError, match='outside'):
        check_sequences((np.array([0, 2]), np.array([-1, 3])), 10, 'f')
    with pytest.raises(ValueError, match='pair'):
        check_sequences(np.zeros(3), 10, 'f')
    m = UserGRU(4, device='cpu')
    with pytest.raises(ValueError, match='H = 4'):
        m.transform((np.array([0, 1]), np.array([0])), np.zeros((5, 3), np.float32))
    with pytest.raises(ValueError, match='shape'):
        m.load_state_dict({k: np.zeros((2, 2)) for k in NAMES})
    with pytest.raises(ValueError):
        UserGRU(4, opt='rmsprop', device='cpu')
