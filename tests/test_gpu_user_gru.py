"""GRU user encoder on the GPU (user_model.UserGRU) against the fp64 oracle (tests/user_gru_oracle.py), its recommendations, the
learning check on make_sequences data and the CLI's --user_sequences."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import rel_err  # noqa: E402
from user_gru_oracle import NAMES, adam_tf, gru_states, loss_and_grads  # noqa: E402

from dae_rnn_news_recommendation_b200.user_model import Packed, UserGRU, history_matrix, negatives_from_draws  # noqa: E402

M32 = np.uint64(0xFFFFFFFF)


def _philox_first_word(p, batch, epoch, seed):
    """Philox4x32-10's first output word at counter (p, batch, epoch lo, epoch hi), key seed (NumPy, uint64 lanes)."""
    c = [np.asarray(p, np.uint64) & M32, np.full(np.shape(p), batch, np.uint64), np.full(np.shape(p), epoch & 0xFFFFFFFF, np.uint64),
         np.full(np.shape(p), epoch >> 32, np.uint64)]
    k = [np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)]
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & M32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & M32]
        k = [(k[0] + np.uint64(0x9E3779B9)) & M32, (k[1] + np.uint64(0xBB67AE85)) & M32]
    return c[0]


def _data(U, H, N, max_len, seed):
    """Lengths covering 1, 2, max_len and longer than max_len, plus random ones; embeddings of moderate scale."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 4, U)
    lens[:6] = [1, 2, max_len, max_len + 3, 2 * max_len, 1]
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    items = rng.integers(0, N, int(indptr[-1])).astype(np.int32)
    emb = (rng.standard_normal((N, H)) * 0.5).astype(np.float32)
    return indptr, items, emb


def _params(m):
    return {k: v.double().numpy() for k, v in m.state_dict().items()}


def _grads(m):
    H, g = m.dim, m.grad.cpu().double().numpy()
    hh, ih = g[:m.nW].reshape(3 * H, H + 1), g[m.nW:].reshape(3 * H, H + 1)
    return {'weight_ih_l0': ih[:, :H], 'weight_hh_l0': hh[:, :H], 'bias_ih_l0': ih[:, H], 'bias_hh_l0': hh[:, H]}


def _batch(m, pk, emb_d, epoch=0, batch=0):
    m.stats.zero_()
    m._forward_backward(pk, emb_d, epoch, batch)
    torch.cuda.synchronize()
    b = m._buf
    neg = b['neg'][:pk.P].cpu().numpy()
    Hs = b['Hs'][:pk.P].cpu().double().numpy()
    seqs, negs, states = [], [], []
    for i in range(pk.B):
        pos = [pk.position(i, t) for t in range(int(pk.L[i]))]
        seqs.append(pk.items[pos])
        negs.append(neg[pos[:-1]])
        states.append(Hs[pos])
    return float(m.stats.item()) / pk.terms, seqs, negs, states, neg


@pytest.mark.parametrize('H,U,max_len', [(37, 300, 10), (500, 140, 8)])
def test_batch_against_oracle(H, U, max_len):
    N = 900
    indptr, items, emb = _data(U, H, N, max_len, seed=H)
    m = UserGRU(H, max_len=max_len, batch_users=U, seed=1)
    pk = Packed(indptr, items, np.arange(U), max_len)
    loss, seqs, negs, states, neg = _batch(m, pk, torch.from_numpy(emb).cuda(), epoch=3, batch=7)
    # negatives: Philox restated on the host, never the positive
    has = pk.nxt >= 0
    c = _philox_first_word(np.flatnonzero(has), 7, 3, 1)
    assert np.array_equal(neg[has], negatives_from_draws(pk.nxt[has], c, N))
    assert (neg[~has] == -1).all() and (neg[has] != pk.nxt[has]).all()
    o_loss, o_grads, o_states = loss_and_grads(_params(m), seqs, negs, emb)
    assert rel_err(np.concatenate(states), np.concatenate(o_states)) < 1e-4
    assert rel_err(loss, o_loss) < 1e-4, (loss, o_loss)
    g = _grads(m)
    for k in NAMES:
        assert rel_err(g[k], o_grads[k]) < 1e-4, (k, rel_err(g[k], o_grads[k]))


def test_adam_five_steps():
    H, U, N, max_len = 37, 200, 500, 9
    indptr, items, emb = _data(U, H, N, max_len, seed=5)
    m = UserGRU(H, max_len=max_len, batch_users=U, seed=2, learning_rate=1e-2)
    pk = Packed(indptr, items, np.arange(U), max_len)
    emb_d = torch.from_numpy(emb).cuda()
    p = _params(m)
    mom = {k: np.zeros_like(v) for k, v in p.items()}
    vel = {k: np.zeros_like(v) for k, v in p.items()}
    for step in range(1, 6):
        _, seqs, negs, _, _ = _batch(m, pk, emb_d)
        m._optimizer_step()
        _, g, _ = loss_and_grads(p, seqs, negs, emb)
        for k in NAMES:
            adam_tf(p[k], g[k], mom[k], vel[k], step, 1e-2)
    got = _params(m)
    for k in NAMES:
        assert rel_err(got[k], p[k]) < 5e-3, (k, rel_err(got[k], p[k]))


def test_transform_oracle_batch_invariance_and_training_states():
    H, U, N, max_len = 37, 333, 700, 12
    indptr, items, emb = _data(U, H, N, max_len, seed=9)
    indptr = np.concatenate([indptr[:5], [indptr[4]], indptr[5:]])   # one user without reads
    U += 1
    m = UserGRU(H, max_len=max_len, batch_users=U, seed=4)
    out = m.transform((indptr, items), emb)
    assert out.shape == (U, H) and out.dtype == np.float32
    assert not out[4].any()
    seqs = [items[indptr[u]:indptr[u + 1]][-max_len:] for u in range(U)]
    p = {k: torch.from_numpy(v) for k, v in _params(m).items()}
    want = np.stack([h[-1].detach().numpy() if len(h) else np.zeros(H) for h in gru_states(p, seqs, emb)])
    assert rel_err(out, want) < 1e-4
    assert np.array_equal(m.transform((indptr, items), emb, to_host=False).cpu().numpy(), out)   # no wait on the host in between
    m.batch_users = 77
    assert rel_err(m.transform((indptr, items), emb), out) < 1e-6
    # the training forward's last states
    pk = Packed(indptr, items, np.arange(U), max_len)
    m._buffers(pk.P, pk.B)
    _, _, _, states, _ = _batch(m, pk, torch.from_numpy(emb).cuda())
    last = np.stack([s[-1] for s in states])
    assert rel_err(last, out[pk.order]) < 1e-6
    # a CPU torch.nn.GRU loaded from the state dict reproduces transform
    g = torch.nn.GRU(H, H, batch_first=True)
    g.load_state_dict(m.state_dict())
    for u in (0, 1, 2, 3, 100):
        with torch.no_grad():
            y, _ = g(torch.from_numpy(emb[seqs[u]])[None])
        assert rel_err(out[u], y[0, -1].numpy()) < 1e-4


def _clustered(N, H, classes, seed, spread=0.6):
    rng = np.random.default_rng(seed)
    labels = rng.integers(0, classes, N)
    emb = (rng.standard_normal((classes, H))[labels] + spread * rng.standard_normal((N, H))).astype(np.float32) / np.sqrt(H)
    return labels, emb


def test_recommend_exclusions_padding_candidates():
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.synth import make_sequences
    N, H = 1500, 48
    labels, emb = _clustered(N, H, 6, 0)
    indptr, items, _ = make_sequences(400, labels, mean_len=30, seed=1, holdout=False)
    indptr = np.concatenate([[0, 0], indptr[1:]])                                     # user 0 reads nothing
    items = items.copy()
    m = UserGRU(H, max_len=10, seed=0, num_epochs=1).fit((indptr, items), emb)
    seq_copy = (indptr.copy(), items.copy())
    idx, score = m.recommend((indptr, items), emb, k=10)
    assert np.array_equal(indptr, seq_copy[0]) and np.array_equal(items, seq_copy[1])    # the caller's arrays are left as they were
    U = len(indptr) - 1
    assert idx.shape == (U, 10) and (idx[0] == -1).all() and np.isneginf(score[0]).all()
    for u in range(1, U):
        assert not np.isin(idx[u], items[indptr[u]:indptr[u + 1]]).any()             # the whole history, beyond max_len
    prof = m.transform((indptr, items), emb)
    s = prof[1:] @ emb.T
    np.testing.assert_allclose(score[1:, 0], np.array([np.max(np.where(np.isin(np.arange(N), items[indptr[u]:indptr[u + 1]]), -np.inf,
                                                                              s[u - 1])) for u in range(1, U)]), rtol=1e-4, atol=1e-4)
    cand = np.arange(0, N, 3)
    ic, _ = m.recommend((indptr, items), emb, k=10, candidates=cand)
    assert np.isin(ic[1:], cand).all()
    for u in range(1, U):
        assert not np.isin(ic[u], items[indptr[u]:indptr[u + 1]]).any()
    # helpers.recommend: given profiles equal to the mean profiles reproduce the default path bit for bit
    hist = history_matrix(indptr, items, N)
    a = helpers.recommend(hist, emb, k=10)
    b = helpers.recommend(hist, emb, k=10, profiles=helpers.user_profiles(hist, emb))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    with pytest.raises(ValueError, match='profiles'):
        helpers.recommend(hist, emb, profiles=np.zeros((U, H + 1), np.float32))


def _learning_numbers():
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.synth import make_sequences
    N, H = 3000, 64
    labels, emb = _clustered(N, H, 8, 11)
    indptr, items, targets = make_sequences(8000, labels, mean_len=20, session_len=5, seed=12)
    U = len(indptr) - 1
    has = targets >= 0
    tg = sp.csr_matrix((np.ones(int(has.sum()), np.float32), (np.flatnonzero(has), targets[has])), shape=(U, N))
    m = UserGRU(H, max_len=50, batch_users=512, num_epochs=8, learning_rate=3e-3, seed=0).fit((indptr, items), emb)
    gru = helpers.recommendation_recall(m.recommend((indptr, items), emb, k=10)[0], tg)['hit_rate']
    hist = history_matrix(indptr, items, N)
    mean = helpers.recommendation_recall(helpers.recommend(hist, emb, k=10)[0], tg)['hit_rate']
    return gru, mean, m.train_loss


# hit@10 on the held-out next read measured on an H100 80GB HBM3: see DESIGN 4.10; the asserted margin is half the measured gap
LEARNING_MARGIN = 0.028


def test_learning_beats_mean_profile():
    gru, mean, losses = _learning_numbers()
    print('hit@10: GRU %.4f, mean profile %.4f; train loss %s' % (gru, mean, ['%.4f' % x for x in losses]))
    assert losses[-1] < losses[0]
    assert gru - mean > LEARNING_MARGIN, (gru, mean)


def test_cli_user_sequences(capsys, tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    from dae_rnn_news_recommendation_b200.synth import make_sequences
    argv = ['--model_name', 'synseq', '--synthetic', '1200', '--max_features', '2000', '--num_epochs', '2', '--batch_size', '200',
            '--seed', '3', '--top_k', '5']
    trX, _, trL, _ = cli.prepare_synthetic(cli.check_flags(cli.build_parser().parse_args(argv)))
    indptr, items, targets = make_sequences(300, trL, mean_len=8, seed=4)
    np.savez(tmp_path / 's.npz', indptr=indptr, items=items, targets=targets)
    model = cli.main(argv + ['--user_sequences', str(tmp_path / 's.npz'), '--user_epochs', '2'])
    printed = capsys.readouterr().out
    idx = np.load(model.data_dir + 'user_gru_top_k_index.npy')
    score = np.load(model.data_dir + 'user_gru_top_k_score.npy')
    assert idx.shape == score.shape == (300, 5) and idx.dtype == np.int32
    assert os.path.isfile(model.data_dir + 'user_gru.npz')
    assert 'users (GRU): hit rate@5' in printed and 'mean profile: hit rate@5' in printed
    for k in ('user_gru_hit_rate', 'user_gru_recall', 'user_mean_hit_rate', 'user_mean_recall'):
        assert 0.0 <= model.evaluation[k] <= 1.0
