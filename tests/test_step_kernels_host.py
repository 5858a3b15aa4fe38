"""CPU checks of tests/step_kernel_oracle.py: its references agree with the autograd oracle (oracle/dae_oracle.py) for every
activation x loss, its scales bound the values they belong to, and its CSR builders reach the edges the GPU kernel tests rely on."""
import numpy as np
import pytest
import torch

import step_kernel_oracle as so
from oracle import dae_oracle as do


def _close(a, b, tol=1e-10):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    assert np.all(np.abs(a - b) <= tol * (1.0 + np.abs(b))), float(np.max(np.abs(a - b)))


@pytest.mark.parametrize('enc', so.ACTS)
@pytest.mark.parametrize('dec', so.ACTS)
@pytest.mark.parametrize('loss', so.LOSSES)
def test_references_match_autograd(enc, dec, loss):
    """One fp64 forward / backward of the step through dae_oracle (autograd): E, the row losses, dL/dZ, dA, dbh and the sparse dW
    equal the closed forms of step_kernel_oracle."""
    B, F, H = 7, 40, 5
    rng = np.random.default_rng(9 * so.ACTS.index(enc) + 3 * so.ACTS.index(dec) + so.LOSSES.index(loss))
    x = so.edge_csr(B, F, mean_nnz=6, kind='binary' if loss == 'cross_entropy' else 'tfidf', seed=3, long_row=False)
    xc = so.mask_values(x, 0.3, seed=4)
    in_scale = 0.75
    W = rng.normal(0, 0.4, (F, H))
    bh = rng.normal(0, 0.3, H)
    bv = rng.normal(0, 0.3, F)
    if loss == 'cross_entropy' and dec != 'sigmoid':   # keep D inside (0, 1) where the loss is finite
        W *= 0.05
        bv = rng.uniform(0.3, 0.7, F)
    w = rng.random(B) * 2
    w[2] = 0.0
    t = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    Wt, bht, bvt = t(W), t(bh), t(bv)
    Xc = torch.from_numpy(np.asarray(xc.todense(), np.float64)) * in_scale
    A = Xc @ Wt + bht
    A.retain_grad()
    E = do._act(enc)(A) - do._act(enc)(bht)     # do.encode, with A kept for its gradient
    E.retain_grad()
    _close(E.detach().numpy(), do.encode(Xc, Wt, bht, enc).detach().numpy(), 1e-14)
    z = E @ Wt.t() + bvt
    z.retain_grad()
    D = do._act(dec)(z)
    xd = torch.from_numpy(np.asarray(x.todense(), np.float64))
    rl = do.row_loss(xd, D, loss)
    L = do.weighted_loss(xd, D, loss, torch.from_numpy(w))
    dE_extra = torch.from_numpy(rng.normal(0, 0.1, (B, H)))
    (L + (E * dE_extra).sum()).backward()

    E_ref, s_E, A_ref = so.encode_fwd(xc, W, bh, enc, in_scale)
    _close(E_ref, E.detach().numpy())
    _close(A_ref, A.detach().numpy())
    assert np.all(s_E >= np.abs(E_ref))

    dZ, s_dZ, lt, s_l = so.decode_loss(z.detach().numpy(), x, w, w.sum(), dec, loss)
    _close(dZ, z.grad.numpy())
    _close(lt.sum(1), rl.detach().numpy())
    assert np.all(s_dZ >= np.abs(dZ) * (1 - 1e-12)) and np.all(s_l.sum(1) >= np.abs(lt.sum(1)) * (1 - 1e-12))

    # the encode backward gets dL/dE (decode path + the extra term), as the step hands it over: dE = dZ W, dE_add = the extra term
    dE_dec = E.grad.numpy() - dE_extra.numpy()
    r = so.encode_bwd(xc, E_ref, dE_dec, dE_extra.numpy(), bh, enc, in_scale)
    _close(r['dA'][0], A.grad.numpy(), 1e-9)
    _close(r['dbh'][0], bht.grad.numpy(), 1e-9)
    # W's gradient = the sparse encode part + the dense decode part dZ^T E
    _close(r['dW'][0] + dZ.T @ E.detach().numpy(), Wt.grad.numpy(), 1e-9)
    _close(dZ.sum(0), bvt.grad.numpy(), 1e-9)
    for k in ('dA', 'dbh', 'dW'):
        assert np.all(r[k][1] >= np.abs(r[k][0]) * (1 - 1e-12)), k


def test_decode_saturation_follows_fp32_model():
    """Where sigmoid(z) rounds to 1 in fp32, D = 1: CE gives -log(1e-16) for x = 0 and a zero dZ, as the fp32 model computes."""
    z = np.array([[90.0, -90.0, 0.5, 30.0]])
    x = np.array([[0.0, 1.0, 1.0, 1.0]])
    dZ, s_dZ, lt, _ = so.decode_loss(z, x, None, 1.0, 'sigmoid', 'cross_entropy')
    assert dZ[0, 0] == 0.0 and dZ[0, 3] == 0.0 and s_dZ[0, 0] == 0.0
    assert abs(lt[0, 0] + np.log(1e-16)) < 1e-12 and abs(lt[0, 1] + np.log(1e-16)) < 1e-9 and lt[0, 3] == 0.0


@pytest.mark.parametrize('opt', ['gradient_descent', 'ada_grad', 'momentum', 'adam'])
def test_optimizer_reference_matches_oracle(opt):
    """Five steps of optimizer_steps == five OracleDAE.apply_gradients in fp64 (the TF-1.12 rules)."""
    F, H = 6, 3
    rng = np.random.default_rng(5)
    W0 = rng.normal(0, 1, (F, H))
    o = do.OracleDAE(W0, opt=opt, learning_rate=0.05, momentum=0.7, triplet_strategy='none', dtype=torch.float64)
    theta = np.concatenate([W0.ravel(), np.zeros(H), np.zeros(F)])
    grads = [rng.normal(0, 1, theta.size) for _ in range(5)]
    for g in grads:
        o.apply_gradients([torch.from_numpy(g[:F * H].reshape(F, H)), torch.from_numpy(g[F * H:F * H + H]),
                           torch.from_numpy(g[F * H + H:])])
    s1 = np.full(theta.size, 0.1) if opt == 'ada_grad' else None
    p, _, _, scale = so.optimizer_steps(opt, theta, grads, 0.05, momentum=0.7, slot1=s1, fp32_betas=False)
    want = np.concatenate([o.W.detach().numpy().ravel(), o.bh.detach().numpy(), o.bv.detach().numpy()])
    _close(p, want, 1e-12)
    assert np.all(scale >= np.abs(p))
    p32 = so.optimizer_steps(opt, theta, grads, 0.05, momentum=0.7, slot1=s1)[0]   # fp32 betas: Adam moves by O(1e-5) of lr
    _close(p32, want, 1e-12 if opt != 'adam' else 1e-4)


def test_bf16_split_matches_torch():
    x = np.random.default_rng(0).normal(0, 3, 1000).astype(np.float32)
    x[:4] = [0.0, -0.0, 1e-30, 3.0e38]
    hi, lo = so.bf16_split(x)
    t = torch.from_numpy(x)
    th = t.to(torch.bfloat16)
    tl = (t - th.float()).to(torch.bfloat16)
    assert np.array_equal(hi, th.view(torch.int16).numpy().view(np.uint16))
    assert np.array_equal(lo, tl.view(torch.int16).numpy().view(np.uint16))


@pytest.mark.parametrize('F', [8, 63, 129, 1000, 8193])
def test_edge_csr_reaches_the_edges(F):
    n = 160
    m = so.edge_csr(n, F, mean_nnz=10, seed=1)
    m2 = m.copy()
    m2.sort_indices()
    assert np.array_equal(m.indices, m2.indices) and m.has_canonical_format
    stored = set(m.indices.tolist())
    assert {0, F - 1} <= stored
    assert set(so.boundary_columns(F).tolist()) <= stored
    for b in (16, 64, 128):
        for c in range(b, F, b):
            assert {c - 1, c} <= stored
    assert m.indptr[4] == m.indptr[3]                                     # an empty row
    row = lambda i: m.indices[m.indptr[i]:m.indptr[i + 1]]
    chunk = np.bincount(row(2) // 16)
    assert chunk.max() > 3                                                 # > 3 stored entries in one 16-column chunk
    if F >= 64:
        half = np.bincount(row(1) // 64)
        assert half.max() == 64                                            # a fully stored 64-column half tile
    if F > 600:
        assert len(row(4)) > 512
    if F > 8:
        assert np.bincount(m.indices, minlength=F).max() > 64              # one column crosses chunks of 32 and 64 entries
    xc = so.mask_values(m, 0.3, seed=2)
    assert np.all(xc.data[xc.indptr[5]:xc.indptr[6]] == 0) and xc.indptr[6] > xc.indptr[5]
