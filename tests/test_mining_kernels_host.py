"""CPU checks of mining_kernel_oracle.py: its references against fp64 autograd of oracle/dae_oracle.py and against the reference's
brute-force loops, the fp32 positive-count helpers, the edge builders, and the two float32 facts behind the sweep's fixed
positive test and its series for small loss terms."""
import numpy as np
import pytest
import torch

import mining_kernel_oracle as mo
from oracle import dae_oracle as od


def _batch(sizes, H, seed, ties=True):
    """A label-sorted batch with integer-valued E (S exact in fp32 and fp64), ties in S planted by repeated rows."""
    lo, hi, lab, nv = mo.segments(sizes)
    rng = np.random.default_rng(seed)
    E = rng.integers(-2, 3, (len(lab), H)).astype(np.float64)
    if ties and len(lab) > 4:
        E[3] = E[1]
        E[-1] = E[0]
    return lo, hi, lab, nv, E


@pytest.mark.parametrize('sizes', [[3, 2, 4], [1, 5, 1, 2], [2, 2], [6]])
def test_batch_all_against_autograd_and_bruteforce(sizes):
    lo, hi, lab, nv, E = _batch(sizes, 3, seed=len(sizes))
    B = len(lab)
    Et = torch.tensor(E, dtype=torch.float64, requires_grad=True)
    loss, w, frac, npos = od.batch_all_triplet_loss(torch.tensor(lab), Et)
    loss.backward()
    S32 = torch.tensor(E @ E.T, dtype=torch.float32)
    G, Gs, l, ls, cnt, _ = mo.batch_all_rows(S32, np.arange(B), lo, hi, nv)
    assert np.allclose((G + G.T) @ E, Et.grad.numpy(), rtol=1e-12, atol=1e-15)     # G = dL/dS: dL/dE = (G + G^T) E
    assert l.sum() / (nv + 1e-16) == pytest.approx(loss.item(), rel=1e-12, abs=1e-15)
    assert cnt.sum() == int(npos)
    assert np.array_equal(mo.count_all(S32, lo, hi), cnt)
    bf = od.batch_all_bruteforce(lab, E)
    assert cnt.sum() == bf['num']
    assert l.sum() / (nv + 1e-16) == pytest.approx(bf['loss'], rel=1e-12, abs=1e-15)
    # pos_triplets_only: counts in G, the loss over positive triplets
    Gp, _, lp, _, cp, _ = mo.batch_all_rows(S32, np.arange(B), lo, hi, nv, pos_only=True)
    assert np.array_equal(cp, cnt)
    assert lp.sum() / (cp.sum() + 1e-16) == pytest.approx(bf['loss_pos'], rel=1e-12, abs=1e-15)
    assert np.all(Gp.sum(1) == 0.0)
    assert np.array_equal(-np.where(Gp < 0, Gp, 0).sum(1), cp.astype(np.float64))


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_batch_hard_against_autograd_and_bruteforce(seed):
    sizes = [3, 4, 2, 2, 3]      # no singleton: the brute force loop has no hardest positive for one
    _, _, lab, _, E = _batch(sizes, 2, seed=seed)
    E = np.abs(E) + 1.0     # S > 0: the graph's masked zeros and row max never win, as in the brute force loop
    rng = np.random.default_rng(seed)
    perm = rng.permutation(len(lab))          # batch_hard needs no sorted order
    lab, E = lab[perm], E[perm]
    B = len(lab)
    Et = torch.tensor(E, dtype=torch.float64, requires_grad=True)
    loss, w, frac, num = od.batch_hard_triplet_loss(torch.tensor(lab), Et)
    loss.backward()
    S32 = (E @ E.T).astype(np.float32)
    ref = mo.batch_hard_rows(S32, lab, np.arange(B))
    na = float(ref['active'].sum())
    G, _ = mo.batch_hard_scaled(ref, na)
    assert np.allclose((G + G.T) @ E, Et.grad.numpy(), rtol=1e-12, atol=1e-15)
    assert np.array_equal(ref['weight'], w.detach().numpy())
    assert na == float(num)
    assert ref['softplus'].sum() / (na + 1e-16) == pytest.approx(float(loss), rel=1e-12, abs=1e-15)
    bf = od.batch_hard_bruteforce(lab, E)
    assert bf['num'] == na
    assert ref['softplus'].sum() / (na + 1e-16) == pytest.approx(bf['loss'], rel=1e-12, abs=1e-15)


def test_batch_hard_masked_ties():
    """All negatives below zero: hn = 0 is taken by the masked zeros; a singleton reaches hp through the row max (dm path)."""
    lab = np.array([0, 0, 1, 2], np.float32)
    E = np.array([[2.0, 0.0], [-1.0, 1.0], [-1.0, 0.0], [-0.5, -2.0]])
    Et = torch.tensor(E, requires_grad=True)
    loss, w, _, num = od.batch_hard_triplet_loss(torch.tensor(lab), Et)
    loss.backward()
    S32 = (E @ E.T).astype(np.float32)
    ref = mo.batch_hard_rows(S32, lab, np.arange(4))
    G, _ = mo.batch_hard_scaled(ref, float(ref['active'].sum()))
    assert np.allclose((G + G.T) @ E, Et.grad.numpy(), rtol=1e-12, atol=1e-15)
    assert np.array_equal(ref['weight'], w.detach().numpy())
    assert (S32[0, 2:] < 0).all() and ref['active'][0]


@pytest.mark.parametrize('H', [1, 5, 40])
def test_explicit_against_autograd(H):
    rng = np.random.default_rng(H)
    B, alpha = 6, 0.7
    E, Ep, En = (rng.normal(0, 3, (B, H)) for _ in range(3))
    ts = [torch.tensor(a, requires_grad=True) for a in (E, Ep, En)]
    loss = od.explicit_triplet_loss(*ts) * float(np.float32(alpha))
    loss.backward()
    z = np.zeros((B, H))
    ref = mo.explicit(E, Ep, En, alpha, z, z, z)
    for t, name in zip(ts, ('dE', 'dEp', 'dEn')):
        assert np.allclose(ref[name][0], t.grad.numpy(), rtol=1e-12, atol=1e-15)
    assert ref['loss'][0].mean() * float(np.float32(alpha)) == pytest.approx(float(loss), rel=1e-12)


def test_count_helpers_follow_the_reference_expression():
    rng = np.random.default_rng(0)
    for e in (-40, -34, -31, -30, -29, -20, 0):
        sj = (rng.normal(0, 1, 50) * 2.0 ** e).astype(np.float32)
        sk = np.concatenate([sj, np.nextafter(sj, np.float32(np.inf)), (rng.normal(0, 1, 50) * 2.0 ** e)]).astype(np.float32)
        want = sum(int(np.float32(b) - np.float32(a) > np.float32(1e-16)) for a in sj for b in sk)
        assert mo.count_positive(sj, sk) == want
        assert mo.count_positive(torch.from_numpy(sj), torch.from_numpy(sk)) == want
        thr = np.array([mo.pos_threshold(a) for a in sj])
        assert int((sk[None, :] > thr[:, None]).sum()) == want


def test_pos_threshold_is_the_largest_non_positive_value():
    rng = np.random.default_rng(1)
    vals = np.concatenate([rng.normal(0, 1, 200) * 2.0 ** rng.integers(-60, -20, 200), [0.0, -1e-16, 1e-16, -2e-16, 2.0 ** -29,
                                                                                        -(2.0 ** -29), 2.0 ** -30]])
    for a in vals.astype(np.float32):
        t = mo.pos_threshold(a)
        nxt = np.nextafter(t, np.float32(np.inf))
        assert np.float32(t - a) <= np.float32(1e-16) < np.float32(nxt - a), a


def test_finding_positive_band():
    """The reference counts S_ik = nextafter(S_ij) as positive at S_ij = 1.5 * 2^-30; the test S_ik > fp32(S_ij + 1e-16) does not."""
    a = np.float32(1.5 * 2.0 ** -30)
    b = np.nextafter(a, np.float32(np.inf))
    assert np.float32(b - a) > np.float32(1e-16)
    assert not (b > np.float32(a + np.float32(1e-16)))
    assert mo.pos_threshold(a) == a
    for a, b in mo.band_pairs(20):
        assert (np.float32(b - a) > np.float32(1e-16)) != (b > np.float32(a + np.float32(1e-16)))
        e = np.floor(np.log2(abs(float(a))))
        assert e in (-35, -32, -31, -30)


def test_finding_small_loss_terms():
    """fp32's 1 + e^-17 is 1, so lg2(1 + e) loses the term: below e = 2^-12 the sweep adds the series (e - e^2 / 2) / ln 2, within
    e^2 / 3 <= 2^-25 of the term, evaluated in fp32 as fma(-e / 2, e, e)."""
    assert np.float32(1) + np.float32(np.exp(-17.0)) == 1
    assert np.log1p(np.exp(-17.0)) > 0.0
    for e in (2.0 ** -12, 2.0 ** -24, np.exp(-80.0)):
        assert abs((e - e * e / 2) - np.log1p(e)) <= (e * e / 3 + 2.0 ** -50) * np.log1p(e)   # (+ fp64 rounding)
        e32 = np.float32(e)
        series = np.float32(np.float64(np.float32(-0.5) * e32) * np.float64(e32) + np.float64(e32))   # one fp32 fma
        assert abs(float(series) - np.log1p(float(e32))) <= 2.0 ** -23 * np.log1p(float(e32))


def test_edge_builders():
    lo, hi, lab, nv = mo.segments([1, 2, 31, 32, 33, 511, 512, 513])
    assert np.array_equal(np.unique(hi - lo), [1, 2, 31, 32, 33, 511, 512, 513])
    assert np.all(lab[lo] == lab) and np.all(lab[hi - 1] == lab)
    n = hi - lo
    B = len(lab)
    assert nv == float(np.sum((n - 1.0) * (B - n)))
    for R, tier in ((9.99, 0), (10.0, 1), (79.99, 1), (80.0, 2), (500.0, 2)):
        h = np.float32(R * 0.5)
        row = np.array([-h, 0.0, h], np.float32)
        assert mo.tier_of(row) == tier
    S = torch.tensor([0.0, 1.0, 1.0, 1.5, 0.0])     # anchor 0, positive 1; negatives: a tie, one above, one below
    out = mo.batch_all_anchor(S, 0, 0, 2, 3.0)
    assert out['count'] == 1 and out['tier'] == 0
    assert out['g'][2].item() == pytest.approx(0.5 / 3.0, rel=1e-15)     # sigma(0) / NV at the tie
