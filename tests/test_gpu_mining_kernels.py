"""The mining branch of the training step called kernel by kernel through the C ABI, against the fp64 references of
mining_kernel_oracle.py, element by element (|got - want| <= c * scale + tiny; the scales are derived there): the Gram, sym and
block dE2 GEMMs and their operand splits, the batch_all sweep (shared-memory and tiled, plain and deterministic, the anchor-row
blocks), batch_hard, the explicit triplets and the step finalize.  S is built directly, not from E, so that each edge of the
sweep is reached on purpose; G rows depend only on their own row of S, so at large B a chosen set of anchors is checked in full:
every edge anchor and a random sample."""
import numpy as np
import pytest
import torch

import mining_kernel_oracle as mo

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SENT = -7.0          # sentinel for memory a kernel must not touch
BF16_SENT = 0x7F7F   # a bf16 bit pattern no kernel writes here (3.4e38)
STAT_NUM, STAT_SUM_W, STAT_N_VALID, STAT_TSUM, STAT_N_ACTIVE = 4, 5, 6, 8, 9


def _cabi():
    from dae_rnn_news_recommendation_b200 import _cabi
    return _cabi


def _call(name, *args):
    _cabi().call(name, *args)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _np(t):
    torch.cuda.synchronize()
    return t.detach().cpu().numpy().astype(np.float64)


def _check(name, got, want, scale, c=mo.C_HEAD, tiny=1e-30):
    """Element-wise |got - want| <= c * scale + tiny; returns the worst err / bound (printed, so that a run with -s shows how
    tight each bound is)."""
    got = np.atleast_1d(np.asarray(got, np.float64))
    want = np.atleast_1d(np.asarray(want, np.float64))
    scale = np.atleast_1d(np.asarray(scale, np.float64))
    err = np.abs(got - want)
    bound = c * scale + tiny
    bad = ~(err <= bound)
    ratio = np.where(np.isfinite(err), err / bound, np.inf)
    worst = float(ratio.max()) if ratio.size else 0.0
    print('ratio %-40s %.3e' % (name, worst))
    if bad.any():
        idx = np.argwhere(bad)[:5]
        w = np.unravel_index(np.argmax(ratio), err.shape)
        raise AssertionError('%s: %d of %d elements outside c*scale (c=%g); first %s; worst at %s: got %r want %r scale %r' %
                             (name, int(bad.sum()), bad.size, c, idx.tolist(), w, got[w], want[w], scale[w]))
    return worst


def _bits16(t):
    torch.cuda.synchronize()
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def _bf16_sentinel(rows, cols):
    return torch.full((rows, cols), BF16_SENT, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def _split_bits_ok(G, gh, gl, B):
    """g_hi / g_lo equal the bf16 split of G bit for bit in columns < B and keep their sentinels beyond."""
    h = G[:, :B].to(torch.bfloat16)
    l = (G[:, :B] - h.float()).to(torch.bfloat16)
    assert torch.equal(gh[:, :B].view(torch.int16), h.view(torch.int16))
    assert torch.equal(gl[:, :B].view(torch.int16), l.view(torch.int16))
    assert bool((gh[:, B:].view(torch.int16) == BF16_SENT).all()) and bool((gl[:, B:].view(torch.int16) == BF16_SENT).all())


# ---------------------------------------------------------------------------------------------------------------------------------
# batch_all: S builders
# ---------------------------------------------------------------------------------------------------------------------------------
RANGES = (9.99, 10.0, 79.99, 80.0, 500.0, 3.0, 30.0)   # tier 0 / 1 and 1 / 2 edges, deep tier 2, typical tier-0 and tier-1 rows


def _base_S(B, lds, seed):
    """Rows of uniform values whose ranges cycle through RANGES, each range planted exactly (its min and max), NaN beyond B."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    R = torch.tensor([RANGES[r % len(RANGES)] for r in range(B)], dtype=torch.float32, device=DEV)
    half = (R * 0.5)[:, None]
    S = torch.full((B, lds), float('nan'), device=DEV)
    S[:, :B] = (torch.rand(B, B, generator=g, device=DEV) - 0.5) * R[:, None]
    if B >= 2:
        c0 = torch.randint(0, B, (B,), generator=g, device=DEV)
        c1 = (c0 + 1 + torch.randint(0, B - 1, (B,), generator=g, device=DEV)) % B
        r = torch.arange(B, device=DEV)
        S[r, c0] = -half[:, 0]
        S[r, c1] = half[:, 0]
    return S


def _pos_neg(B, lo, hi, i):
    pidx = np.r_[lo:i, i + 1:hi]
    kidx = np.r_[0:lo, hi:B]
    return pidx, kidx


def _plant_ties(S, B, lo, hi, i):
    """Exact ties S_ik = S_ij for up to 5 (j, k) of anchor i; the negatives holding the row's min and max are left alone, so its
    range (its tier) is unchanged.  Returns the number of ties planted."""
    pidx, kidx = _pos_neg(B, lo, hi, i)
    row = S[i, :B]
    keep = {int(row.argmin()), int(row.argmax())}
    kidx = np.array([k for k in kidx if k not in keep], np.int64)
    m = min(len(pidx), len(kidx), 5)
    if m == 0:
        return 0
    before = float(row.max() - row.min())
    kt, pt = torch.from_numpy(kidx[:m]).to(DEV), torch.from_numpy(pidx[:m]).to(DEV)
    S[i, kt] = S[i, pt]
    assert bool((S[i, kt] == S[i, pt]).all()) and float(S[i, :B].max() - S[i, :B].min()) == before
    return m


def _plant_far(S, B, lo, hi, i, tier, seed):
    """Every triplet of anchor i separated by 17 to 80 (tier 2: x in [-80, -17], range 80) or 17 to 55 (tier 1): the loss terms
    are e^x, 1e-35 to 4e-8, below fp32's 1 + e."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    (p0, p1), (n0, n1) = ((20.0, 30.0), (-50.0, 3.0)) if tier == 2 else ((10.0, 15.0), (-40.0, -7.0))
    seg = torch.arange(lo, hi, device=DEV)
    S[i, :B] = n0 + (n1 - n0) * torch.rand(B, generator=g, device=DEV)
    S[i, seg] = p0 + (p1 - p0) * torch.rand(hi - lo, generator=g, device=DEV)
    S[i, lo] = p1
    _, kidx = _pos_neg(B, lo, hi, i)
    S[i, int(kidx[0])] = n0


def _plant_band(S, B, lo, hi, i, seed):
    """Anchor i's row in the 2^-30 band: its positives take values a and its negatives the values b just past the reference's
    threshold for them (mo.band_pairs), where fp32(b - a) > 1e-16 but b <= fp32(a + 1e-16)."""
    pidx, kidx = _pos_neg(B, lo, hi, i)
    pairs = mo.band_pairs(max(1, min(len(pidx), len(kidx), 64)), seed=seed)
    a = np.array([p[0] for p in pairs], np.float32)
    b = np.array([p[1] for p in pairs], np.float32)
    S[i, :B] = torch.from_numpy(np.resize(b, B)).to(DEV)
    S[i, torch.from_numpy(np.r_[lo:hi]).to(DEV)] = torch.from_numpy(np.resize(a, hi - lo)).to(DEV)


def _edge_anchors(lo, hi, B, extra, seed, n_random=6):
    """first / last anchors of every segment, both sides of the 512-row positive chunk, the given extra anchors, a random sample"""
    out = set(int(a) for a in extra)
    for s0 in np.unique(lo):
        s1 = int(hi[s0])
        for a in (s0, s0 + 1, s1 - 2, s1 - 1, s0 + 511, s0 + 512, s0 + 513):
            if s0 <= a < s1:
                out.add(int(a))
    rng = np.random.default_rng(seed)
    out.update(rng.choice(B, size=min(B, n_random), replace=False).tolist())
    return np.array(sorted(out), np.int64)


def _sweep(name, S, lds, B, lo_d, hi_d, nv, pos_only, ldg, ld_split, slots=None):
    G = torch.full((B, ldg), SENT, device=DEV)
    gh, gl = _bf16_sentinel(B, ld_split), _bf16_sentinel(B, ld_split)
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    stats[STAT_N_VALID] = nv
    args = [S.data_ptr(), lds, B, lo_d.data_ptr(), hi_d.data_ptr(), G.data_ptr(), ldg, stats.data_ptr(), pos_only, gh.data_ptr(),
            gl.data_ptr(), ld_split]
    if slots is not None:
        _call(name, *args, slots.data_ptr(), _st())
    else:
        _call(name, *args, _st())
    torch.cuda.synchronize()
    return G, gh, gl, stats


def _check_batch_all(S, B, lo, hi, nv, anchors, pos_only, tiled, label):
    """Runs the plain and the deterministic sweep and checks G (chosen anchors, element-wise), the split, NUM (all anchors, exactly),
    the loss slots and dae_triplet_loss_sum."""
    lds = S.shape[1]
    ldg, ld_split = B + 5, (B + 7) // 8 * 8 + 8
    lo_d, hi_d = torch.from_numpy(lo).to(DEV), torch.from_numpy(hi).to(DEV)
    G, gh, gl, st = _sweep('dae_triplet_batch_all', S, lds, B, lo_d, hi_d, nv, pos_only, ldg, ld_split)
    slots = torch.full((B,), float('nan'), dtype=torch.float64, device=DEV)
    Gd, ghd, gld, std = _sweep('dae_triplet_batch_all_det', S, lds, B, lo_d, hi_d, nv, pos_only, ldg, ld_split, slots)
    assert torch.equal(G.view(torch.int32), Gd.view(torch.int32))
    assert bool((G[:, B:] == SENT).all())
    _split_bits_ok(G, gh, gl, B)
    _split_bits_ok(Gd, ghd, gld, B)
    counts = mo.count_all(S, lo, hi)
    assert st[STAT_NUM].item() == float(counts.sum()) and std[STAT_NUM].item() == float(counts.sum())
    Gr, Gs, loss, loss_s, cnt, tiers = mo.batch_all_rows(S[torch.from_numpy(anchors).to(DEV)], anchors, lo, hi, nv, bool(pos_only),
                                                          tiled, B=B)
    assert np.array_equal(cnt, counts[anchors])
    Gn = _np(G[torch.from_numpy(anchors).to(DEV), :B])
    if pos_only:
        assert np.array_equal(Gn, Gr), label + ': pos_only G holds exact counts'
    else:
        _check(label + ' G', Gn, Gr, Gs)
    sl = _np(slots)
    _check(label + ' loss', sl[anchors], loss, loss_s)
    assert np.all(np.isfinite(sl))
    st2 = torch.zeros(16, dtype=torch.float64, device=DEV)
    _call('dae_triplet_loss_sum', slots.data_ptr(), B, st2.data_ptr(), _st())
    tot = float(np.sum(sl))
    assert abs(st2[STAT_TSUM].item() - tot) <= 1e-13 * max(np.abs(sl).sum(), 1e-300)
    assert abs(st[STAT_TSUM].item() - tot) <= 1e-13 * max(np.abs(sl).sum(), 1e-300)
    return tiers, sl[anchors], loss


def _forced(tiled):
    class _Ctx:
        def __enter__(self):
            if tiled:
                _call('dae_triplet_config', 1)

        def __exit__(self, *a):
            _call('dae_triplet_config', 0)
    return _Ctx()


# (B, class sizes): segment sizes 1, 2, 31, 32, 33, 511, 512, 513; negatives counts 1 (B = 33), 1023 (4095), 1024 (4097),
# 1025 (4096), 2049 (9800)
BATCH_ALL_SHAPES = [
    (1, [1]),
    (2, [1, 1]),
    (33, [32, 1]),
    (127, [31, 33, 2, 61]),
    (129, [33, 32, 64]),
    (800, [511, 2, 287]),
    (4095, [3072, 1023]),
    (4096, [3071, 1024, 1]),
    (4097, [3073, 512, 512]),
    (9800, [7751, 513, 512, 511, 33, 32, 31, 2, 1, 414]),
]


@pytest.mark.parametrize('B,sizes', BATCH_ALL_SHAPES, ids=[str(s[0]) for s in BATCH_ALL_SHAPES])
def test_batch_all_edges(B, sizes):
    """Rows whose ranges are 9.99, 10.0, 79.99, 80.0, 500 and 3 (the tier edges), exact ties, lds / ldg / ld_split > B; the
    shared-memory sweep and the tiled one (forced at B <= 4096, natural above)."""
    assert sum(sizes) == B
    lo, hi, _, nv = mo.segments(sizes)
    lds = B + 3
    S = _base_S(B, lds, seed=B)
    valid = [a for a in range(B) if hi[a] - lo[a] >= 2 and hi[a] - lo[a] < B]
    tie_rows = valid[1::max(1, len(valid) // 4)][:4]
    planted = sum(_plant_ties(S, B, int(lo[a]), int(hi[a]), a) for a in tie_rows)
    assert planted > 0 or B < 127
    anchors = _edge_anchors(lo, hi, B, tie_rows + valid[:len(RANGES)], seed=B) if B > 129 else np.arange(B)
    seen = set()
    for tiled in ([False, True] if B <= 4096 else [True]):
        with _forced(tiled and B <= 4096):
            tiers, _, _ = _check_batch_all(S, B, lo, hi, nv, anchors, 0, tiled, 'B=%d tiled=%d' % (B, tiled))
            seen.update(t for t in tiers if t is not None)
    if B >= 127:
        assert seen == {0, 1, 2}


@pytest.mark.parametrize('B,sizes', [(129, [33, 32, 64]), (800, [511, 2, 287]), (4097, [3073, 512, 512])], ids=['129', '800', '4097'])
def test_batch_all_pos_only(B, sizes):
    """pos_only = 1: the loss over positive triplets and G = the exact positive counts, ties and band rows included."""
    lo, hi, _, nv = mo.segments(sizes)
    S = _base_S(B, B, seed=B + 1)
    S[:, :B] *= 0.05
    valid = [a for a in range(B) if 2 <= hi[a] - lo[a] < B]
    assert _plant_ties(S, B, int(lo[valid[0]]), int(hi[valid[0]]), valid[0]) > 0
    _plant_band(S, B, int(lo[valid[-1]]), int(hi[valid[-1]]), valid[-1], seed=3)
    anchors = _edge_anchors(lo, hi, B, [valid[0], valid[-1]], seed=B) if B > 129 else np.arange(B)
    for tiled in ([False, True] if B <= 4096 else [True]):
        with _forced(tiled and B <= 4096):
            _check_batch_all(S, B, lo, hi, nv, anchors, 1, tiled, 'pos_only B=%d tiled=%d' % (B, tiled))


@pytest.mark.parametrize('B,sizes', [(800, [511, 2, 287]), (9800, [7751, 513, 512, 511, 33, 32, 31, 2, 1, 414])], ids=['800', '9800'])
def test_batch_all_band_count(B, sizes):
    """Anchors whose S values lie in the 2^-30 band, where the reference's test fp32(S_ik - S_ij) > 1e-16 and the test
    S_ik > fp32(S_ij + 1e-16) disagree: NUM must follow the reference, and so must pos_only's counts."""
    lo, hi, _, nv = mo.segments(sizes)
    S = _base_S(B, B, seed=B + 2)
    valid = [a for a in range(B) if 2 <= hi[a] - lo[a] < B]
    band = [valid[0], valid[len(valid) // 2], valid[-1]]
    for n, a in enumerate(band):
        _plant_band(S, B, int(lo[a]), int(hi[a]), a, seed=n)
    anchors = np.array(sorted(set(band)), np.int64)
    for tiled in ([False, True] if B <= 4096 else [True]):
        with _forced(tiled and B <= 4096):
            for pos_only in (0, 1):
                _check_batch_all(S, B, lo, hi, nv, anchors, pos_only, tiled, 'band B=%d tiled=%d pos=%d' % (B, tiled, pos_only))


@pytest.mark.parametrize('B,sizes', [(800, [511, 2, 287]), (9800, [7751, 513, 512, 511, 33, 32, 31, 2, 1, 414])], ids=['800', '9800'])
def test_batch_all_far_triplets_loss(B, sizes):
    """Anchors whose triplets are all separated by 17 to 80 (tier 2) or 17 to 55 (tier 1): every loss term is e^x < 2^-24, so
    fp32's 1 + e is 1; the anchor's loss must still be sum e^x within its bound."""
    lo, hi, _, nv = mo.segments(sizes)
    S = _base_S(B, B, seed=B + 4)
    valid = [a for a in range(B) if 2 <= hi[a] - lo[a] < B]
    far = {valid[0]: 2, valid[len(valid) // 2]: 1, valid[-1]: 2, valid[-2]: 1}
    for n, (a, tier) in enumerate(far.items()):
        _plant_far(S, B, int(lo[a]), int(hi[a]), a, tier, seed=n)
    anchors = np.array(sorted(far), np.int64)
    for tiled in ([False, True] if B <= 4096 else [True]):
        with _forced(tiled and B <= 4096):
            tiers, _, _ = _check_batch_all(S, B, lo, hi, nv, anchors, 0, tiled, 'far B=%d tiled=%d' % (B, tiled))
            assert [far[a] for a in anchors] == tiers


@pytest.mark.parametrize('tiled', [0, 1])
def test_batch_all_tier0_terms_near_one(tiled):
    """Tier-0 anchors whose triplets all sit at x in [-9.2, -8.8] (range 9.2): each loss term is about 1e-4 and one lg2.approx of
    a product of four t = 1 + e just above 1 carries four of them, so a bias of lg2.approx near 1 would show here.  Each anchor's
    loss within its bound; the mean signed relative error over the anchors is printed (a bias shows as a mean far from zero)."""
    B, sizes = 800, [64, 736]
    lo, hi, _, nv = mo.segments(sizes)
    S = _base_S(B, B, seed=21)
    g = torch.Generator(device=DEV).manual_seed(22)
    anchors = np.arange(64)
    for i in anchors:
        S[i, :B] = -4.6 + 0.2 * torch.rand(B, generator=g, device=DEV)
        S[i, :64] = 4.4 + 0.2 * torch.rand(64, generator=g, device=DEV)
        S[i, 0], S[i, B - 1] = 4.6, -4.6
    with _forced(tiled):
        tiers, got, want = _check_batch_all(S, B, lo, hi, nv, anchors, 0, bool(tiled), 'tier0 near 1 tiled=%d' % tiled)
    assert tiers == [0] * len(anchors)
    rel = (got - want) / want
    print('tier0 near 1 tiled=%d: relative loss error mean %.3e, max |.| %.3e' % (tiled, rel.mean(), np.abs(rel).max()))


@pytest.mark.parametrize('det', [0, 1])
def test_batch_all_rows_blocks(det):
    """dae_triplet_batch_all_rows(_det): anchor blocks with row0 > 0 and a short last block, G_blk against the reference rows."""
    B, sizes, R = 1000, [511, 2, 33, 454], 384
    lo, hi, _, nv = mo.segments(sizes)
    S = _base_S(B, B + 3, seed=7)
    lo_d, hi_d = torch.from_numpy(lo).to(DEV), torch.from_numpy(hi).to(DEV)
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    stats[STAT_N_VALID] = nv
    slots = torch.full((B,), float('nan'), dtype=torch.float64, device=DEV)
    ldg, ld_split = B + 5, B + 8
    for r0 in range(R, B, R):          # blocks 1 and 2 (232 rows): row0 > 0, the last one short
        n = min(R, B - r0)
        Sb = S[r0:r0 + n].contiguous()
        G = torch.full((n, ldg), SENT, device=DEV)
        gh, gl = _bf16_sentinel(n, ld_split), _bf16_sentinel(n, ld_split)
        args = [Sb.data_ptr(), Sb.shape[1], r0, n, B, lo_d.data_ptr(), hi_d.data_ptr(), G.data_ptr(), ldg, stats.data_ptr(), 0,
                gh.data_ptr(), gl.data_ptr(), ld_split]
        if det:
            _call('dae_triplet_batch_all_rows_det', *args, slots.data_ptr(), _st())
        else:
            _call('dae_triplet_batch_all_rows', *args, _st())
        torch.cuda.synchronize()
        _split_bits_ok(G, gh, gl, B)
        assert bool((G[:, B:] == SENT).all())
        Gr, Gs, loss, loss_s, cnt, _ = mo.batch_all_rows(Sb, np.arange(r0, r0 + n), lo, hi, nv, tiled=True, B=B)
        _check('rows G r0=%d' % r0, _np(G[:, :B]), Gr, Gs)
        if det:
            _check('rows loss r0=%d' % r0, _np(slots[r0:r0 + n]), loss, loss_s)
    counts = mo.count_all(S, lo, hi)
    assert stats[STAT_NUM].item() == float(counts[R:].sum())
    if det:
        assert bool(torch.isnan(slots[:R]).all())


# ---------------------------------------------------------------------------------------------------------------------------------
# batch_hard
# ---------------------------------------------------------------------------------------------------------------------------------
def _hard_problem(B, seed):
    """Dyadic S (multiples of 1/4 in [-5, 5]: many natural ties) with planted rows:
    0: two positives tied at the minimum;  1: two negatives tied at the maximum;  2: the row max tied;
    3: every negative < 0 (hn = 0, the masked zeros take the tie);  4: a singleton (no positive: the dm path);
    5: td exactly 0;  6: inactive (hn < hp)."""
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, max(2, B // 6), B).astype(np.float32)
    lab[:7] = [0, 0, 0, 1, 1e6, 1, 0]     # every planted row has the positives / negatives its case needs; row 4 is alone
    S = (rng.integers(-20, 21, (B, B)) / 4.0).astype(np.float32)
    same = lab[None, :] == lab[:, None]
    S[4, 5], S[4, 6] = -5.0, 1.0           # the singleton: hn >= 1 > hp = min S + m: active
    if B >= 7:
        for r in range(7):
            pos = [c for c in range(B) if same[r, c] and c != r]
            neg = [c for c in range(B) if not same[r, c]]
            if r == 0 and len(pos) >= 2:
                S[r, pos] = 2.0
                S[r, pos[:2]] = -6.0
            elif r == 1 and len(neg) >= 2:
                S[r, neg] = -1.0
                S[r, neg[:2]] = 6.0
            elif r == 2:
                S[r, :2] = 7.0
                S[r, 2:] = np.minimum(S[r, 2:], 6.5)
            elif r == 3:
                S[r, neg] = -np.abs(S[r, neg]) - 0.25
            elif r == 5 and pos and neg:
                S[r, :] = 1.0
            elif r == 6 and pos and neg:
                S[r, pos + [r]] = 3.0
                S[r, neg] = -3.0
    return S, lab


def _hard_run(S_d, lab_d, B, ldg, det):
    G = torch.full((B, ldg), SENT, device=DEV)
    w = torch.full((B,), SENT, device=DEV)
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    slots = torch.full((B,), float('nan'), dtype=torch.float64, device=DEV)
    args = [S_d.data_ptr(), S_d.shape[1], B, lab_d.data_ptr(), G.data_ptr(), ldg, w.data_ptr(), stats.data_ptr()]
    if det:
        _call('dae_triplet_batch_hard_det', *args, slots.data_ptr(), _st())
    else:
        _call('dae_triplet_batch_hard', *args, _st())
    torch.cuda.synchronize()
    return G, w, stats, slots


@pytest.mark.parametrize('B', [7, 300, 4097])
@pytest.mark.parametrize('det', [0, 1])
def test_batch_hard(B, det):
    """G element-wise against fp64 autodiff of the reference graph; weights, SUM_W and N_ACTIVE exactly; the loss slots."""
    S, lab = _hard_problem(B, seed=B)
    lds, ldg = B + 2, B + 3
    S_d = torch.full((B, lds), float('nan'), device=DEV)
    S_d[:, :B] = torch.from_numpy(S).to(DEV)
    G, w, stats, slots = _hard_run(S_d, torch.from_numpy(lab).to(DEV), B, ldg, det)
    ref = mo.batch_hard_rows(S, lab, np.arange(B))
    na = float(ref['active'].sum())
    Gr, Gs = mo.batch_hard_scaled(ref, na)
    _check('hard G B=%d' % B, _np(G[:, :B]), Gr, Gs, c=mo.C_FP32)
    assert bool((G[:, B:] == SENT).all())
    assert np.array_equal(_np(w), ref['weight'])
    assert stats[STAT_N_ACTIVE].item() == na
    assert stats[STAT_SUM_W].item() == ref['weight'].sum()
    if det:
        _check('hard loss slots B=%d' % B, _np(slots), ref['softplus'], ref['softplus'], c=mo.C_FP32)
    else:
        _check('hard loss sum B=%d' % B, stats[STAT_TSUM].item(), ref['softplus'].sum(), ref['softplus'].sum(), c=mo.C_FP32)
    _assert_hard_cases(ref)


def _assert_hard_cases(ref):
    """the planted rows of _hard_problem reached their cases"""
    assert ref['tp'][0] >= 2 and ref['tp_masked'][0] == 0                    # two positives tied at the minimum
    assert ref['tn'][1] >= 2 and ref['hn'][1] > 0                            # two negatives tied at the maximum
    assert ref['tm'][2] >= 2                                                  # the row max tied
    assert ref['hn'][3] == 0 and ref['tn'][3] >= 2                           # hn = 0, taken by the masked zeros
    assert ref['tp_masked'][4] > 0 and ref['active'][4]                      # the singleton: hp through the row max (dm)
    assert not ref['active'][5] and ref['td'][5] == 0.0                      # td exactly 0
    assert not ref['active'][6]                                               # inactive
    assert ref['active'].any() and not ref['active'].all()


@pytest.mark.parametrize('det', [0, 1])
def test_batch_hard_rows_and_finish(det):
    """dae_triplet_batch_hard_rows(_det) on anchor blocks (row0 > 0, a short last block), unscaled G_blk; then
    dae_triplet_batch_hard_finish: SUM_W and dE2 *= 1 / (N_ACTIVE + 1e-16)."""
    B, R, H = 1000, 384, 37
    S, lab = _hard_problem(B, seed=11)
    lab_d = torch.from_numpy(lab).to(DEV)
    w = torch.zeros(B, device=DEV)
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    slots = torch.full((B,), float('nan'), dtype=torch.float64, device=DEV)
    ref_all = mo.batch_hard_rows(S, lab, np.arange(B))
    _assert_hard_cases(ref_all)
    for r0 in range(0, B, R):
        n = min(R, B - r0)
        Sb = torch.from_numpy(S[r0:r0 + n]).to(DEV)
        G = torch.full((n, B + 1), SENT, device=DEV)
        args = [Sb.data_ptr(), B, r0, n, B, lab_d.data_ptr(), G.data_ptr(), B + 1, w.data_ptr(), stats.data_ptr()]
        if det:
            _call('dae_triplet_batch_hard_rows_det', *args, slots.data_ptr(), _st())
        else:
            _call('dae_triplet_batch_hard_rows', *args, _st())
        _check('hard rows G r0=%d' % r0, _np(G[:, :B]), ref_all['g'][r0:r0 + n], ref_all['g_scale'][r0:r0 + n], c=mo.C_FP32)
    na = float(ref_all['active'].sum())
    assert stats[STAT_N_ACTIVE].item() == na
    assert np.array_equal(_np(w), ref_all['weight'])
    dE2 = torch.randn(B, H + 3, device=DEV)
    dE0 = _np(dE2)
    _call('dae_triplet_batch_hard_finish', w.data_ptr(), B, stats.data_ptr(), dE2.data_ptr(), H, H + 3, _st())
    assert stats[STAT_SUM_W].item() == ref_all['weight'].sum()
    got = _np(dE2)
    want = dE0[:, :H] / (na + 1e-16)
    _check('hard finish dE2', got[:, :H], want, np.abs(want), c=2.0 ** -22)
    assert np.array_equal(got[:, H:], dE0[:, H:])
    if det:
        _check('hard rows loss', _np(slots), ref_all['softplus'], ref_all['softplus'], c=mo.C_FP32)


# ---------------------------------------------------------------------------------------------------------------------------------
# explicit triplets
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H', [1, 31, 33, 500])
@pytest.mark.parametrize('det', [0, 1])
def test_explicit(H, det):
    """|dp| up to 100 (sigma saturates), ld > H, nonzero initial dE / dEp / dEn; their padding columns untouched."""
    B, ld, alpha = 37, H + 3, 0.7
    rng = np.random.default_rng(H)
    E = rng.normal(0, 1, (B, ld)).astype(np.float32)
    Ep = rng.normal(0, 1, (B, ld)).astype(np.float32)
    En = rng.normal(0, 1, (B, ld)).astype(np.float32)
    dp0 = (E[:, :H].astype(np.float64) * (Ep[:, :H] - En[:, :H])).sum(1)
    target = np.linspace(-100, 100, B)
    f = np.where(np.abs(dp0) > 1e-3, target / np.where(np.abs(dp0) > 1e-3, dp0, 1.0), 1.0)
    Ep = (Ep * f[:, None]).astype(np.float32)
    En = (En * f[:, None]).astype(np.float32)
    d0 = [rng.normal(0, 0.01, (B, ld)).astype(np.float32) for _ in range(3)]
    dev = [torch.from_numpy(a).to(DEV) for a in (E, Ep, En)]
    dd = [torch.from_numpy(a.copy()).to(DEV) for a in d0]
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    slots = torch.full((B,), float('nan'), dtype=torch.float64, device=DEV)
    args = [dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), B, H, ld, alpha, dd[0].data_ptr(), dd[1].data_ptr(),
            dd[2].data_ptr(), stats.data_ptr()]
    if det:
        _call('dae_triplet_explicit_det', *args, slots.data_ptr(), _st())
    else:
        _call('dae_triplet_explicit', *args, _st())
    ref = mo.explicit(E[:, :H], Ep[:, :H], En[:, :H], alpha, d0[0][:, :H], d0[1][:, :H], d0[2][:, :H])
    for k, name in enumerate(('dE', 'dEp', 'dEn')):
        got = _np(dd[k])
        _check('explicit %s H=%d' % (name, H), got[:, :H], *ref[name])
        assert np.array_equal(got[:, H:], d0[k][:, H:].astype(np.float64))
    assert stats[STAT_N_ACTIVE].item() == B
    if det:
        _check('explicit loss H=%d' % H, _np(slots), *ref['loss'])
    else:
        _check('explicit loss sum H=%d' % H, stats[STAT_TSUM].item(), ref['loss'][0].sum(), ref['loss'][1].sum())


# ---------------------------------------------------------------------------------------------------------------------------------
# GEMMs and operand splits
# ---------------------------------------------------------------------------------------------------------------------------------
def _split(src, rows, cols, ld_dst, ones_col=-1, scale=1.0):
    hi, lo = _bf16_sentinel(rows, ld_dst), _bf16_sentinel(rows, ld_dst)
    _call('dae_split_bf16', src.data_ptr(), rows, cols, src.stride(0), hi.data_ptr(), lo.data_ptr(), ld_dst, ones_col, float(scale),
          _st())
    return hi, lo


def _pad8(n):
    return (n + 7) // 8 * 8


def _gemm(M, N, K, alpha, A, a_mn, Bm, b_mn, C, accumulate, k_splits=1):
    _call('dae_gemm_bf16x3', M, N, K, float(alpha), A[0].data_ptr(), A[1].data_ptr(), A[0].stride(0), a_mn, Bm[0].data_ptr(),
          Bm[1].data_ptr(), Bm[0].stride(0), b_mn, C.data_ptr(), C.stride(0), 0, -1, None, k_splits, accumulate, _st())
    torch.cuda.synchronize()


@pytest.mark.parametrize('B', [129, 800, 4097])
@pytest.mark.parametrize('H', [7, 500])
def test_gram_gemm(B, H):
    """S = E.E^T (both operands K-major), k_splits 1 and stream-K, ldc > B: element-wise against fp64 with the bf16x3 bound."""
    E = torch.randn(B, H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(B + H))
    E[:, 0] *= 30.0                       # columns of very different magnitude
    Ehl = _split(E, B, H, _pad8(H))
    want, bound = mo.gemm(E, E)
    for ks in (1, -1):
        S = torch.full((B, B + 3), SENT, device=DEV)
        _gemm(B, B, H, 1.0, Ehl, 0, Ehl, 0, S, 0, ks)
        _check('gram B=%d H=%d ks=%d' % (B, H, ks), _np(S[:, :B]), want, bound)
        assert bool((S[:, B:] == SENT).all())


def _sym_inputs(B, H, seed):
    """G >= 0 and E >= 0: every product has one sign, so the accumulator's rounding cannot cancel and the bound is approached."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    G = torch.randn(B, B, device=DEV, generator=g).abs() * torch.rand(B, 1, device=DEV, generator=g)
    E = torch.randn(B, H, device=DEV, generator=g).abs()
    return G, E


@pytest.mark.parametrize('B,H', [(129, 7), (800, 500), (4097, 64)])
@pytest.mark.parametrize('accumulate', [0, 1])
@pytest.mark.parametrize('det', [0, 1])
def test_sym_gemm(B, H, accumulate, det):
    """dE2 = alpha (G + G^T) E (+ C) in one launch, alpha = -0.37: element-wise against fp64."""
    alpha = -0.37
    G, E = _sym_inputs(B, H, seed=B + H)
    Ghl = _split(G, B, B, _pad8(B))
    Ehl = _split(E, B, H, _pad8(H))
    C = torch.randn(B, H + 1, device=DEV) if accumulate else torch.full((B, H + 1), SENT, device=DEV)
    C0 = C[:, :H].clone()
    args = [B, H, float(alpha), Ghl[0].data_ptr(), Ghl[1].data_ptr(), Ghl[0].stride(0), Ehl[0].data_ptr(), Ehl[1].data_ptr(),
            Ehl[0].stride(0), C.data_ptr(), C.stride(0), accumulate]
    if det:
        ws_bytes = _cabi().query('dae_gemm_det_workspace')
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
        _call('dae_gemm_sym_bf16x3_det', *args, ws.data_ptr(), ws_bytes, _st())
    else:
        _call('dae_gemm_sym_bf16x3', *args, _st())
    A = torch.cat([G, G.t()], 1)
    Bt = torch.cat([E.t(), E.t()], 1)
    want, bound = mo.gemm(A, Bt, alpha, C0 if accumulate else None, K_eff=2 * ((B + 63) // 64 * 64))
    got = _np(C)
    _check('sym B=%d acc=%d det=%d' % (B, accumulate, det), got[:, :H], want, bound)
    if not accumulate:
        assert np.all(got[:, H:] == SENT)


def test_block_de2_gemms():
    """The two dE2 GEMMs of a mining block (engine._mining_blocked), both accumulating:
    dE2[r0:r0+n] += a G_blk.E (G_blk K-major, M = n, K = B) and dE2 += a G_blk^T.E[r0:r0+n] (G_blk MN-major, M = B, K = n)."""
    B, H, r0, n, a = 1000, 500, 768, 232, 0.6
    g = torch.Generator(device=DEV).manual_seed(5)
    Gb = torch.randn(n, B, device=DEV, generator=g)
    E = torch.randn(B, H, device=DEV, generator=g)
    Ghl = _split(Gb, n, B, _pad8(B))
    Ehl = _split(E, B, H, _pad8(H))
    dE2 = torch.randn(B, H, device=DEV, generator=g)
    start = dE2.clone()
    _gemm(n, H, B, a, Ghl, 0, (Ehl[0], Ehl[1]), 1, dE2[r0:], 1)
    w1, b1 = mo.gemm(Gb, E.t().contiguous(), a, start[r0:r0 + n])
    got = _np(dE2)
    _check('block dE2 G.E', got[r0:r0 + n], w1, b1)
    assert np.array_equal(got[:r0], _np(start[:r0]))
    mid = dE2.clone()
    _gemm(B, H, n, a, Ghl, 1, (Ehl[0][r0:], Ehl[1][r0:]), 1, dE2, 1)
    w2, b2 = mo.gemm(Gb.t().contiguous(), E[r0:r0 + n].t().contiguous(), a, mid)
    _check('block dE2 G^T.E', _np(dE2), w2, b2)


def test_split_bf16_bits():
    """dae_split_bf16 with scale and ones_col, and dae_sym_split_bf16 with alpha, bit for bit against NumPy (round to nearest
    even at the halfway points, zero padding)."""
    rows, cols = 37, 45
    rng = np.random.default_rng(0)
    src = (rng.normal(0, 1, (rows, cols + 3)) * 10.0 ** rng.integers(-20, 20, (rows, cols + 3))).astype(np.float32)
    src[0, :6] = [1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 0.0, -0.0, 2.0 ** -130]
    src_d = torch.from_numpy(src).to(DEV)
    ld = _pad8(cols + 1)
    for scale in (1.0, 0.3):
        hi, lo = _split(src_d, rows, cols, ld, ones_col=cols, scale=scale)
        eh, el = mo.split_ref(src, cols, ld, cols, scale)
        assert np.array_equal(_bits16(hi), eh) and np.array_equal(_bits16(lo), el)
    B = 45
    G = src[:B, :B] if rows >= B else rng.normal(0, 1, (B, B)).astype(np.float32)
    G_d = torch.from_numpy(np.ascontiguousarray(G)).to(DEV)
    ld = _pad8(B) + 8
    hi, lo = _bf16_sentinel(B, ld), _bf16_sentinel(B, ld)
    _call('dae_sym_split_bf16', G_d.data_ptr(), B, B, -0.37, hi.data_ptr(), lo.data_ptr(), ld, _st())
    eh, el = mo.sym_split_ref(G, ld, -0.37)
    assert np.array_equal(_bits16(hi), eh) and np.array_equal(_bits16(lo), el)


# ---------------------------------------------------------------------------------------------------------------------------------
# dae_step_finalize
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B', [1, 800, 32768])
@pytest.mark.parametrize('strategy', [0, 1, 2, 3])
def test_step_finalize(B, strategy):
    """All four strategies, row_loss and parts, weight NULL and non-NULL, the stats_log row chosen by ctl[1]: against fp64
    within 2^-36 relative; the parts path's per-row fp32 sums bit for bit (a one-hot weight isolates one row's sum in SUM_LW)."""
    rng = np.random.default_rng(B + strategy)
    n_parts = 17
    parts = (rng.random((n_parts, B)) * 10.0 ** rng.integers(-3, 3, (n_parts, B))).astype(np.float32)
    row_loss = mo.part_sums(parts)
    weight = rng.integers(0, 4, B).astype(np.float32)
    stats_in = np.zeros(16)
    stats_in[STAT_SUM_W] = float(weight.sum()) + 0.5
    stats_in[STAT_N_VALID] = 12345.0
    stats_in[STAT_NUM] = 678.0
    stats_in[STAT_TSUM] = 3.25
    stats_in[STAT_N_ACTIVE] = float(max(1, B // 3))
    alpha = 0.3
    ctl = torch.tensor([0, 2, 1, 0], dtype=torch.int64, device=DEV)
    parts_d = torch.from_numpy(parts).to(DEV)
    rl_d = torch.from_numpy(row_loss).to(DEV)
    w_d = torch.from_numpy(weight).to(DEV)
    for use_parts in (False, True):
        for wt in (None, weight):
            stats = torch.from_numpy(stats_in).to(DEV)
            log = torch.full((4, 16), -5.0, dtype=torch.float64, device=DEV)
            _call('dae_step_finalize', None if use_parts else rl_d.data_ptr(), parts_d.data_ptr() if use_parts else None,
                  n_parts if use_parts else 0, None if wt is None else w_d.data_ptr(), B, strategy, alpha, stats.data_ptr(),
                  log.data_ptr(), ctl.data_ptr(), _st())
            want, mag = mo.finalize(row_loss, wt, strategy, alpha, stats_in)
            got = _np(stats)
            scale = np.abs(want)
            scale[[0, 1, 7]] += mag / (stats_in[STAT_SUM_W] + 1e-16) * np.array([1.0, 1.0, stats_in[STAT_SUM_W] + 1e-16])
            _check('finalize B=%d s=%d parts=%d w=%d' % (B, strategy, use_parts, wt is not None), got, want, scale, c=2.0 ** -36)
            lg = _np(log)
            assert np.array_equal(lg[2], got)
            assert np.all(lg[[0, 1, 3]] == -5.0)
    for i in sorted({0, B // 2, B - 1}):   # per-row fp32 part sums, bit for bit
        oh = np.zeros(B, np.float32)
        oh[i] = 1.0
        stats = torch.from_numpy(stats_in).to(DEV)
        oh_d = torch.from_numpy(oh).to(DEV)
        _call('dae_step_finalize', None, parts_d.data_ptr(), n_parts, oh_d.data_ptr(), B, strategy, alpha, stats.data_ptr(), None,
              None, _st())
        assert _np(stats)[7] == float(row_loss[i])
