"""fp64 references of the training step's mining branch (the Gram / sym / block dE2 GEMMs, the batch_all sweep, batch_hard, the
explicit triplets, the step finalize), for the kernel-level tests.  Tests only.

As in step_kernel_oracle.py, every reference returns the value AND a per-element error scale, and a kernel passes when, for every
element, |got - want| <= c * scale + tiny.  Here the scale is the first-order error bound itself (absolute units), derived below
from the kernel's arithmetic; c = C_HEAD = 2 leaves a factor of two.  The input is always the fp32 S (or E) the kernel was given;
a difference of two fp32 values is exact in fp64.

batch_all, tiers 0-2 (triplet.cu).  For anchor i, positive j and negative k, x = S_ik - S_ij, sigma = 1 / (1 + e^-x).
  G_ij = -sum_k sigma / NV,  G_ik = +sum_j sigma / NV,  G_ii = 0;  anchor loss = sum softplus(x).
  One sigma.  The kernel forms e = e^x as u_j v_k with u = ex2((mid - S_ij) log2e), v = ex2((S_ik - mid) log2e) around the row
  midpoint mid = (max + min) / 2 (tier 2: ex2(-|x| log2e) with x rounded in fp32).  Each exponent argument is rounded twice
  (the difference and the product with log2e) and log2e once: 3 x 2^-24 |S - mid| in x, so dx <= 2^-22 D with
  D = |S_ij - mid| + |S_ik - mid|; the two ex2.approx add about 2^-22 each to e: 2^-21.  Through d sigma / d ln e = sigma (1 - sigma):
      err(sigma) <= sigma (1 - sigma) (2^-21 + 2^-22 D + 2^-50) + 2^-20 sigma + 2^-126
  2^-20 sigma covers the rounded products and the reciprocal after e (tier 0: t = 1 + e for four triplets multiplied into one P,
  rcp.approx of P and the products back out: about seven roundings and one rcp, 2^-21); 2^-50 covers the staged positive
  threshold (below), 2^-126 the flush to zero of ex2.approx.ftz.
  The sums.  A row sum runs per thread over its k tiles (4 adds per 128-column tile; tier 0: 1 add of a 3-deep pair sum), then
  over the 32 lanes (5), in the tiled kernel per 1024-negative chunk plus one carry per chunk; a column sum adds 4 terms per
  32-row j tile, one partial per j tile and the 8 warp slabs.  A chain of L adds of positive terms is off by at most L 2^-24 of
  its sum; the scale by (float)(1 / NV) adds 2 more.
      err(G_ij) <= [sum_k err(sigma) + (L_row + 2) 2^-24 sum_k sigma] / NV         (same for G_ik with L_col)
  The loss.  softplus(x) = ln 2 x sum of lg2 terms.  Per triplet: 2^-21 softplus (x log2e rounded in tier 2; lg2.approx's
  relative error for large arguments) and sigma times the error of e; 2^-125 for terms flushed to zero.  Per lg2.approx
  evaluation 2^-22 absolute (one per four triplets in tier 0, one per triplet in tiers 1 and 2), and per formed t = 1 + e its
  rounding, 2 x 2^-24 absolute (tier 0: with its share of the three products of t's).  In tiers 1 and 2 the kernel takes
  lg2(t) only for e >= 2^-12 (tier 2: e = e^-|x|); below it adds the series (e - e^2 / 2) / ln 2, within e^2 / 3 <= 2^-25 of
  the term (inside the 2^-21 per term), and no absolute error.  The thread's fp32 accumulator adds L_loss terms between fp64
  flushes (per tile 4 in tier 0 and 16 in tiers 1-3; the tiled kernel flushes after every (512, 1024) chunk pair): L_loss 2^-24
  sum softplus.  That chain bound is a worst case, so the loss sits further below its bound than G does; a dropped or
  mis-evaluated term still exceeds it.
  The count.  The reference counts a triplet when fp32(S_ik - S_ij) > fp32(1e-16); count_positive does exactly that, and the
  kernel's count must equal it.

pos_triplets_only (tier 3).  The loss sums softplus over the positive triplets only and G holds counts: -#k at a positive, +#j
  at a negative, exactly.  The kernel takes x = fp32(S_ik - t_j) from the staged threshold t_j, which differs from S_ij only when
  |S_ij| < 2^-29, and then by about 1e-16: the 2^-50 above.

batch_hard.  m, hn, hp, td and the tie counts are computed in fp32 as the reference does (S + m (1 - ap) and an S, equality on
  the fp32 values), then the gradient of its graph in fp64: -q / tp at the hp ties, +an q / tn at the hn ties (masked zeros
  count as ties and take their share), and dm / tm at the row-max ties with dm = -q tp_masked / tp, the gradient that reaches m
  through masked argmin entries; q = sigma(td) for active anchors.  G = that / (N_active + 1e-16).  A few fp32 operations and
  the accurate expf per entry: C_FP32 = 2^-20 of the sum of the terms' magnitudes.  Weights, SUM_W and N_ACTIVE are integers
  and exact.

explicit.  dp = sum_h e ep - e en, summed by each lane over H / 32 pairs and then over the warp: err(dp) <= (2 ceil(H / 32) +
  5) 2^-24 sum_h |e ep| + |e en|.  sigma(-dp) moves by sigma (1 - sigma) err(dp) plus 2^-21 sigma; each gradient update is a
  fp32 multiply-add on top of the given dE / dEp / dEn.

GEMMs (bf16x3).  |C - C_ref| <= c_K |alpha| sum_k |a_k b_k| (+ 2^-24 |C_prev| when accumulating), with
  c_K = 2 x 2^-17 + 2^-16 + (3 K / 16) 2^-23 + 2^-22.  bf16 keeps 8 significant bits: hi = rn(a) is within 2^-8 |a|, and
  lo = rn(a - hi) leaves a - hi - lo within 2^-8 of |a - hi| < 2^-8 of a power of two no larger than |a|, so 2^-17 |a| per
  operand; the dropped lo.lo term is up to 2^-16 |a b|.  Three products per 16-deep wgmma step go into an fp32 accumulator
  whose internal adder NVIDIA does not document (taken as truncating: (3 K / 16) 2^-23), and the stream-K partial tiles are
  added with atomics: 2^-22.  The product part alone reaches 2^-15.1 of |a b| (NumPy, 2e6 random normal products), which is what
  the Gram at K = 7 shows on an H100 (2^-15.1 of sum |a b| at a diagonal entry, all products of one sign).

finalize (loss.cu step_finalize_kernel): the fp64 formulas; the per-row losses of the `parts` path are fp32 sums in part order,
  restated in NumPy float32 (part_sums).
"""
import math

import numpy as np
import torch

C_HEAD = 2.0
C_FP32 = 2.0 ** -20
U = 2.0 ** -24
LN2 = math.log(2.0)
EPS = 1e-16
POS_MARGIN = np.float32(1e-16)
SERIES_E = 2.0 ** -12          # tiers 1 and 2: below this e the kernel adds (e - e^2 / 2) / ln 2 instead of lg2(1 + e)


# ---------------------------------------------------------------------------------------------------------------------------
# the positive test
# ---------------------------------------------------------------------------------------------------------------------------
def count_positive(sj, sk):
    """#{(j, k): fp32(S_ik - S_ij) > fp32(1e-16)} -- the reference's test (triplet_loss_utils.py:114), in fp32.  sj, sk: 1-d
    float32 torch tensors (any device) or NumPy arrays."""
    if isinstance(sj, np.ndarray):
        sj, sk = np.asarray(sj, np.float32), np.asarray(sk, np.float32)
        return int(((sk[None, :] - sj[:, None]) > POS_MARGIN).sum())
    d = sk.float()[None, :] - sj.float()[:, None]
    return int((d > float(POS_MARGIN)).sum())


def _ordered(f):
    b = int(np.float32(f).view(np.int32))
    return -(b & 0x7FFFFFFF) if b < 0 else b


def _from_ordered(o):
    b = ((-o) | 0x80000000) if o < 0 else o
    return np.array([b & 0xFFFFFFFF], np.uint32).view(np.float32)[0]


def pos_threshold(a):
    """The largest fp32 b with fp32(b - a) <= fp32(1e-16): a triplet is positive exactly when S_ik > t.  t = a for |a| >= 2^-29;
    below, a bisection on the ordered-integer encoding of fp32 (the kernel's staging loop does the same)."""
    a = np.float32(a)
    if abs(a) >= np.float32(2.0 ** -29):
        return a
    lo, hi = _ordered(a), _ordered(np.float32(a + np.float32(1e-15)))   # fp32(lo - a) = 0 passes, fp32(hi - a) ~ 1e-15 fails
    while hi - lo > 1:
        mid = lo + (hi - lo) // 2
        if np.float32(_from_ordered(mid) - a) <= POS_MARGIN:
            lo = mid
        else:
            hi = mid
    return _from_ordered(lo)


def band_pairs(n, seed=0):
    """n fp32 pairs (a, b) on which the reference's test fp32(b - a) > 1e-16 and the test b > fp32(a + 1e-16) disagree: a in
    [2^-35, 2^-34) or [2^-32, 2^-29), either sign, b the fp32 value just past the reference's threshold."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        e = rng.choice([-35, -32, -31, -30])
        a = np.float32(rng.choice([-1.0, 1.0]) * rng.uniform(1.0, 2.0) * 2.0 ** e)
        b = np.nextafter(pos_threshold(a), np.float32(np.inf))
        if (np.float32(b - a) > POS_MARGIN) != (b > np.float32(a + POS_MARGIN)):
            out.append((a, b))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# segments of a label-sorted batch
# ---------------------------------------------------------------------------------------------------------------------------
def segments(sizes):
    """seg_lo / seg_hi of a label-sorted batch whose classes have the given sizes (in order), their labels, and N_valid."""
    sizes = np.asarray(sizes, np.int64)
    B = int(sizes.sum())
    ends = np.cumsum(sizes)
    lab = np.repeat(np.arange(len(sizes), dtype=np.float32), sizes)
    lo = np.repeat(ends - sizes, sizes).astype(np.int32)
    hi = np.repeat(ends, sizes).astype(np.int32)
    n = sizes.astype(np.float64)
    return lo, hi, lab, float(np.sum(n * (n - 1.0) * (B - n)))


def tier_of(row):
    """The tier the sweep picks for a fp32 row (range = fp32(max - min): < 10 -> 0, < 80 -> 1, else 2)."""
    r = np.asarray(row, np.float32)
    rng = np.float32(r.max() - r.min())
    return 0 if rng < np.float32(10.0) else (1 if rng < np.float32(80.0) else 2)


# ---------------------------------------------------------------------------------------------------------------------------
# batch_all (tiers 0-2) and pos_triplets_only (tier 3)
# ---------------------------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def batch_all_anchor(s, i, lo, hi, nv, pos_only=False, tiled=False):
    """Reference of one anchor row.  s: the fp32 row S[i, :B] (torch; the work runs on its device in fp64).
    Returns dict g, g_scale (fp64 [B]), loss, loss_scale, count (positive triplets, fp32 test), tier."""
    B = s.numel()
    dev = s.device
    nj, nk = hi - lo, B - (hi - lo)
    out = {'g': torch.zeros(B, dtype=torch.float64, device=dev), 'g_scale': torch.zeros(B, dtype=torch.float64, device=dev),
           'loss': 0.0, 'loss_scale': 0.0, 'count': 0, 'tier': None}
    if nj <= 1 or nk == 0:
        return out
    s32 = s.float()
    sd = s32.double()
    mx, mn = s32.max(), s32.min()
    rng = float((mx - mn).item())
    tier = 3 if pos_only else (0 if rng < 10.0 else (1 if rng < 80.0 else 2))
    out['tier'] = tier
    mid = float((np.float32(0.5) * (np.float32(mx.item()) + np.float32(mn.item()))))
    pidx = torch.cat([torch.arange(lo, i, device=dev), torch.arange(i + 1, hi, device=dev)])
    kidx = torch.cat([torch.arange(0, lo, device=dev), torch.arange(hi, B, device=dev)])
    sj, sk = sd[pidx], sd[kidx]
    x = sk[None, :] - sj[:, None]
    pos = (s32[kidx][None, :] - s32[pidx][:, None]) > float(POS_MARGIN)
    out['count'] = int(pos.sum())
    sig = torch.sigmoid(x)
    sp = torch.logaddexp(x, torch.zeros((), dtype=torch.float64, device=dev))
    D = (sj - mid).abs()[:, None] + (sk - mid).abs()[None, :]
    if tier == 3:
        posd = pos.double()
        out['g'][pidx] = -posd.sum(1)
        out['g'][kidx] = posd.sum(0)
        spp = sp * posd
        n_t = float(posd.sum())
        per = 2.0 ** -21 * spp + sig * posd * (2.0 ** -21 + 2.0 ** -22 * D + 2.0 ** -50)
        n_lg2 = n_t
        adds = 16
        out['loss'] = float(spp.sum())
        loss_sum = out['loss']
    else:
        err_sig = sig * (1.0 - sig) * (2.0 ** -21 + 2.0 ** -22 * D + 2.0 ** -50) + 2.0 ** -20 * sig + 2.0 ** -126
        inv = 1.0 / (nv + EPS)
        if tiled:
            l_row = 4 * _cdiv(min(nk, 1024), 128) + 5 + _cdiv(nk, 1024)
        else:
            l_row = 4 * _cdiv(nk, 128) + 5
        l_col = 4 + _cdiv(nj, 32) + 8
        rs, cs = sig.sum(1), sig.sum(0)
        out['g'][pidx] = -rs * inv
        out['g'][kidx] = cs * inv
        out['g_scale'][pidx] = (err_sig.sum(1) + (l_row + 2) * U * rs) * inv
        out['g_scale'][kidx] = (err_sig.sum(0) + (l_col + 2) * U * cs) * inv
        per = 2.0 ** -21 * sp + sig * (2.0 ** -21 + 2.0 ** -22 * D + 2.0 ** -50) + 2.0 ** -125
        if tier == 0:
            n_t = float(x.numel())
            n_lg2 = float((nj - 1) * _cdiv(nk, 4))
            adds = 4
        else:   # t = 1 + e and lg2 only where e >= 2^-12 (a margin of 1e-3 in x counts the borderline ones); below, the series
            n_t = float((x >= math.log(SERIES_E) - 1e-3).sum())
            n_lg2 = n_t
            adds = 16
        out['loss'] = float(sp.sum())
        loss_sum = out['loss']
    pj, pk = _cdiv(nj, 32) * 32, _cdiv(nk, 128) * 128
    if tiled:
        tiles = (min(pj, 512) // 32) * (min(pk, 1024) // 128)
    else:
        tiles = (pj // 32) * (pk // 128)
    l_loss = tiles * adds
    out['loss_scale'] = float(per.sum()) + LN2 * 2.0 ** -22 * n_lg2 + 2.0 * U * n_t + l_loss * U * loss_sum
    return out


def count_all(S, lo, hi):
    """The number of positive triplets of every anchor (fp32 test), O(B^2 log B): per class, its rows' negatives sorted, and each
    positive's threshold (pos_threshold) located in them.  S: torch fp32 [B x >= B] (whole batch); lo, hi: NumPy segments."""
    B = len(lo)
    S = S[:, :B].float()
    out = np.zeros(B, np.int64)
    starts = np.unique(lo)
    for s0 in starts:
        s1 = int(hi[s0])
        rows = S[s0:s1]
        neg = torch.cat([rows[:, :s0], rows[:, s1:]], 1)
        if neg.shape[1] == 0 or s1 - s0 < 2:
            continue
        srt = neg.sort(1).values.contiguous()
        thr = rows[:, s0:s1].clone()
        small = thr.abs() < 2.0 ** -29
        if bool(small.any()):
            vals = thr[small]
            uniq, inv = torch.unique(vals, return_inverse=True)
            t = torch.tensor([float(pos_threshold(np.float32(v))) for v in uniq.tolist()], dtype=torch.float32, device=S.device)
            thr[small] = t[inv]
        idx = torch.arange(s1 - s0, device=S.device)
        thr[idx, idx] = float('inf')     # the anchor is not its own positive
        above = neg.shape[1] - torch.searchsorted(srt, thr.contiguous(), right=True)
        out[s0:s1] = above.sum(1).cpu().numpy()
    return out


def batch_all_rows(S, anchors, lo, hi, nv, pos_only=False, tiled=False, B=None):
    """batch_all_anchor over the anchors; S[r] is the row of anchors[r] (torch fp32 [n x >= B]).  Returns stacked arrays
    (NumPy fp64): G, G scale, loss, loss scale, count per anchor, and the tiers."""
    B = S.shape[1] if B is None else B
    rows = [batch_all_anchor(S[r, :B], int(a), int(lo[a]), int(hi[a]), nv, pos_only, tiled) for r, a in enumerate(anchors)]
    G = torch.stack([o['g'] for o in rows]).cpu().numpy()
    Gs = torch.stack([o['g_scale'] for o in rows]).cpu().numpy()
    return (G, Gs, np.array([o['loss'] for o in rows]), np.array([o['loss_scale'] for o in rows]),
            np.array([o['count'] for o in rows], np.int64), [o['tier'] for o in rows])


# ---------------------------------------------------------------------------------------------------------------------------
# batch_hard
# ---------------------------------------------------------------------------------------------------------------------------
def batch_hard_rows(S, labels, anchors):
    """S: fp32 NumPy [n x B], row r of anchor anchors[r]; labels [B].  Returns the UNSCALED gradient rows g and their scale, the
    per-anchor active flag, td (fp32), softplus(td), and the weight contributions of these rows (fp64 [B])."""
    S = np.asarray(S, np.float32)
    lab = np.asarray(labels, np.float32)
    n, B = S.shape
    anchors = np.asarray(anchors)
    cols = np.arange(B)
    same = lab[None, :] == lab[anchors][:, None]
    ap = (same & (cols[None, :] != anchors[:, None])).astype(np.float32)
    an = (~same).astype(np.float32)
    m = S.max(1)
    hn = (an * S).max(1)
    shifted = S + m[:, None] * (np.float32(1.0) - ap)
    hp = shifted.min(1)
    td = np.maximum(hn - hp, np.float32(0.0))
    active = td > 0
    eq_p = shifted == hp[:, None]
    eq_n = (an * S) == hn[:, None]
    eq_m = S == m[:, None]
    tp = eq_p.sum(1).astype(np.float64)
    tpm = (eq_p & (ap == 0)).sum(1).astype(np.float64)
    tn = eq_n.sum(1).astype(np.float64)
    tm = eq_m.sum(1).astype(np.float64)
    tdd = td.astype(np.float64)
    q = np.where(active, 1.0 / (1.0 + np.exp(-tdd)), 0.0)
    dm = -q * tpm / tp
    a_p = np.where(eq_p, -(q / tp)[:, None], 0.0)
    a_n = np.where(eq_n, (an * (q / tn)[:, None]), 0.0)
    a_m = np.where(eq_m, (dm / tm)[:, None], 0.0)
    g = (a_p + a_n + a_m) * active[:, None]
    g_scale = (np.abs(a_p) + np.abs(a_n) + np.abs(a_m)) * active[:, None]
    w = np.zeros(B)
    for r in np.nonzero(active)[0]:
        w += (S[r] == hp[r]).astype(np.float64) + (S[r] == hn[r]).astype(np.float64)
        w[anchors[r]] += 1.0
    sp = np.where(active, np.logaddexp(tdd, 0.0), 0.0)
    return {'g': g, 'g_scale': g_scale, 'active': active, 'td': td, 'softplus': sp, 'weight': w, 'hn': hn, 'hp': hp, 'm': m,
            'tp': tp, 'tp_masked': tpm, 'tn': tn, 'tm': tm}


def batch_hard_scaled(ref, n_active):
    """G = g / (N_active + 1e-16) and its scale (the kernel's fp32 scale by (float)(1 / N) adds two roundings, within C_FP32)."""
    inv = 1.0 / (n_active + EPS)
    return ref['g'] * inv, ref['g_scale'] * inv


# ---------------------------------------------------------------------------------------------------------------------------
# explicit triplets
# ---------------------------------------------------------------------------------------------------------------------------
def explicit(E, Ep, En, alpha, dE0, dEp0, dEn0):
    """Rows of (E, Ep, En) fp32 [B x H]; returns {name: (value, bound)} for dE, dEp, dEn and the per-row loss softplus(-dp)."""
    e, ep, en = (np.asarray(a, np.float64) for a in (E, Ep, En))
    B, H = e.shape
    dp = (e * ep - e * en).sum(1)
    s_dp = (2 * _cdiv(H, 32) + 5) * U * (np.abs(e * ep) + np.abs(e * en)).sum(1)
    x = -dp
    sg = 1.0 / (1.0 + np.exp(-x))
    sp = np.logaddexp(x, 0.0)
    a = float(np.float32(alpha))
    c = a * sg / B
    dc = abs(a) / B * (sg * (1.0 - sg) * s_dp + 2.0 ** -21 * sg + 2.0 ** -126) + 2.0 ** -22 * np.abs(c)
    out = {}
    for name, base, term, mag in (('dE', dE0, en - ep, np.abs(en) + np.abs(ep)), ('dEp', dEp0, -e, np.abs(e)),
                                  ('dEn', dEn0, e, np.abs(e))):
        b0 = np.asarray(base, np.float64)
        val = b0 + c[:, None] * term
        bound = 3 * U * (np.abs(b0) + np.abs(c)[:, None] * mag) + dc[:, None] * np.abs(term)
        out[name] = (val, bound)
    out['loss'] = (sp, sg * s_dp + 2.0 ** -22 * sp + 2.0 ** -126)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# GEMMs
# ---------------------------------------------------------------------------------------------------------------------------
def gemm_c(K):
    return 2.0 * 2.0 ** -17 + 2.0 ** -16 + (3.0 * K / 16.0) * 2.0 ** -23 + 2.0 ** -22


def gemm(A, Bm, alpha=1.0, C0=None, K_eff=None):
    """C = alpha A Bm^T (+ C0), A [M x K], Bm [N x K] (fp32 inputs, torch; fp64 on their device).  Returns (C, bound) as NumPy."""
    Ad, Bd = A.double(), Bm.double()
    a = float(np.float32(alpha))
    C = a * (Ad @ Bd.t())
    s = abs(a) * (Ad.abs() @ Bd.abs().t())
    K = A.shape[1] if K_eff is None else K_eff
    bound = gemm_c(K) * s
    if C0 is not None:
        C0d = C0.double()
        C = C + C0d
        bound = bound + U * (C0d.abs() + C.abs())
    return C.cpu().numpy(), bound.cpu().numpy()


def bf16_rn(x):
    """float32 -> bf16 (round to nearest even) as uint16 bits."""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_split(v):
    """hi = rn(v), lo = rn(v - hi) (v float32), as uint16 bit patterns."""
    v = np.asarray(v, np.float32)
    hi = bf16_rn(v)
    lo = bf16_rn((v - (hi.astype(np.uint32) << 16).view(np.float32)).astype(np.float32))
    return hi, lo


def split_ref(src, cols, ld_dst, ones_col, scale):
    """dae_split_bf16: v = src * scale (fp32) in columns < cols, 0 up to ld_dst, 1 in ones_col; its (hi, lo) bits."""
    src = np.asarray(src, np.float32)
    rows = src.shape[0]
    v = np.zeros((rows, ld_dst), np.float32)
    v[:, :cols] = src[:, :cols] * np.float32(scale)
    if 0 <= ones_col < ld_dst:
        v[:, ones_col] = 1.0
    return bf16_split(v)


def sym_split_ref(G, ld, alpha):
    """dae_sym_split_bf16: v = alpha * (G + G^T) in fp32 (the sum first), 0 in the columns [B, ld); its (hi, lo) bits."""
    G = np.asarray(G, np.float32)
    B = G.shape[0]
    v = np.zeros((B, ld), np.float32)
    v[:, :B] = np.float32(alpha) * (G + G.T)
    return bf16_split(v)


# ---------------------------------------------------------------------------------------------------------------------------
# finalize
# ---------------------------------------------------------------------------------------------------------------------------
def part_sums(parts):
    """The parts path's per-row losses: parts [n_parts x B] added in part order in fp32."""
    parts = np.asarray(parts, np.float32)
    acc = np.zeros(parts.shape[1], np.float32)
    for p in range(parts.shape[0]):
        acc = (acc + parts[p]).astype(np.float32)
    return acc


def finalize(row_loss, weight, strategy, alpha, stats):
    """dae_step_finalize in fp64 (loss.cu step_finalize_kernel).  row_loss: fp32 per-row losses; weight: fp32 or None; stats: the
    16 input slots.  Returns (16 output slots, the sum of |l w| -- the scale of SUM_LW and AE_LOSS)."""
    l = np.asarray(row_loss, np.float32).astype(np.float64)
    w = np.ones_like(l) if weight is None else np.asarray(weight, np.float32).astype(np.float64)
    out = np.array(stats, np.float64).copy()
    s = float((l * w).sum())
    mag = float(np.abs(l * w).sum())
    ae = s / (out[5] + EPS)
    tl = frac = num = 0.0
    if strategy == 1:
        nv = out[6]
        tl = out[8] / (nv + EPS)
        num = out[4]
        frac = num / (nv + EPS)
    elif strategy == 2:
        na = out[9]
        tl = out[8] / (na + EPS)
        num = na
        frac = na / float(len(l))
    elif strategy == 3:
        tl = out[8] / out[9]
    out[7], out[1], out[2], out[3], out[4] = s, ae, tl, frac, num
    out[0] = ae if strategy == 0 else ae + float(np.float32(alpha)) * tl
    return out, mag
