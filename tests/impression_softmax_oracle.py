"""fp64 reference of dae_impression_softmax_loss (csrc/impressions.cu) with per-element error bounds, the NumPy restatement of its
draws and of Floyd's algorithm, and a float32 emulation of the kernel in its operation order.  Tests only.

As in impression_kernel_oracle.py, a reference returns (value, scale) and a kernel passes when |got - want| <= C_FP32 scale +
tiny for every element; every scale is PER_U (2 u / C_FP32) times a first-order worst case in units of u = 2^-24, so the bound
is twice that worst case.  CUDA's expf and __fdividef are within 2 ulp (4 u), logf within 1 ulp, fmaf rounds once.

Draws.  Click c of impression id (global), r its ordinal among the impression's clicks: u_d = word d & 3 of Philox4x32-10, key
  (seed lo, seed hi), counter (id lo, r, epoch lo, d >> 2).  S_c = N when K = 0 or K >= |N|; otherwise Floyd's algorithm over
  the ordinals into N (item order): for d = 0 .. K - 1, j = |N| - K + d, t = floor(u_d (j + 1) / 2^32), take j if t is already
  chosen, else t.

Per click c, over A_c = {c} + S_c with exact scores s, M = max_A s, x_k = s_k - M, Z = Sum_A e^{x_k}, p_k = e^{x_k} / Z:
  Scores.  |s^ - s| <= u d_k with d_k = L S_k, L = ceil(H / 32) + 5, S_k = Sum_i |h_i e_ki| (impression_kernel_oracle.scores).
    Through p: dp_j = p_j (ds_j - Sum_k p_k ds_k), so |dp_j| <= u p_j (d_j + dbar), dbar = Sum_A p_k d_k.
  Each e_k is expf of a rounded difference: (|x_k| + 4) u relative; the full path (S_c = N) takes e^{s_n - M_c} as
    expf(s_n - M_N) expf(M_N - M_c), (|x_k| + 8) u.  Z sums |S_c| + 1 positive terms: lanes then the 5-level tree then the last
    add or fma, at most ceil(|S_c| / 32) + 6 roundings of Z:
                                          zeta = Sum_A p_k (|x_k| + 8) + ceil(|S_c| / 32) + 6   (|Z^ - Z| <= zeta u Z).
    rz = __fdividef(1, Z): zeta + 4.
  Non-click n in S_c: p = e rz rounds once more, and the weights of n summed over the clicks that score it (sequentially in the
    sampled path, |C| adds at most; in the full path the per-lane fma sum and tree of R = Sum_c e^{M_N - M_c} / Z_c, then the
    product, ceil(|C| / 32) + 6): per term
                                          p_n (|x_n| + 8 + zeta + 4 + |C| + 6 + d_n + dbar).
  The click's weight p_c - 1 = fmaf(e_c, rz, -1):     p_c (|x_c| + 8 + zeta + 4 + d_c + dbar) + |p_c - 1|.
  g_j = fp32(scale w_j) rounds once; dh_p[i] = the fmaf chain over the M_p candidates of position p with a nonzero weight, in
    item order (M_p <= the size of the union of the A_c), adding at most M_p u Sum_j |g_j e_ji|:
                                          scale_dh = Sum_j |scale| |e_ji| ((M_p + 2) |w_j| + scale_w,j).
  The loss l_c = logf(Z) - x_c: Z's error (zeta), logf's 2 u |log Z|, x_c's rounding |x_c|, the subtraction |l_c|, and the scores
    through dl/ds_k = p_k - [k = c]:      zeta + 2 |log Z| + |x_c| + |l_c| + (1 - p_c) d_c + Sum_{k != c} p_k d_k.
    Each l_c is added to an fp64 sum (rounding far below the bound).
"""
import numpy as np

from impression_kernel_oracle import C_FP32, PER_U, TINY, WORST, check, emu_dot, fma, lanes, usable, xor_tree  # noqa: F401
from salt_pepper_oracle import philox4x32_10

f32 = np.float32
M32 = 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------------------------------
# draws
# ---------------------------------------------------------------------------------------------------------------------------
def draws(seed, epoch, ids, r, K):
    """uint64 [n, K]: u_d of click ordinal r[i] of impression ids[i] (broadcast), d = 0 .. K - 1."""
    ids, r = np.broadcast_arrays(np.asarray(ids, np.uint64).reshape(-1), np.asarray(r, np.uint64).reshape(-1))
    d = np.arange(K, dtype=np.uint64)
    c = philox4x32_10((ids[:, None], r[:, None], np.uint64(epoch & M32), (d >> np.uint64(2))[None, :]),
                      (seed & M32, (seed >> 32) & M32))
    words = np.stack(c, 0)                                        # [4, n, K]
    return np.take_along_axis(words, (d & np.uint64(3)).astype(np.int64)[None, None, :].repeat(ids.size, 1), 0)[0]


def floyd(u, nn, K, collision_rule=True):
    """Floyd's algorithm on the draws u [K]: the chosen ordinals into N, in the order chosen."""
    sel = []
    for d in range(K):
        j = nn - K + d
        t = int((int(u[d]) * (j + 1)) >> 32)
        sel.append(j if (collision_rule and t in sel) else t)
    return sel


def negative_sets(clicked_q, imp_id, K, seed, epoch):
    """[(c, S_c)] for one impression: c the position of each click in item order, S_c the positions of its negatives (sorted)."""
    c = np.asarray(clicked_q) != 0
    cpos, npos = np.flatnonzero(c), np.flatnonzero(~c)
    nn = npos.size
    if K == 0 or K >= nn:
        return [(int(x), npos) for x in cpos]
    u = draws(seed, epoch, imp_id, np.arange(cpos.size), K)
    return [(int(x), np.sort(npos[floyd(u[r], nn, K)])) for r, x in enumerate(cpos)]


# ---------------------------------------------------------------------------------------------------------------------------
# the fp64 reference and its bounds
# ---------------------------------------------------------------------------------------------------------------------------
def softmax_loss(h, emb, pos_indptr, indptr, items, clicked, ids, K, seed, epoch, scale, H):
    """dae_impression_softmax_loss: (dh [P, H], dh scale, loss sum, loss-sum scale, sets) with sets[q] = negative_sets of
    impression q (None when skipped)."""
    h, emb64 = np.asarray(h, np.float64)[:, :H], np.asarray(emb, np.float64)[:, :H]
    pos_indptr, indptr = np.asarray(pos_indptr, np.int64), np.asarray(indptr, np.int64)
    items, clicked = np.asarray(items, np.int64), np.asarray(clicked) != 0
    P = h.shape[0]
    sc = abs(float(f32(scale)))
    L = lanes(H)
    dh, sdh = np.zeros((P, H)), np.zeros((P, H))
    loss = loss_scale = 0.0
    sets = {}
    ok = usable(indptr, clicked)
    for p in range(P):
        rows = []                                            # (item, w, scale_w) of every candidate at p
        for q in range(int(pos_indptr[p]), int(pos_indptr[p + 1])):
            if not ok[q]:
                sets[q] = None
                continue
            b0, b1 = indptr[q], indptr[q + 1]
            it, c = items[b0:b1], clicked[b0:b1]
            E = emb64[it]
            s = E @ h[p]
            dl = L * (np.abs(E * h[p]).sum(1))
            sets[q] = negative_sets(c, int(ids[q]), K, seed, epoch)
            nc = int(c.sum())
            w, sw = np.zeros(it.size), np.zeros(it.size)
            for cp, S in sets[q]:
                A = np.concatenate([[cp], S])
                x = s[A] - s[A].max()
                e = np.exp(x)
                Z = e.sum()
                pr = e / Z
                dbar = (pr * dl[A]).sum()
                zeta = (pr * (np.abs(x) + 8)).sum() + -(-S.size // 32) + 6
                w[S] += pr[1:]
                sw[S] += pr[1:] * (np.abs(x[1:]) + 8 + zeta + 4 + nc + 6 + dl[S] + dbar)
                w[cp] = pr[0] - 1.0
                sw[cp] = pr[0] * (abs(x[0]) + 8 + zeta + 4 + dl[cp] + dbar) + abs(pr[0] - 1.0)
                lc = np.log(Z) - x[0]
                loss += lc
                loss_scale += zeta + 2 * abs(np.log(Z)) + abs(x[0]) + abs(lc) + (1 - pr[0]) * dl[cp] + (pr[1:] * dl[S]).sum()
            cand = np.flatnonzero(w != 0)
            rows.append((it[cand], w[cand], sw[cand]))
        if not rows:
            continue
        it = np.concatenate([r[0] for r in rows])
        w = np.concatenate([r[1] for r in rows])
        sw = np.concatenate([r[2] for r in rows])
        E = emb64[it]
        dh[p] = float(f32(scale)) * (w @ E)
        sdh[p] = sc * (((it.size + 2) * np.abs(w) + sw) @ np.abs(E))
    return dh, PER_U * sdh, loss, PER_U * loss_scale, sets


# ---------------------------------------------------------------------------------------------------------------------------
# float32 emulation, in the kernel's operation order
# ---------------------------------------------------------------------------------------------------------------------------
def _lane_sums(v, op):
    """Per-lane sequential reduction of v (lane l takes entries l, l + 32, ...) with op, fp32: [32]."""
    out = np.zeros(32, f32)
    for k, x in enumerate(v):
        out[k % 32] = op(out[k % 32], x)
    return out


def emu_softmax_loss(h, emb, pos_indptr, indptr, items, clicked, ids, K, seed, epoch, scale, H, mutate=None):
    """impression_softmax_loss_kernel in fp32: (dh [P, H] fp32, loss sum).  mutate: None, or 'no_max' (the max not subtracted)
    or 'no_minus_one' (the click's weight p_cc in place of p_cc - 1), for the host tests that show the bounds catch them."""
    h, emb = np.asarray(h, f32), np.asarray(emb, f32)
    items, clicked = np.asarray(items, np.int64), np.asarray(clicked) != 0
    P = h.shape[0]
    dh = np.zeros((P, H), f32)
    total = 0.0
    sc = f32(scale)
    one = f32(1)
    with np.errstate(over='ignore', under='ignore', invalid='ignore'):
        for p in range(P):
            d = np.zeros(H, f32)
            for q in range(int(pos_indptr[p]), int(pos_indptr[p + 1])):
                b0, m = int(indptr[q]), int(indptr[q + 1] - indptr[q])
                it, c = items[b0:b0 + m], clicked[b0:b0 + m]
                nc = int(c.sum())
                nn = m - nc
                if nc == 0 or nn == 0:
                    continue
                s = emu_dot(h[p], emb[it], H)
                w = np.zeros(m, f32)
                minus = f32(0) if mutate == 'no_minus_one' else f32(-1)
                if K == 0 or K >= nn:
                    mn = f32(s[~c].max()) if mutate != 'no_max' else f32(0)
                    t = _lane_sums([np.exp(f32(s[k] - mn)) if not c[k] else f32(0) for k in range(m)], lambda a, b: f32(a + b))
                    tn = xor_tree(t)
                    r = np.zeros(32, f32)
                    for k in np.flatnonzero(c):
                        mc = max(s[k], mn) if mutate != 'no_max' else f32(0)
                        xc = f32(s[k] - mc)
                        ec, en = f32(np.exp(xc)), f32(np.exp(f32(mn - mc)))
                        z = fma(en, tn, ec)
                        rz = f32(one / z)
                        total += float(f32(f32(np.log(z)) - xc))
                        r[k % 32] = fma(en, rz, r[k % 32])
                        w[k] = fma(ec, rz, minus)
                    rn = xor_tree(r)
                    for k in np.flatnonzero(~c):
                        w[k] = f32(f32(np.exp(f32(s[k] - mn))) * rn)
                else:
                    npos = np.flatnonzero(~c)
                    for r, cp in enumerate(np.flatnonzero(c)):
                        u = draws(seed, epoch, int(ids[q]), r, K)[0]
                        pos = npos[floyd(u, nn, K)]
                        sd = emu_dot(h[p], emb[it[pos]], H)
                        scc = s[cp]
                        mc = f32(max(scc, sd.max())) if mutate != 'no_max' else f32(0)
                        xc = f32(scc - mc)
                        ec = f32(np.exp(xc))
                        e = np.zeros(32, f32)
                        e[:K] = np.exp((sd - mc).astype(f32)).astype(f32)
                        z = f32(xor_tree(e) + ec)
                        rz = f32(one / z)
                        w[pos] = (w[pos] + (e[:K] * rz).astype(f32)).astype(f32)
                        w[cp] = fma(ec, rz, minus)
                        total += float(f32(f32(np.log(z)) - xc))
                for k in range(m):
                    g = f32(sc * w[k])
                    if g != 0:
                        d = fma(g, emb[it[k], :H], d)
            dh[p] = d
    return dh, total


# ---------------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------------
def impression_ids(rng, n):
    """n distinct global impression ids spread over [0, 2^32), the largest 2^32 - 1."""
    ids = np.unique(rng.integers(0, 2 ** 32 - 1, n + 16, dtype=np.uint64))[:n].astype(np.int64)
    rng.shuffle(ids)
    ids[-1] = 2 ** 32 - 1
    assert np.unique(ids).size == n
    return ids
