"""fp64 references of the two impression kernels (csrc/impressions.cu) with per-element error bounds, float32 emulations of both
kernels in their operation order, and the edge inputs the kernel tests share.  Tests only.

As in gru_kernel_oracle.py, a reference returns (value, scale) and a kernel passes when, for every element,

    |got - want| <= C_FP32 * scale + tiny.

Here every scale is PER_U = 2 u / C_FP32 times a first-order worst case counted in units of u = 2^-24 (fp32 rounding), so the
bound is twice that worst case; the factor 2 holds the second-order terms (below n u = 3e-4 of the first-order ones for the
longest sums here).  The fp32 inputs are taken exact; 1 ulp <= 2 u relative.  CUDA's expf and __fdividef are within 2 ulp (4 u),
log1pf within 1 ulp, sqrtf and the fp32 '/' are correctly rounded, fmaf rounds once.  With L = ceil(H / 32) + 5:

Scores (both kernels).  Lane l sums its ceil(H / 32) products with fmaf, each rounding at most u of the running sum, and the
  5-level xor tree rounds once per level: |s^ - s| <= L u S with S = Sum_j |q_j e_j|.            scale_s = L S.
  Cosine s / (|q| |e|): qq and ee are sums of non-negative terms (L u relative); sqrtf halves that and rounds once, the product
  and the divide round once each: the denominator carries (L + 3) u relative, the quotient one more.
                                                    scale_cos = L S / (|q| |e|) + (L + 4) |cos|.
  A zero q or e scores exactly 0 (scale 0).

dh of dae_impression_rank_loss, position p, column i.  For impression q at p with clicked set C, non-clicked N, m = |C| + |N|:
  x = s_n - s_c from the kernel's scores:           |x^ - x| <= u scale_x,   scale_x = L (S_n + S_c) + |x|.
  sigma(x) = __fdividef(1, 1 + expf(-x)): expf 4 u of e^-x, the add u of 1 + e^-x, the divide 4 u: 9 u of sigma, plus sigma's
    slope sigma (1 - sigma) on x's error.  (Where 1 + e^-x > 2^126 __fdividef returns 0: an absolute error below 2^-126, far
    under tiny.)
  w_j = Sum_k +-sigma over the n_j = |other class| candidates k, in index order, in fp32 (the 256-score chunks carry s_w in
    shared memory, so this is one sequential sum): its rounding adds at most n_j u Sum_k sigma = n_j u |w_j|:
                                                    scale_w = (n_j + 9) |w_j| + Sum_k sigma (1 - sigma) scale_x.
  coef = fp32(scale / (|C| |N|)) rounds once (1/(|C||N|) is fp64-accurate), g = coef w_j once more: |g^ - g| <= u |coef|
    (2 |w_j| + scale_w).
  dh_p[i] = fmaf over every candidate t of every usable impression at p, M_p of them in all: the accumulation adds at most
    M_p u Sum_t |g_t e_ti|:                         scale_dh = Sum_t |coef_t| |e_ti| ((M_p + 2) |w_t| + scale_w,t).
  Rows without a usable impression are exactly 0.
The loss: softplus(x) = max(x, 0) + log1pf(expf(-|x|)): x's error through the slope sigma, expf's 4 u of e through log1p (at most
  4 u of log1p(e), as e / (1 + e) <= log1p(e)), log1pf's 2 u and the add's u: sigma scale_x + 7 softplus.  Lane j sums its terms
  of one chunk pair in fp32 (lj, n_B = the non-clicked candidates of chunk B: n_B u Sum softplus), the rest is fp64.  Per term
                                                    scale_l = (sigma scale_x + (7 + n_B) softplus(x)) / (|C| |N|),
  and the loss sum is checked against Sum scale_l.

Metrics: impression_oracle.metrics on the kernel's own scores.
"""
import numpy as np

from gru_kernel_oracle import C_FP32, TINY, WORST, check, sigmoid, softplus  # noqa: F401  (re-exported for the tests)

U = 2.0 ** -24
PER_U = 2 * U / C_FP32        # a scale of PER_U k is a bound of 2 k u
CHUNK = 256                   # kImpChunk
f32 = np.float32


def lanes(H):
    """L: the longest lane's fma count plus the tree's 5 levels."""
    return -(-H // 32) + 5


# ---------------------------------------------------------------------------------------------------------------------------
# scores
# ---------------------------------------------------------------------------------------------------------------------------
def _dot_abs(Q, E, rows=8192):
    """Row-wise Sum_j q_j e_j and Sum_j |q_j e_j| in fp64, in blocks of rows."""
    n = Q.shape[0]
    s, S = np.empty(n), np.empty(n)
    for a in range(0, n, rows):
        q, e = np.asarray(Q[a:a + rows], np.float64), np.asarray(E[a:a + rows], np.float64)
        s[a:a + rows] = (q * e).sum(1)
        S[a:a + rows] = np.abs(q * e).sum(1)
    return s, S


def scores(q, emb, indptr, items, cosine, H):
    """dae_impression_metrics' scores: (value, scale) for every shown article of every impression (row i of q against
    emb[items[k]] for k in [indptr[i], indptr[i + 1]))."""
    q, emb = np.asarray(q)[:, :H], np.asarray(emb)[:, :H]
    row = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    Q, E = q[row], emb[np.asarray(items, np.int64)]
    s, S = _dot_abs(Q, E)
    L = lanes(H)
    if not cosine:
        return s, PER_U * L * S
    nq = np.sqrt((np.asarray(q, np.float64) ** 2).sum(1))[row]
    ne = np.sqrt((np.asarray(emb, np.float64) ** 2).sum(1))[np.asarray(items, np.int64)]
    ok = (nq > 0) & (ne > 0)
    den = np.where(ok, nq * ne, 1.0)
    c = np.where(ok, s / den, 0.0)
    return c, np.where(ok, PER_U * (L * S / den + (L + 4) * np.abs(c)), 0.0)


# ---------------------------------------------------------------------------------------------------------------------------
# impression loss
# ---------------------------------------------------------------------------------------------------------------------------
def usable(indptr, clicked):
    """Boolean [I]: at least one click and one non-click."""
    m = np.diff(indptr)
    cs = np.concatenate([[0], np.cumsum(np.asarray(clicked) != 0, dtype=np.int64)])
    nc = cs[indptr[1:]] - cs[indptr[:-1]]
    return (nc > 0) & (nc < m)


def rank_loss(h, emb, pos_indptr, indptr, items, clicked, scale, H):
    """dae_impression_rank_loss: (dh [P, H], dh scale, loss sum, loss-sum scale).  scale is the kernel's float argument."""
    import scipy.sparse as sp
    h, emb = np.asarray(h, np.float64)[:, :H], np.asarray(emb)[:, :H]
    pos_indptr, indptr = np.asarray(pos_indptr, np.int64), np.asarray(indptr, np.int64)
    items, clicked = np.asarray(items, np.int64), np.asarray(clicked) != 0
    P = h.shape[0]
    sc = float(f32(scale))
    L = lanes(H)
    ok = usable(indptr, clicked)
    pos_of = np.repeat(np.arange(P), np.diff(pos_indptr))          # the position of each impression id below pos_indptr[P]
    mq = np.diff(indptr)[:pos_of.size] * ok[:pos_of.size]
    M = np.bincount(pos_of, weights=mq, minlength=P)               # M_p: the fma count of row p
    t_pos, t_item, t_g, t_a = [], [], [], []
    loss = loss_scale = 0.0
    for q in np.flatnonzero(ok[:pos_of.size]):
        p = pos_of[q]
        b0, b1 = indptr[q], indptr[q + 1]
        it, c = items[b0:b1], clicked[b0:b1]
        s, S = _dot_abs(np.broadcast_to(h[p], (it.size, H)), emb[it])
        x = s[~c][None, :] - s[c][:, None]                         # [|C|, |N|]: s_n - s_c
        sx = L * (S[~c][None, :] + S[c][:, None]) + np.abs(x)
        sg = sigmoid(x)
        slope = sg * (1.0 - sg) * sx
        nc, nn = int(c.sum()), int((~c).sum())
        w = np.empty(it.size)
        w[~c], w[c] = sg.sum(0), -sg.sum(1)
        sw = np.empty(it.size)
        sw[~c] = (nc + 9) * sg.sum(0) + slope.sum(0)
        sw[c] = (nn + 9) * sg.sum(1) + slope.sum(1)
        inv = 1.0 / (nc * nn)
        coef = sc * inv
        t_pos.append(np.full(it.size, p))
        t_item.append(it)
        t_g.append(coef * w)
        t_a.append(abs(coef) * ((M[p] + 2) * np.abs(w) + sw))
        sp_ = softplus(x)
        chunk_nn = np.bincount(np.flatnonzero(~c) // CHUNK, minlength=-(-it.size // CHUNK))
        n_b = chunk_nn[np.flatnonzero(~c) // CHUNK][None, :]
        loss += sp_.sum() * inv
        loss_scale += (sg * sx + (7 + n_b) * sp_).sum() * inv
    if not t_pos:
        return np.zeros((P, H)), np.zeros((P, H)), 0.0, 0.0
    tp, ti = np.concatenate(t_pos), np.concatenate(t_item)
    shape = (P, tp.size)
    cols = np.arange(tp.size)
    G = sp.csr_matrix((np.concatenate(t_g), (tp, cols)), shape=shape)
    A = sp.csr_matrix((np.concatenate(t_a), (tp, cols)), shape=shape)
    E = np.asarray(emb, np.float64)[ti]
    return np.asarray(G @ E), PER_U * np.asarray(A @ np.abs(E)), loss, PER_U * loss_scale


# ---------------------------------------------------------------------------------------------------------------------------
# float32 emulations, in the kernels' operation order
# ---------------------------------------------------------------------------------------------------------------------------
def fma(a, b, c):
    """fmaf: the fp32 product is exact in fp64; the sum then rounds twice (fp64, fp32), which can differ from one rounding by an
    ulp on rare ties: close enough for an emulation checked against a bound."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def xor_tree(v):
    """warp_sum over the last axis (32 lanes): v += shfl_xor(v, o) for o = 16 .. 1, in fp32."""
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., idx ^ o]).astype(f32)
    return v[..., 0]


def emu_dot(a, B, H, sq=False):
    """Lane-strided fmaf (lane l takes columns l, l + 32, ...) then the xor tree: a [H] against every row of B [n, H].  With sq,
    also the rows' squared norms, summed the same way (the metrics kernel's fused loop)."""
    nl = -(-H // 32)
    A = np.zeros(nl * 32, f32)
    A[:H] = a[:H]
    BB = np.zeros((B.shape[0], nl * 32), f32)
    BB[:, :H] = B[:, :H]
    s = np.zeros((B.shape[0], 32), f32)
    e = np.zeros((B.shape[0], 32), f32)
    for r in range(nl):
        blk = BB[:, r * 32:(r + 1) * 32]
        s = fma(A[None, r * 32:(r + 1) * 32], blk, s)
        if sq:
            e = fma(blk, blk, e)
    return (xor_tree(s), xor_tree(e)) if sq else xor_tree(s)


def emu_scores(q, emb, indptr, items, cosine, H):
    """impression_metrics_kernel's fp32 scores."""
    out = np.zeros(int(indptr[-1]), f32)
    for i in range(len(indptr) - 1):
        b0, b1 = int(indptr[i]), int(indptr[i + 1])
        if b1 == b0:
            continue
        dot, ee = emu_dot(q[i], emb[np.asarray(items[b0:b1], np.int64)], H, sq=True)
        if not cosine:
            out[b0:b1] = dot
            continue
        qn = np.sqrt(emu_dot(q[i], q[i][None, :], H)[0]).astype(f32)
        ok = (qn > 0) & (ee > 0)
        den = (qn * np.sqrt(ee).astype(f32)).astype(f32)
        out[b0:b1] = np.where(ok, dot / np.where(ok, den, f32(1)), f32(0)).astype(f32)
    return out


def emu_sigmoid(x):
    e = np.exp(-x).astype(f32)
    d = (f32(1) + e).astype(f32)
    return np.where(d > f32(2.0 ** 126), f32(0), (f32(1) / d).astype(f32))   # __fdividef(1, y) = 0 for y > 2^126


def emu_softplus(x):
    return (np.maximum(x, f32(0)) + np.log1p(np.exp(-np.abs(x)).astype(f32)).astype(f32)).astype(f32)


def emu_rank_loss(h, emb, pos_indptr, indptr, items, clicked, scale, H):
    """impression_rank_loss_kernel in fp32: (dh [P, H] fp32, loss sum)."""
    h, emb = np.asarray(h, f32), np.asarray(emb, f32)
    items, clicked = np.asarray(items, np.int64), np.asarray(clicked) != 0
    P = h.shape[0]
    dh = np.zeros((P, H), f32)
    total = 0.0
    sc = f32(scale)
    with np.errstate(over='ignore', under='ignore'):
        for p in range(P):
            d = np.zeros(H, f32)
            for q in range(int(pos_indptr[p]), int(pos_indptr[p + 1])):
                b0, m = int(indptr[q]), int(indptr[q + 1] - indptr[q])
                it, c = items[b0:b0 + m], clicked[b0:b0 + m]
                nc = int(c.sum())
                nn = m - nc
                if nc == 0 or nn == 0:
                    continue
                inv = 1.0 / (float(nc) * float(nn))
                coef = f32(float(sc) * inv)
                l_imp = 0.0
                for a0 in range(0, m, CHUNK):
                    na = min(CHUNK, m - a0)
                    sa, fa = emu_dot(h[p], emb[it[a0:a0 + na]], H), c[a0:a0 + na]
                    sw = np.zeros(na, f32)
                    for c0 in range(0, m, CHUNK):
                        nb = min(CHUNK, m - c0)
                        sb, fb = (sa, fa) if c0 == a0 else (emu_dot(h[p], emb[it[c0:c0 + nb]], H), c[c0:c0 + nb])
                        other = fb[None, :] != fa[:, None]
                        xc = (sb[None, :] - sa[:, None]).astype(f32)          # j clicked: x = s_k - s_j
                        xn = (sa[:, None] - sb[None, :]).astype(f32)          # j not clicked: x = s_j - s_k
                        terms = np.where(other, np.where(fa[:, None], -emu_sigmoid(xc), emu_sigmoid(xn)), f32(0))
                        sw = np.add.accumulate(np.concatenate([sw[:, None], terms], 1), axis=1, dtype=f32)[:, -1]
                        lt = np.where(other & fa[:, None], emu_softplus(xc), f32(0))
                        lj = np.add.accumulate(np.concatenate([np.zeros((na, 1), f32), lt], 1), axis=1, dtype=f32)[:, -1]
                        l_imp += float(lj.astype(np.float64).sum())
                    for t in range(na):
                        g = f32(coef * sw[t])
                        d = fma(g, emb[it[a0 + t], :H], d)
                total += l_imp * inv
            dh[p] = d
    return dh, total


def emu_metrics(scores, indptr, clicked):
    """impression_metrics_kernel's metrics from fp32 scores: ([I, 4], [I, 2] = 2 x the AUC numerator and the sum of the clicked
    ranks).  Ranks and the AUC numerator are counted in integers chunk by chunk, as the kernel does; MRR and the DCGs are summed
    per lane (clicked candidate j is lane j % 32) and then over the xor tree in fp64."""
    s_all, c_all = np.asarray(scores, f32), np.asarray(clicked) != 0
    n_imp = len(indptr) - 1
    out = np.full((n_imp, 4), np.nan)
    ints = np.zeros((n_imp, 2), np.int64)
    for i in range(n_imp):
        b0, m = int(indptr[i]), int(indptr[i + 1] - indptr[i])
        s, c = s_all[b0:b0 + m], c_all[b0:b0 + m]
        nc = int(c.sum())
        nn = m - nc
        if nc == 0 or nn == 0:
            continue
        auc2, rsum = 0, 0
        rr, g5, g10 = np.zeros(32), np.zeros(32), np.zeros(32)
        for j in np.flatnonzero(c):
            gt = tie_before = below_n = tie_n = 0
            for k0 in range(0, m, CHUNK):
                sk, fk = s[k0:k0 + CHUNK], c[k0:k0 + CHUNK]
                kk = k0 + np.arange(sk.size)
                gt += int((sk > s[j]).sum())
                tie_before += int(((sk == s[j]) & (kk < j)).sum())
                below_n += int(((sk < s[j]) & ~fk).sum())
                tie_n += int(((sk == s[j]) & ~fk).sum())
            rank = gt + tie_before
            auc2 += 2 * below_n + tie_n
            rsum += rank
            rr[j % 32] += 1.0 / float(rank + 1)
            if rank < 10:
                g = 1.0 / np.log2(float(rank + 2))
                g10[j % 32] += g
                if rank < 5:
                    g5[j % 32] += g
        rr, g5, g10 = (_tree64(v) for v in (rr, g5, g10))
        i5 = i10 = 0.0
        for r in range(min(10, nc)):
            g = 1.0 / np.log2(float(r + 2))
            i10 += g
            if r < 5:
                i5 += g
        ints[i] = auc2, rsum
        out[i] = auc2 / (2.0 * nc * nn), rr / nc, g5 / i5, g10 / i10
    return out, ints


def _tree64(v):
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[idx ^ o]
    return float(v[0])


# ---------------------------------------------------------------------------------------------------------------------------
# edge inputs
# ---------------------------------------------------------------------------------------------------------------------------
X_EDGES = (100.0, -100.0, 88.0, -88.0, 30.0, -30.0, 0.0, 1e-3)


def _clicks(rng, m, p=0.3):
    c = (rng.random(m) < p).astype(np.uint8)
    if m > 1:
        j = int(rng.integers(0, m))
        c[j], c[(j + 1) % m] = 1, 0
    return c


def loss_case(rng, H, n_pos, N=6000):
    """Edge inputs of dae_impression_rank_loss: (h [n_pos, H], emb [N, H], pos_indptr, indptr, items, clicked, info).  Impressions
    of 0, 1, 2, 255, 256, 257, 511, 512, 513 and 5 000 articles; clicks all in the first chunk, all in the last, a single click,
    a single non-click; skipped impressions (empty, all clicked, none clicked) beside usable ones and alone; one position showing
    the same articles in three impressions; article N - 1; pairs with x = s_n - s_c at X_EDGES (h along e_n - e_c).  The
    positions with impressions are spread over [0, n_pos), most positions have none.  info: {'skipped_only': positions whose
    impressions are all skipped, 'x_pos': the positions of the X_EDGES pairs}."""
    emb = (rng.standard_normal((N, H)) / np.sqrt(H)).astype(f32)
    h = (rng.standard_normal((n_pos, H)) * rng.choice([0.1, 1.0, 3.0], (n_pos, 1))).astype(f32)
    live = np.unique(np.linspace(0, n_pos - 2, min(n_pos, 90) - 1).astype(np.int64))
    rng.shuffle(live)
    live = list(live) + [n_pos - 1]                                  # the last position is popped first
    imps = []                                                        # (position, items, clicks)

    def add(p, m, c=None, items=None):
        it = rng.choice(N, m, replace=False) if items is None else np.asarray(items)
        imps.append((p, it.astype(np.int32), _clicks(rng, m) if c is None else np.asarray(c, np.uint8)))

    for m in (0, 1, 2, 255, 256, 257, 511, 512, 513, 5000):
        p = live.pop()
        add(p, m)
        if m < 2:                                                    # skipped: a usable impression follows at the same position
            add(p, int(rng.integers(2, 20)))
    p = live.pop()
    add(p, 700, np.arange(700) < 40)                                 # every click in the first chunk
    add(p, 0)                                                        # skipped impressions beside usable ones
    add(p, 9, np.ones(9))
    add(p, 700, np.arange(700) >= 530)                               # every click in the last chunk
    add(p, 12, np.zeros(12))
    p = live.pop()
    add(p, 300, np.arange(300) == 299)                               # a single click
    add(p, 300, np.arange(300) != 0)                                 # a single non-click
    c5000 = np.zeros(5000, np.uint8)
    c5000[rng.choice(5000, 700, replace=False)] = 1
    add(live.pop(), 5000, c5000)                                     # |C| = 700 spread over 20 chunks
    skipped_only = [live.pop(), live.pop()]
    add(skipped_only[0], 0)
    add(skipped_only[0], 5, np.ones(5))
    add(skipped_only[1], 7, np.zeros(7))
    p = live.pop()                                                   # the same articles in three impressions, and row N - 1
    base = rng.choice(N - 1, 30, replace=False)
    add(p, 31, None, np.concatenate([base, [N - 1]]))
    add(p, 20, None, np.concatenate([base[:19], [N - 1]]))
    add(p, 10, None, base[5:15])
    x_pos = []
    for x in X_EDGES:
        p = live.pop()
        cl, nx = rng.choice(N, 2, replace=False)
        d = emb[nx].astype(np.float64) - emb[cl]
        h[p] = (x * d / max(float(d @ d), 1e-30)).astype(f32)
        add(p, 2, [1, 0], [cl, nx])
        x_pos.append(p)
    while live:                                                      # the rest: 1 - 3 short impressions each
        p = live.pop()
        for _ in range(int(rng.integers(1, 4))):
            add(p, int(rng.integers(2, 20)))
    imps.sort(key=lambda t: t[0])                                    # stable: a position's impressions keep their order
    pos = np.array([t[0] for t in imps], np.int64)
    pos_indptr = np.zeros(n_pos + 1, np.int64)
    np.cumsum(np.bincount(pos, minlength=n_pos), out=pos_indptr[1:])
    indptr = np.concatenate([[0], np.cumsum([t[1].size for t in imps])]).astype(np.int64)
    items = np.concatenate([t[1] for t in imps]).astype(np.int32)
    clicked = np.concatenate([t[2] for t in imps]).astype(np.uint8)
    return h, emb, pos_indptr, indptr, items, clicked, {'skipped_only': skipped_only, 'x_pos': x_pos}


def metrics_case(rng, H, n_imp, N=3000):
    """Edge inputs of dae_impression_metrics: (q [n_imp, H], emb [N, H], indptr, items, clicked, info).  Ties across the
    256-score chunk boundary (articles with identical rows), 100 clicks (four 32-lane groups), single clicks ranked exactly 4, 5,
    9 and 10 under both metrics (info['rank'] maps impression -> rank), 13 clicks (the ideal DCG capped at 10), empty and
    single-candidate impressions, a zero query and zero articles; short random impressions fill the rest."""
    emb = (rng.standard_normal((N, H)) / np.sqrt(H)).astype(f32)
    unit = np.arange(200)                                            # unit rows: linear and cosine rank them alike
    emb[unit] /= np.linalg.norm(emb[unit].astype(np.float64), axis=1, keepdims=True).astype(f32)
    emb[N - 16:N - 4] = emb[N - 4]                                   # articles N - 16 .. N - 4: identical rows
    zero = [N - 3, N - 2]
    emb[zero] = 0
    q = rng.standard_normal((n_imp, H)).astype(f32)
    lists = []
    rank = {}
    dup = np.arange(N - 16, N - 3)
    it = rng.choice(N - 16, 600, replace=False)
    it[248:248 + dup.size] = dup                                     # ties at positions 248 .. 260, across 256
    c = np.zeros(600, np.uint8)
    c[[250, 255, 257, 260, 10, 400]] = 1
    lists.append((it, c))
    lists.append((rng.choice(N - 16, 300, replace=False), (np.arange(300) % 3 == 0).astype(np.uint8)))   # 100 clicks
    lists.append((rng.choice(N - 16, 40, replace=False), (np.arange(40) % 3 == 1).astype(np.uint8)[:40]))  # 13 clicks
    lists.append((np.array([], np.int32), np.array([], np.uint8)))
    lists.append((np.array([5]), np.array([1], np.uint8)))
    lists.append((np.array([6]), np.array([0], np.uint8)))
    lists.append((np.concatenate([rng.choice(N - 16, 8, replace=False), zero]), _clicks(rng, 10)))
    zq = len(lists)
    lists.append((rng.choice(N - 16, 9, replace=False), _clicks(rng, 9)))                              # the zero query
    for r in (4, 5, 9, 10, 0, 14):
        i = len(lists)
        it = rng.choice(unit, 15, replace=False)
        s = emb[it].astype(np.float64) @ q[i].astype(np.float64)
        c = np.zeros(15, np.uint8)
        c[np.argsort(-s, kind='stable')[r]] = 1
        lists.append((it, c))
        rank[i] = r
    lists.append((rng.choice(N - 16, 1000, replace=False), _clicks(rng, 1000, 0.05)))
    while len(lists) < n_imp:
        m = int(rng.integers(0, 8))
        lists.append((rng.choice(N, m, replace=False), _clicks(rng, m)))
    q[zq] = 0
    indptr = np.concatenate([[0], np.cumsum([t[0].size for t in lists])]).astype(np.int64)
    items = np.concatenate([t[0] for t in lists]).astype(np.int32)
    clicked = np.concatenate([t[1] for t in lists]).astype(np.uint8)
    return q, emb, indptr, items, clicked, {'rank': rank, 'zero_query': zq, 'zero_items': zero}
