"""fp64 references of the GRU user encoder's kernels (csrc/user_gru.cu) and of the two kernels around the dense similarity GEMM
(csrc/similarity.cu), for the kernel-level tests.  Tests only.

As in step_kernel_oracle.py, a reference returns the value and a per-element error scale, and a kernel passes when, for every
element,

    |got - want| <= c * scale + tiny

with c = C_FP32 (2^-20, 16 units of fp32 rounding u = 2^-24) for the CUDA-core kernels and C_BF16X3 (2^-14) for the GEMMs.  Every
reference starts from the kernel's own fp32 inputs, so a bound covers that kernel's arithmetic and nothing upstream of it.  The
scales, with s(a) = 1 / (1 + e^-a) and the fp32 inputs taken exact:

gather_split and seq_negatives: bit-exact (a copy with a bf16 split; integer arithmetic).

Cell forward, from XP = [x_r | x_z | x_n], HP = [h_r | h_z | h_n] and h_prev:
  r = s(x_r + h_r).  The sum rounds once (u (|x_r| + |h_r|)), which s' = r (1 - r) carries into r; expf, the add and the divide
    add a few u of r itself:                        scale_r = r (1 - r) (|x_r| + |h_r|) + r;  scale_z alike.
  n = tanh(x_n + r h_n).  The pre-activation rounds at most twice (u (|x_n| + |r h_n|)), r's error enters through |h_n|, and
    tanh' = 1 - n^2 carries both; tanhf adds a few u of n:
                                                    scale_n = (1 - n^2) (|x_n| + |r h_n| + |h_n| scale_r) + |n|.
  h = (1 - z) n + z h_prev = n + z (h_prev - n).  An error dz moves h by dz (h_prev - n) (1 - z is exact for z >= 1/2 and rounds
    by u |1 - z| below), an error dn by (1 - z) dn, and each product and the sum round once:
                                                    scale_h = |1 - z| scale_n + |n - h_prev| scale_z + |(1 - z) n| + |z h_prev|.
  The stored gates [r | z | n | hn] carry the scales of r, z, n; hn is a copy (exact).  The next step's operand is the bf16 split of
  the kernel's own fp32 h_out, bit for bit.

Cell backward, from the stored gates (r, z, n, hn), the carry, dh_in and h_prev (all exact inputs).  dh = carry + dh_in rounds
  once, D = |carry| + |dh_in|.
  dn = dh (1 - z) (1 - n^2).  1 - n^2 cancels near |n| = 1: it is computed with an ABSOLUTE error of a few u (1 + n^2), so
                                                    scale_dn = D |1 - z| (1 + n^2);
  dz = dh (h_prev - n) z (1 - z):                   scale_dz = D (|h_prev| + |n|) z |1 - z|;
  dr = dn hn r (1 - r), dn's error included:        scale_dr = scale_dn |hn| r |1 - r|;
  dHP's n-third r dn:                               scale = r scale_dn;   new carry dh z:  scale = D z.
  Each is a product of about six correctly rounded factors: under 8 u of its scale.  The bf16 outputs are compared as hi + lo.
  v - hi is exact in fp32 and below 2^(e-8) for v in [2^e, 2^(e+1)), so lo's rounding leaves at most 2^(e-17) <= 2^-17 |v|; the
  tests add that 2^-17 |v| to the bound (the split alone can reach 0.9 of it), and check that hi = rn_bf16(hi + lo) (except
  where lo is exactly half an ulp of hi: hi + lo is then a tie, which rounds to even) and that dHP's r and z thirds equal dXP's bit
  for bit.

seq_rank_loss, per position p with pos >= 0 (dh = 0 exactly otherwise):
  s+ = h . e+, s- = h . e-: fp32 dot products over H (fma per lane, then a warp tree): scale Sum_j |h_j e_j|, the same rule as
    C_FP32's "few units of the sum of absolute terms".  x = s- - s+ carries both: scale_x = S+ + S-.
  s(x) propagates x's error through s' = s (1 - s) and adds its own relative rounding: scale_s = s (1 - s) scale_x + s.
  softplus(x) = max(x, 0) + log1p(e^-|x|) through softplus' = s(x):  scale_l = s scale_x + softplus(x).
  dh_j = scale s(x) (e-_j - e+_j):                 scale = |scale| (s (1 - s) scale_x |e-_j - e+_j| + s (|e-_j| + |e+_j|)).
  The fp64 loss sum is checked against Sum_p scale_l.

GEMMs (bf16x3 on the tensor cores): C_BF16X3 Sum_k |a_k b_k| on the fp32 operands (step_kernel_oracle.py derives C_BF16X3).

rownorm_split: fp64 x / ||x|| (l2, l1, max) or x (kind 0), scale |x / ||x|||: the fp32 sum over the row stays within a few u of
  its (all non-negative) terms, and the reciprocal, square root and product add a few u more.  Rows whose norm is 0 are untouched.
  hi / lo are the bit-exact split of the kernel's own x_out.

row_argmax: bit-exact against row_argmax() below.
"""
import numpy as np

from step_kernel_oracle import C_BF16X3, C_FP32, bf16_split  # noqa: F401  (re-exported for the tests)

TINY = 1e-30
BF16_PAIR = 2.0 ** -17      # |v - hi - lo| <= 2^-17 |v|: the extra bound of a value compared as its bf16 hi + lo
M32 = np.uint64(0xFFFFFFFF)


# ---------------------------------------------------------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------------------------------------------------------
WORST = {}   # name -> worst err / bound seen in this process (the tests print it)


def check(name, got, want, scale, c, tiny=TINY, extra=None):
    """|got - want| <= c * scale + extra + tiny for every element; the message names the first bad indices and the worst one."""
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    scale = np.broadcast_to(np.asarray(scale, np.float64), want.shape)
    err = np.abs(got - want)
    bound = c * scale + tiny + (0.0 if extra is None else extra)
    bad = ~(err <= bound)
    ratio = np.where(np.isfinite(err), err / bound, np.inf)
    if ratio.size:
        WORST[name] = max(WORST.get(name, 0.0), float(ratio.max()))
    if bad.any():
        idx = np.argwhere(bad)[:5]
        worst = np.unravel_index(np.argmax(ratio), err.shape)
        raise AssertionError('%s: %d of %d elements outside the bound (c=%g); first %s; worst at %s: got %r want %r scale %r' %
                             (name, int(bad.sum()), bad.size, c, idx.tolist(), tuple(int(i) for i in worst), got[worst],
                              want[worst], scale[worst]))


def bf16_value(bits):
    """float32 values of bf16 bit patterns (uint16)."""
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(np.float32)


def check_pair(name, hi, lo, want, scale, c):
    """A value stored as a bf16 hi / lo pair: hi + lo against the fp64 value (bound c scale + 2^-17 |want|), and hi = rn(hi + lo)."""
    v = bf16_value(hi).astype(np.float64) + bf16_value(lo).astype(np.float64)
    check(name, v, want, scale, c, extra=BF16_PAIR * np.abs(want))
    # hi = rn(hi + lo), compared as values (hi = -0 with lo = +0 sums to +0).  The one exception: lo may round to exactly half an
    # ulp of hi (v = 0x3d94801c: hi rounds up, v - hi rounds to -2^-12), and hi + lo is then a tie that rounds to even.
    hv = bf16_value(hi).astype(np.float64)
    h2, _ = bf16_split(v.astype(np.float32))
    half_ulp = np.ldexp(1.0, np.frexp(hv)[1] - 9)
    bad = (bf16_value(h2) != hv) & ~(np.abs(bf16_value(lo)) == half_ulp)
    assert not bad.any(), '%s: hi != rn_bf16(hi + lo) at %s' % (name, np.argwhere(bad)[:5].tolist())


def sigmoid(a):
    """1 / (1 + e^-a) to full relative accuracy on both tails (0.5 (1 + tanh(a / 2)) cancels for a << 0)."""
    a = np.asarray(a, np.float64)
    e = np.exp(-np.abs(a))
    return np.where(a >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def softplus(x):
    x = np.asarray(x, np.float64)
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


# ---------------------------------------------------------------------------------------------------------------------------
# Philox4x32-10 (dae_seq_negatives' draws)
# ---------------------------------------------------------------------------------------------------------------------------
def philox_first_word(p, batch, epoch, seed):
    """Philox4x32-10's first output word at counter (p, batch, epoch lo, epoch hi), key seed (NumPy, uint64 lanes)."""
    c = [np.asarray(p, np.uint64) & M32, np.full(np.shape(p), batch & 0xFFFFFFFF, np.uint64),
         np.full(np.shape(p), epoch & 0xFFFFFFFF, np.uint64), np.full(np.shape(p), (epoch >> 32) & 0xFFFFFFFF, np.uint64)]
    k = [np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)]
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & M32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & M32]
        k = [(k[0] + np.uint64(0x9E3779B9)) & M32, (k[1] + np.uint64(0xBB67AE85)) & M32]
    return c[0]


def seq_negatives(pos, n_items, seed, epoch, batch):
    """dae_seq_negatives: -1 where pos < 0, else (pos + 1 + floor(c (N - 1) / 2^32)) mod N."""
    from dae_rnn_news_recommendation_b200.user_model import negatives_from_draws
    pos = np.asarray(pos, np.int64)
    out = np.full(pos.shape, -1, np.int32)
    has = np.flatnonzero(pos >= 0)
    if has.size:
        out[has] = negatives_from_draws(pos[has], philox_first_word(has, batch, epoch, seed), n_items)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# gather + split, rownorm + split, row arg-max
# ---------------------------------------------------------------------------------------------------------------------------
def gather_split(src, rows, cols, ld_dst, ones_col):
    """dae_gather_split_bf16's hi / lo bit patterns [n_rows x ld_dst]: columns [0, cols) = src[rows], column ones_col = 1 (when
    ones_col >= cols), every other column 0."""
    src = np.asarray(src, np.float32)
    v = np.zeros((len(rows), ld_dst), np.float32)
    v[:, :cols] = src[np.asarray(rows, np.int64), :cols]
    if ones_col >= cols:
        v[:, ones_col] = 1.0
    return bf16_split(v)


def rownorm(X, norm_kind):
    """fp64 rows of X scaled by 1 / ||x|| (norm_kind 2: l2, 1: l1, 3: max, 0: none), rows of norm 0 untouched; returns
    (value, scale)."""
    X = np.asarray(X, np.float64)
    if norm_kind == 0:
        return X.copy(), np.abs(X)
    nrm = {2: lambda a: np.sqrt((a * a).sum(1)), 1: lambda a: np.abs(a).sum(1), 3: lambda a: np.abs(a).max(1)}[norm_kind](X)
    s = np.where(nrm > 0, 1.0 / np.where(nrm > 0, nrm, 1.0), 1.0)
    v = X * s[:, None]
    return v, np.abs(v)


def row_argmax(S, diag_offset, cols=None):
    """dae_row_argmax on the host: per row the first maximum over the non-NaN entries other than column r + diag_offset; -1 / -inf
    when there is none.  Returns (idx int32, val float32)."""
    S = np.asarray(S, np.float32)
    rows = S.shape[0]
    cols = S.shape[1] if cols is None else cols
    idx = np.full(rows, -1, np.int32)
    val = np.full(rows, -np.inf, np.float32)
    for r in range(rows):
        for c in range(cols):
            v = S[r, c]
            if c == r + diag_offset or np.isnan(v):
                continue
            if idx[r] < 0 or v > val[r]:
                idx[r], val[r] = c, v
    return idx, val


# ---------------------------------------------------------------------------------------------------------------------------
# GRU cell
# ---------------------------------------------------------------------------------------------------------------------------
def gru_edge_inputs(rng, n, H):
    """fp32 XP, HP [n x 3H] and h_prev [n x H] reaching the cell's edges: pre-activations from -30 to 30 (row 0 sweeps them),
    n = +-1 in fp32 (row 1), n approaching 1 (row 2), h_prev = 0 (row 3 when n > 3)."""
    f32 = np.float32
    xp = (rng.standard_normal((n, 3 * H)) * rng.choice([0.3, 3.0, 15.0], (n, 1))).astype(f32)
    hp = (rng.standard_normal((n, 3 * H)) * rng.choice([0.3, 3.0, 15.0], (n, 1))).astype(f32)
    xp[0] = np.linspace(-30, 30, 3 * H, dtype=f32)
    hp[0] = 0
    if n > 1:
        xp[1, 2 * H:] = 30.0 * np.sign(rng.standard_normal(H)).astype(f32)
    if n > 2:
        xp[2, 2 * H:] = np.arctanh(1 - 2.0 ** -(np.arange(H) % 20 + 1)).astype(f32)
        hp[2] = 0
    hprev = (rng.standard_normal((n, H)) * 2).astype(f32)
    if n > 3:
        hprev[3] = 0
    return np.clip(xp, -30, 30), np.clip(hp, -30, 30), hprev


def cell_fwd(xp, hp, h_prev, H):
    """One forward step for every row of xp [n x >= 3H] / hp [n x >= 3H] / h_prev [n x H] (None: 0).  Returns {name: (value,
    scale)} for r, z, n, h, and 'hn' (the copied h_n third, exact)."""
    xp = np.asarray(xp, np.float64)[:, :3 * H]
    hp = np.asarray(hp, np.float64)[:, :3 * H]
    hpv = np.zeros((xp.shape[0], H)) if h_prev is None else np.asarray(h_prev, np.float64)[:, :H]
    xr, xz, xn = xp[:, :H], xp[:, H:2 * H], xp[:, 2 * H:]
    hr, hz, hn = hp[:, :H], hp[:, H:2 * H], hp[:, 2 * H:]
    r, z = sigmoid(xr + hr), sigmoid(xz + hz)
    s_r = r * (1.0 - r) * (np.abs(xr) + np.abs(hr)) + r
    s_z = z * (1.0 - z) * (np.abs(xz) + np.abs(hz)) + z
    n = np.tanh(xn + r * hn)
    s_n = (1.0 - n * n) * (np.abs(xn) + np.abs(r * hn) + np.abs(hn) * s_r) + np.abs(n)
    h = (1.0 - z) * n + z * hpv
    s_h = np.abs(1.0 - z) * s_n + np.abs(n - hpv) * s_z + np.abs((1.0 - z) * n) + np.abs(z * hpv)
    return {'r': (r, s_r), 'z': (z, s_z), 'n': (n, s_n), 'h': (h, s_h), 'hn': (hn, np.zeros_like(hn))}


def cell_bwd(dh_in, carry, gates, h_prev, H):
    """One backward step from the stored gates [n x >= 4H] = [r | z | n | hn], the carry [n x H], dh_in (None: 0) and h_prev
    (None: 0).  Returns {name: (value, scale)} for dr, dz, dn, 'rdn' (dHP's n-third) and 'carry' (dh z)."""
    g = np.asarray(gates, np.float64)
    r, z, n, hn = g[:, :H], g[:, H:2 * H], g[:, 2 * H:3 * H], g[:, 3 * H:4 * H]
    c = np.asarray(carry, np.float64)[:, :H]
    di = np.zeros_like(c) if dh_in is None else np.asarray(dh_in, np.float64)[:, :H]
    hpv = np.zeros_like(c) if h_prev is None else np.asarray(h_prev, np.float64)[:, :H]
    dh, D = c + di, np.abs(c) + np.abs(di)
    dn = dh * (1.0 - z) * (1.0 - n * n)
    s_dn = D * np.abs(1.0 - z) * (1.0 + n * n)
    dz = dh * (hpv - n) * z * (1.0 - z)
    s_dz = D * (np.abs(hpv) + np.abs(n)) * z * np.abs(1.0 - z)
    dr = dn * hn * r * (1.0 - r)
    s_dr = s_dn * np.abs(hn) * r * np.abs(1.0 - r)
    return {'dr': (dr, s_dr), 'dz': (dz, s_dz), 'dn': (dn, s_dn), 'rdn': (r * dn, r * s_dn), 'carry': (dh * z, D * z)}


# ---------------------------------------------------------------------------------------------------------------------------
# ranking loss
# ---------------------------------------------------------------------------------------------------------------------------
def seq_rank_loss(h, emb, pos, neg, scale, H):
    """dae_seq_rank_loss for every position: returns (dh, dh scale, loss terms, loss-term scales); rows / terms with pos < 0 are
    exactly 0 (scale 0)."""
    h = np.asarray(h, np.float64)[:, :H]
    emb = np.asarray(emb, np.float64)[:, :H]
    pos, neg = np.asarray(pos, np.int64), np.asarray(neg, np.int64)
    has = pos >= 0
    ep = np.where(has[:, None], emb[np.where(has, pos, 0)], 0.0)
    en = np.where(has[:, None], emb[np.where(has, neg, 0)], 0.0)
    sp, sn = (h * ep).sum(1), (h * en).sum(1)
    s_x = np.abs(h * ep).sum(1) + np.abs(h * en).sum(1)
    x = sn - sp
    sg = sigmoid(x)
    sc = float(np.float32(scale))
    dh = sc * sg[:, None] * (en - ep)
    s_dh = abs(sc) * ((sg * (1.0 - sg) * s_x)[:, None] * np.abs(en - ep) + sg[:, None] * (np.abs(en) + np.abs(ep)))
    lt = np.where(has, softplus(x), 0.0)
    s_lt = np.where(has, sg * s_x + softplus(x), 0.0)
    return dh, s_dh, lt, s_lt


# ---------------------------------------------------------------------------------------------------------------------------
# GEMMs
# ---------------------------------------------------------------------------------------------------------------------------
def gemm_nt(A, B):
    """A [M x K] . B^T [K x N] in fp64 from the fp32 operands, and Sum_k |a_k b_k|."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    return A @ B.T, np.abs(A) @ np.abs(B).T
