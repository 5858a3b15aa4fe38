"""fp64 references of the training step's kernels (K1 encode, K5 encode backward, the decode loss, the optimizer), for the
kernel-level tests.  Tests only.

Every reference returns the value AND a per-element error scale, so that a kernel passes when, for every element,

    |got - want| <= c * scale + tiny

and no tensor's largest entry sets the scale of its small entries.  The scale is the magnitude the kernel's rounding acts on: the
sum of absolute terms of a contraction, the absolute values of the operands of a difference, and an input error carried through
the derivative of what follows.  `c` depends on the kernel's arithmetic:

C_FP32 = 2^-20 (16 units of fp32 rounding) for the CUDA-core kernels: a few correctly rounded operations per element, the accurate
  expf / logf / tanhf, and fp32 sums whose error stays at a few units of their sum of absolute terms for the row lengths here.

C_BF16X3 = 2^-14 for the tensor-core decode.  An operand a is carried as bf16 hi = rn(a) and lo = rn(a - hi), so
  |a - hi - lo| <= 2^-9 |a - hi| <= 2^-18 |a|.  A product of two such operands without its lo.lo term is off by at most
  3 x 2^-18 |a b| (~2^-16.4).  The fp32 accumulation of K <= 1000 products adds well under 2^-18 of the sum of absolute terms,
  the MUFU approximations (ex2 / rcp / lg2 .approx) about 2^-21 relative, and dZ leaves as a bf16 hi / lo pair: another 2^-18.
  Together that is below 2^-15; 2^-14 leaves a factor of two.  lg2.approx is accurate to 2^-22 ABSOLUTE, so row losses also get
  2^-20 per column in `tiny`.

Saturation: where g(z) of a sigmoid or tanh rounds to +-1 in fp32, the reference model (TF, fp32) computes 1 - D + 1e-16 = 1e-16
and g'(z) = 0.  The decode reference takes D = +-1 exactly there, as the fp32 model does, and D = 0 where a sigmoid leaves fp32's
normal range (z < -87); the tests keep pre-activations away from the few units around those thresholds.
"""
import numpy as np
import scipy.sparse as sp

from user_gru_oracle import adam_tf

C_FP32 = 2.0 ** -20
C_BF16X3 = 2.0 ** -14
EPS = 1e-16

ACTS = ('none', 'sigmoid', 'tanh')
LOSSES = ('cross_entropy', 'mean_squared', 'cosine_proximity')


# ---------------------------------------------------------------------------------------------------------------------------
# activations: value, derivative through y = g(x), and the derivative of that with respect to y
# ---------------------------------------------------------------------------------------------------------------------------
def act(name, x):
    x = np.asarray(x, np.float64)
    if name == 'sigmoid':
        return 0.5 * (1.0 + np.tanh(0.5 * x))    # overflow-free 1 / (1 + e^-x)
    if name == 'tanh':
        return np.tanh(x)
    return x.copy()


def act_grad(name, y):
    if name == 'sigmoid':
        return y * (1.0 - y)
    if name == 'tanh':
        return 1.0 - y * y
    return np.ones_like(y)


def act_grad2(name, y):
    """d g'(x) / dy at y = g(x)"""
    if name == 'sigmoid':
        return 1.0 - 2.0 * y
    if name == 'tanh':
        return -2.0 * y
    return np.zeros_like(y)


def saturate(name, d):
    """D as the fp32 kernels see it: +-1 exactly where g(z) rounds to +-1 in fp32, and 0 where a sigmoid underflows fp32's normal
    range (1 / (1 + e^-z) with e^-z = inf).  Returns (D, mask of the saturated entries)."""
    sat = np.zeros(d.shape, bool)
    if name in ('sigmoid', 'tanh'):
        sat = np.abs(d.astype(np.float32)) == 1.0
        if name == 'sigmoid':
            under = np.abs(d) < 2.0 ** -126
            d = np.where(under, 0.0, d)
            sat |= under
        d = np.where(sat & (d != 0.0), np.sign(d), d)
    return d, sat


# ---------------------------------------------------------------------------------------------------------------------------
# CSR helpers
# ---------------------------------------------------------------------------------------------------------------------------
def csr_rows(m, rows=None):
    """fp64 scipy CSR of the batch rows (rows == None: all rows in order)."""
    m = sp.csr_matrix(m, dtype=np.float64)
    return m if rows is None else m[np.asarray(rows)]


def boundary_columns(F):
    """0, F - 1, and both sides of every 16-column boundary (so of every 64- and 128-column boundary too)."""
    cols = {0, F - 1}
    for b in range(16, F, 16):
        cols.update((b - 1, b))
    return np.array(sorted(c for c in cols if 0 <= c < F), np.int64)


def edge_csr(n, F, mean_nnz=20, kind='tfidf', seed=0, long_row=True, planted=True):
    """A canonical CSR batch (sorted columns, no repeats) that reaches the edges of the step's kernels:
    - the boundary columns (boundary_columns) spread over the rows, so every one of them is stored somewhere;
    - row 1: a fully stored 64-column half tile (columns 64..127, or 0..63 when F < 128);
    - row 2: five entries inside one 16-column chunk;
    - row 3: empty; row 4 (if F > 600 and long_row): more than 512 entries;
    - a planted column stored in up to 150 rows (more than two chunks of 64 bucketed entries).
    values: 1.0 (kind='binary') or uniform in [0.05, 1.05) (tf-idf like)."""
    rng = np.random.default_rng(seed)
    sets = [set() for _ in range(n)]
    for i in range(n):
        if i == 3:
            continue
        k = int(min(F, rng.poisson(mean_nnz)))
        sets[i].update(rng.choice(F, size=k, replace=False).tolist())
    bc = boundary_columns(F)
    for j, c in enumerate(bc):
        r = j % n
        sets[(r + 1) % n if r == 3 else r].add(int(c))
    if n > 1:
        lo = 64 if F >= 128 else 0
        sets[1].update(range(lo, min(F, lo + 64)))
    if n > 2:
        base = 16 if F >= 32 else 0
        sets[2].update(range(base, min(F, base + 5)))
    if n > 4 and long_row and F > 600:
        sets[4].update(rng.choice(F, size=min(F, 600), replace=False).tolist())
    if planted and F > 4:
        pc = F // 2 + 3 if F > 8 else F - 2
        for i in range(min(n, 150)):
            if i != 3:
                sets[i].add(pc)
    if n > 3:
        sets[3].clear()
    indptr = np.zeros(n + 1, np.int64)
    indices, values = [], []
    for i, s in enumerate(sets):
        c = np.array(sorted(s), np.int32)
        indices.append(c)
        values.append(np.ones(len(c)) if kind == 'binary' else rng.random(len(c)) + 0.05)
        indptr[i + 1] = indptr[i] + len(c)
    return sp.csr_matrix((np.concatenate(values).astype(np.float32), np.concatenate(indices), indptr), shape=(n, F))


def mask_values(m, frac, seed=1, masked_rows=(5,)):
    """The corrupted copy: same structure, a random `frac` of the values set to 0, and every value of `masked_rows` set to 0."""
    rng = np.random.default_rng(seed)
    out = m.copy()
    keep = rng.random(m.nnz) >= frac
    for r in masked_rows:
        if r < m.shape[0]:
            keep[m.indptr[r]:m.indptr[r + 1]] = False
    out.data = (out.data * keep).astype(np.float32)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# K1: E = f(in_scale X_c W + bh) - f(bh)
# ---------------------------------------------------------------------------------------------------------------------------
def encode_fwd(Xc, W, bh, act_name, in_scale=1.0):
    """Xc: the corrupted batch rows (scipy sparse or dense).  Returns E, scale and the pre-activation A."""
    W = np.asarray(W, np.float64)
    bh = np.asarray(bh, np.float64)
    X = csr_rows(Xc) * float(np.float32(in_scale))
    A = np.asarray(X @ W) + bh
    fa, fb = act(act_name, A), act(act_name, bh)
    absX = abs(X)
    scale = act_grad(act_name, fa) * (np.asarray(absX @ np.abs(W)) + np.abs(bh)) + np.abs(fa) + np.abs(fb)
    return fa - fb, scale, A


# ---------------------------------------------------------------------------------------------------------------------------
# K5: dA = (dE + dE_add) f'(A), dbh, dW += X_c^T dA
# ---------------------------------------------------------------------------------------------------------------------------
def encode_bwd(Xc, E, dE, dE_add, bh, act_name, in_scale=1.0, dW0=None):
    """E is the forward's fp32 output: f(A) is recovered as E + f(bh), as the kernels do.  Returns {name: (value, scale)} for dA,
    dbh and dW (dW = dW0 + X_c^T dA)."""
    E = np.asarray(E, np.float64)
    dE = np.asarray(dE, np.float64)
    dEa = np.zeros_like(dE) if dE_add is None else np.asarray(dE_add, np.float64)
    bh = np.asarray(bh, np.float64)
    X = csr_rows(Xc) * float(np.float32(in_scale))
    fb = act(act_name, bh)
    y = E + fb
    g, g2 = act_grad(act_name, y), act_grad2(act_name, y)
    de, de_mag = dE + dEa, np.abs(dE) + np.abs(dEa)
    dA = de * g
    s_dA = de_mag * (np.abs(g) + np.abs(g2) * (np.abs(E) + np.abs(fb)))
    gb, gb2 = act_grad(act_name, fb), act_grad2(act_name, fb)
    dbh = dA.sum(0) - gb * de.sum(0)
    s_dbh = s_dA.sum(0) + (np.abs(gb) + np.abs(gb2) * np.abs(fb)) * de_mag.sum(0)
    dW0 = np.zeros((X.shape[1], E.shape[1])) if dW0 is None else np.asarray(dW0, np.float64)
    dW = dW0 + np.asarray(X.T @ dA)
    s_dW = np.abs(dW0) + np.asarray(abs(X).T @ s_dA)
    return {'dA': (dA, s_dA), 'dbh': (dbh, s_dbh), 'dW': (dW, s_dW)}


# ---------------------------------------------------------------------------------------------------------------------------
# decode loss: D = g(z), row loss against the clean rows, dZ = w / (sum_w + 1e-16) * dl/dD * g'   (triplet_loss_utils.py:262-275)
# ---------------------------------------------------------------------------------------------------------------------------
def decode_loss(z, X, weight, sum_w, act_name, loss, zs=None, tanh_abs=True):
    """z: fp64 pre-activations (E W^T + bv) [B x F]; X: the clean target rows (scipy sparse or dense); zs: the error scale of z (the
    kernel's input error: sum_k |E_ik W_jk| + |bv_j| + |z_ij| for the fused decode, |Z| + |bv| for the unfused one).
    Returns (dZ, dZ scale, per-element loss terms, their scale) -- a row loss is the sum of its terms, its scale the sum of theirs;
    for the cosine loss the terms are laid out so that their row sum is the loss.  tanh_abs: D = tanh carries an ABSOLUTE error of a
    few units of rounding (1 - 2 / (1 + e^2z) cancels near 0), so D's error scale gets 1 added for tanh."""
    z = np.asarray(z, np.float64)
    X = np.asarray(X.todense() if sp.issparse(X) else X, np.float64)
    zs = np.zeros_like(z) if zs is None else np.asarray(zs, np.float64)
    w = np.ones(z.shape[0]) if weight is None else np.asarray(weight, np.float64)
    sc = (w / (float(sum_w) + EPS))[:, None]
    d, sat = saturate(act_name, act(act_name, z))
    g, g2 = act_grad(act_name, d), act_grad2(act_name, d)
    dd = np.where(sat, 0.0, np.abs(d)) + np.abs(g) * zs        # error scale of D: its own rounding + the input's, through g'
    if act_name == 'tanh' and tanh_abs:
        dd = dd + np.where(sat, 0.0, 1.0)
    if loss == 'cross_entropy':
        a, b = d + EPS, (1.0 - d) + EPS
        with np.errstate(divide='ignore', invalid='ignore'):
            lt = -(X * np.log(a) + (1.0 - X) * np.log(b))
            dl = -X / a + (1.0 - X) / b
            dl2 = X / a ** 2 + (1.0 - X) / b ** 2
        dZ = sc * dl * g
        ddz = sc * (dl2 * g + dl * g2)
        s_dZ = np.abs(dZ) + np.abs(ddz) * dd
        s_l = np.abs(X * np.log(a)) + np.abs((1.0 - X) * np.log(b)) + np.abs(dl) * dd
        return dZ, s_dZ, lt, s_l
    if loss == 'mean_squared':
        e = X - d
        lt = e * e
        dZ = sc * (-2.0 * e) * g
        ddz = sc * 2.0 * (g - e * g2)
        s_dZ = np.abs(dZ) + np.abs(ddz) * dd
        s_l = lt + 2.0 * np.abs(e) * dd
        return dZ, s_dZ, lt, s_l
    assert loss == 'cosine_proximity', loss
    # tf.nn.l2_normalize: v * rsqrt(max(sum v^2, 1e-12)); the clamped branch of max() has zero gradient
    sxx = (X * X).sum(1, keepdims=True)
    sdd = (d * d).sum(1, keepdims=True)
    sxd = (X * d).sum(1, keepdims=True)
    sxd_abs = np.abs(X * d).sum(1, keepdims=True)
    rx = 1.0 / np.sqrt(np.maximum(sxx, 1e-12))
    rd = 1.0 / np.sqrt(np.maximum(sdd, 1e-12))
    rd3 = np.where(sdd >= 1e-12, rd ** 3, 0.0)
    rd5 = np.where(sdd >= 1e-12, rd ** 5, 0.0)
    dl = -rx * (X * rd - sxd * rd3 * d)
    dZ = sc * dl * g
    xdd = (np.abs(X) * dd).sum(1, keepdims=True)              # how far the row sums move with D's error
    ddd = (np.abs(d) * dd).sum(1, keepdims=True)
    br = np.abs(X) * rd + sxd_abs * rd3 * np.abs(d)           # |bracket| with every term taken by magnitude
    dbr = rd3 * (np.abs(X) * ddd + sxd_abs * dd + np.abs(d) * xdd) + 3.0 * rd5 * sxd_abs * np.abs(d) * ddd
    s_dZ = np.abs(sc) * rx * ((np.abs(g) + np.abs(g2) * dd) * br + np.abs(g) * dbr)
    # the loss -sxd rx rd as per-element terms: -x_j d_j rx rd (their row sum)
    lt = -X * d * rx * rd
    s_l = rx * rd * (np.abs(X * d) + np.abs(X) * dd + np.abs(sxd) * rd * rd * np.abs(d) * dd)
    return dZ, s_dZ, lt, s_l


def fused_decode_z(E, W, bv):
    """z = E W^T + bv in fp64 from the fp32 operands, and its error scale for the tensor-core decode."""
    E = np.asarray(E, np.float64)
    W = np.asarray(W, np.float64)
    bv = np.asarray(bv, np.float64)
    z = E @ W.T + bv
    return z, np.abs(E) @ np.abs(W).T + np.abs(bv) + np.abs(z)


# ---------------------------------------------------------------------------------------------------------------------------
# optimizer: TF-1.12 rules (autoencoder.py:451-472)
# ---------------------------------------------------------------------------------------------------------------------------
def optimizer_steps(opt, theta, grads, lr, momentum=0.5, grad_scale=1.0, slot1=None, slot2=None, t0=1, fp32_betas=True):
    """Applies the rule once per gradient in `grads` (t = t0, t0 + 1, ...).  Returns (theta, slot1, slot2, scale of theta).
    The scale sums, over the steps, |theta| and the magnitude of the update times the number of steps its slot has accumulated.
    fp32_betas: Adam's moment decay uses beta1 = fp32(0.9) and beta2 = fp32(0.999) (1 - fp32(0.999) is 1.3e-5 away from 0.001),
    as the kernel does; False: the decimal constants of user_gru_oracle.adam_tf (and of oracle/dae_oracle.py)."""
    p = np.asarray(theta, np.float64).copy()
    s1 = np.zeros_like(p) if slot1 is None else np.asarray(slot1, np.float64).copy()
    s2 = np.zeros_like(p) if slot2 is None else np.asarray(slot2, np.float64).copy()
    scale = np.abs(p)
    m_mag = np.abs(s1)
    for k, g in enumerate(grads):
        g = np.asarray(g, np.float64) * float(np.float32(grad_scale))
        t = t0 + k
        if opt == 'gradient_descent':
            upd = lr * g
            p -= upd
            mag = np.abs(upd)
        elif opt == 'ada_grad':       # accum += g^2 ; var -= lr * g / sqrt(accum)
            s1 += g * g
            upd = lr * g / np.sqrt(s1)
            p -= upd
            mag = np.abs(upd)
        elif opt == 'momentum':       # accum = mu accum + g ; var -= lr accum
            s1[:] = momentum * s1 + g
            m_mag = abs(momentum) * m_mag + np.abs(g)
            p -= lr * s1
            mag = abs(lr) * m_mag
        elif opt == 'adam' and not fp32_betas:
            adam_tf(p, g, s1, s2, t, lr)
            m_mag = 0.9 * m_mag + 0.1 * np.abs(g)
            mag = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) * m_mag / (np.sqrt(s2) + 1e-8)
        elif opt == 'adam':           # beta1, beta2 and eps as the fp32 constants the kernel (and TF's fp32 graph) multiplies by
            b1, b2, eps = float(np.float32(0.9)), float(np.float32(0.999)), float(np.float32(1e-8))
            s1[:] = b1 * s1 + (1.0 - b1) * g
            s2[:] = b2 * s2 + (1.0 - b2) * g * g
            p -= lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) * s1 / (np.sqrt(s2) + eps)
            m_mag = 0.9 * m_mag + 0.1 * np.abs(g)
            mag = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) * m_mag / (np.sqrt(s2) + 1e-8)
        else:
            raise AssertionError(opt)
        scale = scale + np.abs(p) + (k + 1) * mag
    return p, s1, s2, scale


def bf16_split(x):
    """bf16 hi = rn(x), lo = rn(x - hi), as uint16 bit patterns (x: float32 array)."""
    x = np.asarray(x, np.float32)

    def rn(v):
        b = v.astype(np.float32).view(np.uint32).astype(np.uint64)
        r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
        nan = np.isnan(v)
        return np.where(nan, np.uint16(0x7FC0), r)

    hi = rn(x)
    hi_f = (hi.astype(np.uint32) << 16).view(np.float32)
    lo = rn((x - hi_f).astype(np.float32))
    return hi, lo
