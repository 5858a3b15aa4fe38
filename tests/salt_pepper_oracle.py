"""NumPy restatement of dae_salt_pepper_csr: the Philox draws of its device mode and the application of a draw array to a clean CSR
(what utils.salt_and_pepper_noise does with the draws it takes from the NumPy stream)."""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 on uint64 lanes: ctr = 4 arrays (broadcastable), key = 2 scalars / arrays -> the 4 output words."""
    c = [np.asarray(x, np.uint64) & M32 for x in ctr]
    c = list(np.broadcast_arrays(*c))
    k = [np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)]
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & M32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & M32]
        k = [(k[0] + np.uint64(0x9E3779B9)) & M32, (k[1] + np.uint64(0xBB67AE85)) & M32]
    return c


def philox_draws(rows, F, v, seed, epoch):
    """Device-mode draws of the global rows `rows`, packed like utils.salt_and_pepper_draws: uint32[len(rows) x v] = column |
    coin << 31.  Key (seed lo, seed hi); counter (j // 2, r, epoch lo, epoch hi); an even j takes the words (c0, c1), an odd j
    (c2, c3); column = c_a * F >> 32, coin = c_b >> 31."""
    rows = np.asarray(rows, np.uint64).reshape(-1, 1)
    pairs = np.arange((v + 1) // 2, dtype=np.uint64).reshape(1, -1)
    c = philox4x32_10((pairs, rows, np.uint64(epoch & 0xFFFFFFFF), np.uint64(epoch >> 32)), (seed & 0xFFFFFFFF, seed >> 32))
    col = np.empty((rows.shape[0], 2 * pairs.shape[1]), np.uint64)
    coin = np.empty_like(col)
    col[:, 0::2], col[:, 1::2] = (c[0] * np.uint64(F)) >> np.uint64(32), (c[2] * np.uint64(F)) >> np.uint64(32)
    coin[:, 0::2], coin[:, 1::2] = c[1] >> np.uint64(31), c[3] >> np.uint64(31)
    return (col[:, :v] | (coin[:, :v] << np.uint64(31))).astype(np.uint32)


def apply_draws_row(idx, dat, draws_row, lo, hi):
    """One row: clean (indices, values) + its draws -> the corrupted row's (indices int32, values float32), columns ascending.  The
    last draw of a column decides; a column that ends at 0 is not stored; untouched entries keep their value, explicit zeros too."""
    d = np.asarray(draws_row, np.uint32)
    cols = (d & np.uint32(0x7FFFFFFF)).astype(np.int64)
    coin = (d >> np.uint32(31)).astype(bool)
    u, first_rev = np.unique(cols[::-1], return_index=True)
    last = len(d) - 1 - first_rev
    val = np.where(coin[last], np.float32(hi), np.float32(lo)).astype(np.float32)
    keep = val != 0
    idx = np.asarray(idx, np.int64)
    untouched = ~np.isin(idx, u)
    c = np.concatenate([u[keep], idx[untouched]])
    x = np.concatenate([val[keep], np.asarray(dat, np.float32)[untouched]])
    o = np.argsort(c, kind='stable')
    return c[o].astype(np.int32), x[o]


def apply_draws(X, draws, lo, hi, rows=None):
    """Corrupted CSR arrays (indptr int64, indices int32, data float32) of the rows `rows` (default: all) of the canonical CSR X under
    draws uint32[len(rows) x v]."""
    rows = np.arange(X.shape[0]) if rows is None else np.asarray(rows)
    draws = np.asarray(draws, np.uint32).reshape(len(rows), -1)
    ind, dat, ptr = [], [], [0]
    for k, r in enumerate(rows):
        a, b = X.indptr[r], X.indptr[r + 1]
        c, x = apply_draws_row(X.indices[a:b], X.data[a:b], draws[k], lo, hi)
        ind.append(c)
        dat.append(x)
        ptr.append(ptr[-1] + len(c))
    return (np.asarray(ptr, np.int64), np.concatenate(ind).astype(np.int32) if ind else np.zeros(0, np.int32),
            np.concatenate(dat).astype(np.float32) if dat else np.zeros(0, np.float32))


def value_range(X):
    """(lo, hi) as salt_and_pepper_noise takes them: X.min() / X.max() over the whole matrix, implicit zeros included."""
    return float(X.min()), float(X.max())


def cases():
    """(name, canonical CSR, v): binary, tf-idf and negative-valued data, a full matrix (lo != 0), explicit stored zeros, empty rows,
    v = 0, v = F, F = 1, and a small F with a large v (repeated columns with opposite coins are certain)."""
    import scipy.sparse as sp
    rng = np.random.default_rng(7)

    def rand(n, F, dens, vals):
        m = sp.random(n, F, density=dens, format='csr', random_state=rng, data_rvs=vals)
        m.sort_indices()
        return m
    out = []
    out.append(('binary', rand(30, 200, 0.05, lambda k: np.ones(k)), 60))
    out.append(('tfidf', rand(30, 200, 0.05, lambda k: rng.random(k) * 0.9 + 0.05), 60))
    out.append(('negative', rand(30, 200, 0.05, lambda k: rng.random(k) * 2 - 1.5), 60))
    out.append(('full', sp.csr_matrix(rng.random((12, 40)) + 0.5), 15))
    out.append(('full_negative', sp.csr_matrix(-(rng.random((12, 40)) + 0.5)), 15))
    z = rand(25, 120, 0.08, lambda k: rng.random(k) + 0.1)
    rows = np.repeat(np.arange(z.shape[0]), np.diff(z.indptr))
    keep = ~np.isin(rows, [1, 7, 20])                     # empty rows
    data = z.data[keep].copy()
    data[::3] = 0.0                                       # explicit stored zeros
    zc = sp.csr_matrix((data, z.indices[keep], np.concatenate([[0], np.cumsum(np.bincount(rows[keep], minlength=z.shape[0]))])),
                       shape=z.shape)
    assert (zc.data == 0).sum() > 0 and zc.has_sorted_indices
    out.append(('explicit_zeros_empty_rows', zc, 30))
    out.append(('v0', rand(20, 150, 0.05, lambda k: rng.random(k) + 0.1), 0))
    out.append(('vF', rand(20, 150, 0.05, lambda k: rng.random(k) + 0.1), 150))
    out.append(('F1', sp.csr_matrix((rng.random((15, 1)) < 0.5).astype(np.float64) * 0.7), 1))
    out.append(('small_F_large_v', rand(20, 5, 0.3, lambda k: rng.random(k) + 0.1), 50))
    return out


def capacity(X, v):
    """Entries the engine's corrupted-CSR buffers hold: sum over rows of min(F, nnz_r + v)."""
    return int(np.minimum(np.diff(X.indptr) + v, X.shape[1]).sum())
