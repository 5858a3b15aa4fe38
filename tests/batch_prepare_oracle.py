"""Exact NumPy references of the batch preparation (dae_batch_prepare[_next][_blocked], include/dae_sm100.h) and of the Philox mode
of the masking noise (dae_mask_values).  No torch: every output is computed in integers or fp64 and rounded once where the kernel
rounds once, so the GPU tests compare bit for bit.

Label classes follow the reference's tf.equal: two rows share a class iff their labels compare equal.  So -0.0 and +0.0 are one
class, and a NaN label equals nothing, itself included: each NaN row is a class of one.  The kernels order the batch by one total
order key -- NaN after every other label (+inf included), -0.0 folded into +0.0 -- and then by row id."""
import numpy as np

from salt_pepper_oracle import philox4x32_10

STRATEGY_NONE, STRATEGY_BATCH_ALL, STRATEGY_BATCH_HARD = 0, 1, 2
STAT_SLOTS, STAT_SUM_W, STAT_N_VALID = 16, 5, 6
M32 = np.uint64(0xFFFFFFFF)


def batch_rows(perm, offset, B):
    """perm[offset : offset + B] as int64 (perm None: the identity)."""
    if perm is None:
        return np.arange(offset, offset + B, dtype=np.int64)
    return np.asarray(perm[offset:offset + B], np.int64)


def class_order(lab, rows):
    """The kernels' order of a batch: ascending (class key, row id), NaN labels last in row-id order, -0.0 and +0.0 one key."""
    lab = np.asarray(lab, np.float32)
    nan = np.isnan(lab)
    key = np.where(nan, np.float32(0.0), lab) + np.float32(0.0)     # -0.0 + 0.0 = +0.0
    return np.lexsort((rows, key, nan))


def segments(lab_sorted):
    """[seg_lo, seg_hi) of every row of a batch in class order: the rows whose label compares equal to its own (itself included)."""
    lab = np.asarray(lab_sorted, np.float32)
    B = lab.shape[0]
    nn = int(np.count_nonzero(~np.isnan(lab)))
    assert not np.isnan(lab[:nn]).any(), 'NaN labels must come last'
    lo, hi = np.arange(B, dtype=np.int64), np.arange(1, B + 1, dtype=np.int64)     # NaN rows: [i, i + 1)
    lo[:nn] = np.searchsorted(lab[:nn], lab[:nn], side='left')
    hi[:nn] = np.searchsorted(lab[:nn], lab[:nn], side='right')
    return lo.astype(np.int32), hi.astype(np.int32)


def closed_form(lo, hi, B):
    """fp64 closed forms of the B^3 mask reductions: w_i = 2(n-1)(B-n) + sum_{c != c_i} n_c(n_c-1), N_valid = sum_c n_c(n_c-1)(B-n_c),
    with n the size of row i's class.  Every term is an integer below 2^53, so the fp64 values are exact."""
    n = (np.asarray(hi, np.int64) - np.asarray(lo, np.int64)).astype(np.float64)
    T = float(np.sum(n - 1.0))
    NV = float(np.sum((n - 1.0) * (B - n)))
    w = 2.0 * (n - 1.0) * (B - n) + T - n * (n - 1.0)
    return w, NV


def prepare(perm, offset, B, labels_all, strategy):
    """What dae_batch_prepare writes for the batch perm[offset : offset + B]: (rows int32, labels float32, seg_lo int32, seg_hi int32,
    weights float32, stats float64[16]).  The labels are labels_all[rows], so each keeps its bits (-0.0 stays -0.0, NaN payloads
    stay).  strategy none keeps the permutation order, labels 0, one segment [0, B), w = 1 and SUM_W = B."""
    rows = batch_rows(perm, offset, B)
    stats = np.zeros(STAT_SLOTS, np.float64)
    if strategy == STRATEGY_NONE:
        stats[STAT_SUM_W] = float(B)
        return (rows.astype(np.int32), np.zeros(B, np.float32), np.zeros(B, np.int32), np.full(B, B, np.int32),
                np.ones(B, np.float32), stats)
    lab = np.asarray(labels_all, np.float32)[rows]
    o = class_order(lab, rows)
    rows, lab = rows[o], lab[o]
    lo, hi = segments(lab)
    w, NV = closed_form(lo, hi, B)
    if strategy == STRATEGY_BATCH_ALL:
        w = w.astype(np.float32)
        stats[STAT_SUM_W], stats[STAT_N_VALID] = 3.0 * NV, NV
    else:
        w = np.zeros(B, np.float32)             # batch_hard: filled by the miner
    return rows.astype(np.int32), lab, lo, hi, w, stats


def mask_uniforms(nnz, seed, epoch):
    """The Philox mode's draw of every entry: quad q = p // 4 runs Philox4x32-10 on counter (q, q >> 32, epoch, epoch >> 32) under key
    (seed, seed >> 32); entry p takes word p % 4, and u = (word >> 8) * 2^-24, exact in fp32 and fp64."""
    nq = (int(nnz) + 3) // 4
    q = np.arange(nq, dtype=np.uint64)
    e = np.uint64(int(epoch))
    c = philox4x32_10((q & M32, q >> np.uint64(32), e & M32, e >> np.uint64(32)), (int(seed) & 0xFFFFFFFF, int(seed) >> 32))
    words = np.stack(c, axis=1).reshape(-1)[:nnz]
    return (words >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def mask_values(values, keep, frac, seed=0, epoch=0):
    """dae_mask_values: entry p is kept iff keep[p] != 0 (host mask), or else iff u_p >= corr_frac (utils.masking_noise's
    rand(nnz) >= v); a dropped entry becomes +0.0, a kept one keeps its bits."""
    values = np.asarray(values, np.float32)
    if keep is not None:
        k = np.asarray(keep, np.uint8) != 0
    else:
        k = mask_uniforms(values.shape[0], seed, epoch) >= float(np.float32(frac))
    return np.where(k, values, np.float32(0.0)).astype(np.float32)


LABEL_KINDS = ('one', 'distinct', 'c4', 'c300', 'negf', 'ends', 'zeros', 'inf', 'nan1', 'nanmany', 'nanall', 'block')


def batch_labels(B, kind, seed=0):
    """float32[B] labels of one batch, in batch (permutation) order:
    one / distinct / c4 / c300 -- 1, B, 4 and 300 classes;  negf -- negative and fractional labels;
    ends -- singleton classes at the first and the last sorted position;  zeros -- -0.0 and +0.0 mixed, beside +-1;
    inf -- +-inf beside 4 classes;  nan1 / nanmany / nanall -- one NaN, a sixth NaN (with NaN payloads, +-inf and +-0.0), all NaN;
    block -- a class whose sorted segment spans the last 4096-row block boundary below B (the middle when B <= 4096)."""
    rng = np.random.default_rng(seed)
    if kind == 'one':
        lab = np.full(B, 3.0, np.float32)
    elif kind == 'distinct':
        lab = rng.permutation(B).astype(np.float32) * np.float32(0.5) - np.float32(B // 4)
    elif kind == 'c4':
        lab = rng.integers(0, 4, B).astype(np.float32)
    elif kind == 'c300':
        lab = rng.integers(0, 300, B).astype(np.float32)
    elif kind == 'negf':
        lab = (-rng.integers(0, 7, B) * 0.37).astype(np.float32)
    elif kind == 'ends':
        lab = rng.integers(1, 5, B).astype(np.float32)
        i = rng.permutation(B)[:2]
        lab[i[0]] = -5.0
        lab[i[-1]] = 99.0                # B = 1: one row, its own class
    elif kind == 'zeros':
        lab = rng.choice(np.array([-0.0, 0.0, 1.0, -1.0], np.float32), B)
    elif kind == 'inf':
        lab = rng.choice(np.array([-np.inf, np.inf, 0.0, 1.0, 2.0, 3.0], np.float32), B)
    elif kind in ('nan1', 'nanmany', 'nanall'):
        lab = rng.choice(np.array([-np.inf, np.inf, -0.0, 0.0, 1.0, 2.0, -3.5], np.float32), B)
        nan = np.zeros(B, bool)
        nan[rng.permutation(B)[:{'nan1': 1, 'nanmany': max(1, B // 6), 'nanall': B}[kind]]] = True
        payload = (np.uint32(0x7fc00000) | rng.integers(0, 1 << 22, B).astype(np.uint32)) | \
            (rng.integers(0, 2, B).astype(np.uint32) << np.uint32(31))        # quiet NaNs of either sign, any payload
        lab[nan] = payload[nan].view(np.float32)
    elif kind == 'block':
        edge = 4096 * ((B - 1) // 4096) if B > 4096 else B // 2
        n1 = max(0, edge - 100)
        n2 = min(B - n1, 200)
        lab = np.concatenate([np.full(n1, 1.0), np.full(n2, 2.0), np.full(B - n1 - n2, 3.0)]).astype(np.float32)
        lab = lab[rng.permutation(B)]
    else:
        raise AssertionError(kind)
    return lab.astype(np.float32)


def scatter_labels(n_all, perm, offset, lab_batch):
    """labels_all[n_all] whose batch perm[offset : offset + B] reads lab_batch; every other row gets a NaN, so a kernel that reads a
    label outside its batch is seen."""
    labels_all = np.full(n_all, np.nan, np.float32)
    labels_all[batch_rows(perm, offset, lab_batch.shape[0])] = lab_batch
    return labels_all
