"""Host-side utilities with the reference's names and argument meaning (autoencoder/utils.py in the reference).

These are the pieces of the reference's interface that stay on the host (they are the data formats either side of the
hot path): batch slicing, the corruption functions and the Xavier bounds.  During `fit` the engine does NOT call
gen_batches / get_sparse_ind_val_shape per step -- batching happens on the device (dae_batch_prepare) -- but the
functions keep their reference behaviour so user code and the reference's tests keep working.
"""
import numpy as np
import pandas as pd
from scipy import sparse


def xavier_init(fan_in, fan_out, const=1, rng=None):
    """Uniform(-c*sqrt(6/(fan_in+fan_out)), +c*sqrt(...)) weights (reference utils.py:16-26).

    The reference draws with tf.random_uniform (TF's graph-level seed); that stream cannot be reproduced without
    TensorFlow, so this draws from NumPy (`rng` or the global RandomState) and returns a float32 ndarray.
    """
    bound = const * np.sqrt(6.0 / (fan_in + fan_out))
    r = np.random if rng is None else rng
    return r.uniform(-bound, bound, size=(fan_in, fan_out)).astype(np.float32)


def _resolve_batch_size(n_rows, batch_size):
    assert batch_size > 0.
    if batch_size < 1.:
        batch_size = max(round(n_rows * batch_size), 1)
    return int(batch_size)


def _take_rows(obj, idx):
    if isinstance(obj, (pd.DataFrame, pd.Series)):
        return obj.iloc[idx]
    return obj[idx]


def gen_batches(data, data_corrupted, batch_size, data_label=None, random=True):
    """Yield (batch, batch_corrupted[, batch_label]) tuples covering every row once (reference utils.py:29-70).

    batch_size in (0,1) is a fraction of the rows; the shuffle consumes the global NumPy RNG exactly like the
    reference (np.random.shuffle of a Python list), so seeded runs see the same batch order.
    """
    assert batch_size > 0.
    n = data.shape[0]
    assert n == data_corrupted.shape[0]
    assert type(data) == type(data_corrupted), (type(data), type(data_corrupted))
    if isinstance(data, pd.DataFrame):
        assert (data.index == data_corrupted.index).all()
    if data_label is not None:
        assert data_label.ndim == 1 or data_label.shape[1] == 1
    bs = _resolve_batch_size(n, batch_size)
    order = list(range(n))
    if random:
        np.random.shuffle(order)
    for start in range(0, n, bs):
        idx = order[start:start + bs]
        out = (_take_rows(data, idx), _take_rows(data_corrupted, idx))
        if data_label is not None:
            out = out + (_take_rows(data_label, idx),)
        yield out


def gen_batches_triplet(data, data_corrupted, batch_size, random=True):
    """Batches of the dict-of-matrices ('org','pos','neg') input of DenoisingAutoencoderTriplet
    (reference utils.py:73-91; a float batch_size >= 1 is cast to int, which the reference forgets)."""
    assert batch_size > 0.
    n = None
    for key in data:
        assert data[key].shape[0] == data_corrupted[key].shape[0]
        n = data[key].shape[0]
    bs = _resolve_batch_size(n, batch_size)
    order = list(range(n))
    if random:
        np.random.shuffle(order)
    for start in range(0, n, bs):
        idx = order[start:start + bs]
        yield [data[k][idx, :] for k in data], [data_corrupted[k][idx, :] for k in data]


def masking_noise(X, v):
    """Zero a random fraction v of the entries (stored entries for sparse input) (reference utils.py:94-115)."""
    assert 0. <= v <= 1.
    if isinstance(X, np.ndarray):
        keep = np.random.choice(a=[0, 1], size=X.shape, p=[v, 1 - v])
        return keep * X
    coo = X.tocoo(True)
    keep = np.random.rand(coo.nnz) >= v
    out = sparse.coo_matrix((coo.data[keep], (coo.row[keep], coo.col[keep])), shape=coo.shape)
    return out.tocsr()


def masking_keep_mask(X_csr, v):
    """The keep mask masking_noise would draw for a canonical CSR matrix, in CSR storage order, consuming the same
    np.random.rand(nnz) draw (CSR -> COO conversion keeps the storage order)."""
    assert 0. <= v <= 1.
    return np.random.rand(X_csr.nnz) >= v


def salt_and_pepper_noise(X, v):
    """Set v randomly chosen (with replacement) entries per row to the global min or max (reference utils.py:118-144)."""
    out = X.tolil(True) if not isinstance(X, np.ndarray) else X.copy()
    n_features = X.shape[1]
    lo, hi = X.min(), X.max()
    for i in range(X.shape[0]):
        for m in np.random.randint(0, n_features, v):
            out[i, m] = lo if np.random.random() < 0.5 else hi
    return out.tocsr() if not isinstance(X, np.ndarray) else out


def salt_and_pepper_draws(X, v):
    """The draws salt_and_pepper_noise(X, v) takes from the global NumPy stream, in its order -- per row randint(0, F, v), then v
    random() calls (as one random_sample(v): the same numbers) -- packed as uint32[rows x v] = column | (u >= 0.5) << 31, bit 31 set
    where the draw writes the maximum.  dae_salt_pepper_csr applied to them reproduces salt_and_pepper_noise(X, v) bit for bit."""
    n, F = X.shape
    assert F < (1 << 30) and v >= 0
    v = int(v)
    out = np.empty((n, v), dtype=np.uint32)
    for i in range(n):
        m = np.random.randint(0, F, v)
        u = np.random.random_sample(v)
        out[i] = m.astype(np.uint32) | ((u >= 0.5).astype(np.uint32) << np.uint32(31))
    return out


def decay_noise(X, v):
    """X * (1 - v) (reference utils.py:147-159)."""
    return X.copy() * (1. - v)


def get_sparse_ind_val_shape(sparse_m):
    """(indices[nnz,2], values[nnz], shape) of the row-sorted matrix (reference utils.py:162-180) -- the COO triple
    the reference feeds to a TF sparse placeholder.  Kept for API compatibility; the engine consumes CSR directly."""
    m = sparse.csr_matrix(sparse_m)
    m.sort_indices()
    coo = m.tocoo()
    return np.column_stack((coo.row, coo.col)), coo.data, coo.shape


def shard_batch_starts(n_rows, batch_size, world=1, rank=0):
    """Row offsets (into the epoch's shared permutation) of the batches rank `rank` of `world` trains on.

    world == 1: every batch, the last one short (reference utils.py:53).  world > 1 (data parallel): the permutation
    is identical on all ranks (same seed), rank r takes batches r, r+P, r+2P, ... and only FULL groups of P full-size
    batches are used, so every rank runs the same number of steps and the per-step all-reduce always has P contributors.
    """
    starts = list(range(0, n_rows, batch_size))
    if world <= 1:
        return starts
    full = [s for s in starts if s + batch_size <= n_rows]
    groups = len(full) // world
    return [full[g * world + rank] for g in range(groups)]
