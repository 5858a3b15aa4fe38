"""Shared helpers for the parity tests (seeded inputs, tolerances)."""
import numpy as np
import scipy.sparse as sp

REL_TOL = 1e-4  # north_star: embeddings and per-step losses within 1e-4 relative of the fp32 oracle


def rel_err(a, b):
    """NORM-wise relative error: max|a - b| / max|b| (the tensor's largest entry sets the scale)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-30))


def elem_err(a, b, floor=0.1):
    """Element-wise relative error: max_i |a_i - b_i| / max(|b_i|, floor * max|b|) -- every entry is compared with its OWN magnitude;
    entries below `floor` x the tensor's scale (results of cancellation) are compared with that floor instead."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    den = np.maximum(np.abs(b), floor * (np.max(np.abs(b)) + 1e-30))
    return float(np.max(np.abs(a - b) / den))


def random_csr(n, F, nnz_per_row, kind='binary', seed=0):
    rng = np.random.default_rng(seed)
    rows, cols, vals = [], [], []
    for i in range(n):
        k = int(np.clip(rng.poisson(nnz_per_row), 0 if i % 7 == 3 else 1, F))  # some rows empty
        c = np.sort(rng.choice(F, size=k, replace=False))
        rows.append(np.full(k, i))
        cols.append(c)
        vals.append(np.ones(k) if kind == 'binary' else rng.random(k) + 0.05)
    m = sp.csr_matrix((np.concatenate(vals).astype(np.float32), (np.concatenate(rows), np.concatenate(cols))), shape=(n, F))
    m.sort_indices()
    return m


def mask_csr(m, frac, seed=1):
    """same structure, a random `frac` of the values zeroed (what masking noise does)"""
    rng = np.random.default_rng(seed)
    keep = rng.random(m.nnz) >= frac
    out = m.copy()
    out.data = (out.data * keep).astype(np.float32)
    return out, keep


def xavier(F, H, seed=0):
    b = np.sqrt(6.0 / (F + H))
    return np.random.default_rng(seed).uniform(-b, b, (F, H)).astype(np.float32)


class _CAI:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {'data': (int(ptr), False), 'shape': tuple(shape), 'typestr': typestr, 'version': 3}


def device_copy(ptr, shape, typestr, device='cuda:0'):
    """A torch copy (on the device) of the buffer of the given shape and NumPy typestr at the raw device pointer ptr."""
    import torch
    return torch.as_tensor(_CAI(ptr, shape, typestr), device=device).clone()


def snap(ptr, rows, ld, kind='f4'):
    """A copy of the device buffer [rows x ld] at ptr (fp32 'f4' or bf16 bits 'u2') as a NumPy array."""
    import torch
    if ptr is None or rows <= 0:
        return None
    t = device_copy(ptr, (rows, ld), '<f4' if kind == 'f4' else '<i2')
    torch.cuda.synchronize()
    a = t.cpu().numpy()
    return a if kind == 'f4' else a.view(np.uint16)


def snap_vec(ptr, n, typestr):
    import torch
    t = device_copy(ptr, (n,), typestr)
    torch.cuda.synchronize()
    return t.cpu().numpy()


def pair_value(hi, lo):
    """fp64 value hi + lo of two bf16 bit arrays (uint16)."""
    f = lambda b: (np.asarray(b, np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return f(hi) + f(lo)


def load_uci_c1():
    """BASELINE.json configs[0] data (tests/golden/uci_c1.npz, written by tools/make_uci_fixture.py from the UCI corpus with the
    CLI's own preparation): binary CSR train 8000 x 10000 / validate 2000 x 10000, raw counts, category + story labels."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'uci_c1.npz'))
    out = {}
    for split in ('train', 'validate'):
        shape = tuple(int(v) for v in z[split + '_shape'])
        ind, ptr = z[split + '_indices'].astype(np.int32), z[split + '_indptr'].astype(np.int64)
        out[split] = sp.csr_matrix((np.ones(len(ind), dtype=np.float32), ind, ptr), shape=shape)
        out[split + '_counts'] = sp.csr_matrix((z[split + '_counts'].astype(np.float32), ind, ptr), shape=shape)
        for lab in ('category_publish_name', 'story'):
            out['%s_label_%s' % (split, lab)] = z['%s_label_%s' % (split, lab)]
    return out
