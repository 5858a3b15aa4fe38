"""float32 restatements of the bag-of-words profile kernels (dae_csr_profiles, dae_csr_impression_metrics), in their exact order.

Every elementwise NumPy float32 operation is IEEE-rounded and never fused, and np.add.accumulate sums strictly left to right, so
these loops give the kernels' bits: P[u, f] from +0, one rounded product w.x per read in increasing article order; the L2 norm
from the rounded squares in increasing column order; a pair's score from the rounded products over the shared columns in
increasing column order."""
import numpy as np
import scipy.sparse as sp

F32 = np.float32


def _seq_sum(terms):
    """the fp32 sum from +0 of `terms`, left to right"""
    return np.add.accumulate(np.concatenate([np.zeros(1, F32), np.asarray(terms, F32)]), dtype=F32)[-1]


def profiles(w, x, normalise=False):
    """w: canonical CSR [U, N] fp32 (the normalised weights), x: canonical CSR [N, F] fp32 -> canonical CSR [U, F] fp32 holding
    the union of the read rows' columns (explicit zeros included)."""
    indptr, indices, data = [0], [], []
    for u in range(w.shape[0]):
        reads = w.indices[w.indptr[u]:w.indptr[u + 1]]
        weights = w.data[w.indptr[u]:w.indptr[u + 1]].astype(F32)
        cols = np.unique(np.concatenate([x.indices[x.indptr[a]:x.indptr[a + 1]] for a in reads] + [np.zeros(0, np.int32)]))
        acc = np.zeros(cols.size, F32)
        for a, wv in zip(reads, weights):
            c, v = x.indices[x.indptr[a]:x.indptr[a + 1]], x.data[x.indptr[a]:x.indptr[a + 1]].astype(F32)
            pos = np.searchsorted(cols, c)
            acc[pos] = acc[pos] + F32(wv) * v
        if normalise and cols.size:
            n2 = _seq_sum(acc * acc)
            if n2 != 0:
                acc = acc / np.sqrt(F32(n2))
        indptr.append(indptr[-1] + cols.size)
        indices.append(cols.astype(np.int32))
        data.append(acc.astype(F32))
    out = sp.csr_matrix((np.concatenate(data + [np.zeros(0, F32)]), np.concatenate(indices + [np.zeros(0, np.int32)]),
                         np.asarray(indptr, np.int64)), shape=(w.shape[0], x.shape[1]))
    out.has_sorted_indices = True
    return out


def pair_score(q, i, x, a, cosine=False):
    """the score of query row i of CSR q against row a of CSR x (both canonical fp32)"""
    qc, qv = q.indices[q.indptr[i]:q.indptr[i + 1]], q.data[q.indptr[i]:q.indptr[i + 1]].astype(F32)
    xc, xv = x.indices[x.indptr[a]:x.indptr[a + 1]], x.data[x.indptr[a]:x.indptr[a + 1]].astype(F32)
    _, qi, xi = np.intersect1d(qc, xc, assume_unique=True, return_indices=True)
    dot = _seq_sum(qv[qi] * xv[xi])   # intersect1d returns the shared columns increasing
    if not cosine:
        return F32(dot)
    qq, ee = _seq_sum(qv * qv), _seq_sum(xv * xv)
    if qq == 0 or ee == 0:
        return F32(0)
    return F32(dot / (np.sqrt(F32(qq)) * np.sqrt(F32(ee))))


def impression_scores(q, x, indptr, items, cosine=False):
    """scores [nnz] of every shown article of every impression (query row i for impression i)"""
    out = np.zeros(len(items), F32)
    for i in range(len(indptr) - 1):
        for k in range(indptr[i], indptr[i + 1]):
            out[k] = pair_score(q, i, x, items[k], cosine)
    return out


def impression_metrics(scores, indptr, clicked):
    """(AUC, MRR, nDCG@5, nDCG@10) per impression from fp32 scores, the kernels' rank rule: rank_j = #{s_k > s_j} + #{k < j:
    s_k = s_j}; NaN x 4 without a click or without a non-click."""
    out = np.full((len(indptr) - 1, 4), np.nan)
    for i in range(len(indptr) - 1):
        s, c = scores[indptr[i]:indptr[i + 1]], clicked[indptr[i]:indptr[i + 1]] != 0
        nc, nn = int(c.sum()), int((~c).sum())
        if nc == 0 or nn == 0:
            continue
        auc2, rr, g5, g10 = 0, 0.0, 0.0, 0.0
        for j in np.flatnonzero(c):
            rank = int((s > s[j]).sum() + (s[:j] == s[j]).sum())
            auc2 += 2 * int((s[~c] < s[j]).sum()) + int((s[~c] == s[j]).sum())
            rr += 1.0 / (rank + 1)
            if rank < 10:
                g10 += 1.0 / np.log2(rank + 2)
                if rank < 5:
                    g5 += 1.0 / np.log2(rank + 2)
        i5 = sum(1.0 / np.log2(r + 2) for r in range(min(nc, 5)))
        i10 = sum(1.0 / np.log2(r + 2) for r in range(min(nc, 10)))
        out[i] = (auc2 / (2.0 * nc * nn), rr / nc, g5 / i5, g10 / i10)
    return out
