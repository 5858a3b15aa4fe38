"""NumPy restatements of the user encoders' deterministic mode (DESIGN 4.21): the fixed-order sum of the per-position loss slots
(dae_loss_slots_sum), the ordered article gradient (dae_ordered_rows) in float32, and the per-position loss terms in fp64."""
import numpy as np

from impression_softmax_oracle import negative_sets

SLOT_SUM_THREADS = 256   # dae_loss_slots_sum's partials


def slot_sum(slots, out=0.0):
    """out + the sum of slots in dae_loss_slots_sum's order: partial t = slots t, t + 256, ... from +0 in index order, then the
    partials in order from +0, then added to out.  Python floats are IEEE doubles, so each + rounds as the kernel's does."""
    slots = [float(x) for x in np.asarray(slots, np.float64)]
    total = 0.0
    for t in range(SLOT_SUM_THREADS):
        s = 0.0
        for x in slots[t::SLOT_SUM_THREADS]:
            s += x
        total += s
    return float(out) + total


def slot_sum_bound(slots):
    """A bound on |slot_sum - exact sum|: at most n + 256 roundings of partial sums no larger than sum |x|, each off by half an ulp."""
    a = np.abs(np.asarray(slots, np.float64))
    return (a.size + SLOT_SUM_THREADS) * np.finfo(np.float64).eps * float(a.sum())


def ordered_rows(a_slot, a_row, a_coef, src_a, b_slot, src_b, n_slots):
    """dae_ordered_rows in float32: per slot t, the terms with slot t in term order -- the triples (a_slot, a_row, a_coef) over
    src_a first, then (b_slot[p], p, 1) over src_b -- as acc = fl(acc + fl(c * row)) from +0.  Slots < 0 add nothing."""
    cols = (src_a if src_a is not None and len(src_a) else src_b).shape[1]
    out = np.zeros((n_slots, cols), np.float32)
    terms = [(int(s), np.float32(c), src_a[int(r)]) for s, r, c in zip(a_slot, a_row, a_coef) if s >= 0]   # row: any value at -1
    terms += [(int(s), np.float32(1.0), src_b[p]) for p, s in enumerate(b_slot) if s >= 0]
    for s, c, row in terms:
        out[s] = (out[s] + (c * row.astype(np.float32)).astype(np.float32)).astype(np.float32)
    return out


def ordered_rows_fp64(a_slot, a_row, a_coef, src_a, b_slot, src_b, n_slots):
    """The same sums in fp64 (no rounding order)."""
    cols = (src_a if src_a is not None and len(src_a) else src_b).shape[1]
    out = np.zeros((n_slots, cols))
    for s, r, c in zip(a_slot, a_row, a_coef):
        if s >= 0:
            out[s] += float(c) * src_a[int(r)].astype(np.float64)
    for p, s in enumerate(b_slot):
        if s >= 0:
            out[s] += src_b[p].astype(np.float64)
    return out


def _softplus(x):
    return np.logaddexp(0.0, x)


def rank_loss_slots(h, emb, pos, neg):
    """fp64 softplus(h_p . e(neg) - h_p . e(pos)) per position, 0 where pos < 0."""
    h, emb = np.asarray(h, np.float64), np.asarray(emb, np.float64)
    out = np.zeros(len(pos))
    ok = np.asarray(pos) >= 0
    p = np.flatnonzero(ok)
    out[p] = _softplus((h[p] * emb[neg[p]]).sum(1) - (h[p] * emb[pos[p]]).sum(1))
    return out


def impression_loss_slots(h, emb, pos_indptr, indptr, items, clicked, kind, ids=None, K=0, seed=0, epoch=0):
    """fp64 loss per position: the sum over its impressions of the pairwise mean softplus(s_n - s_c) (kind 'pairwise') or of
    log(e^{s_c} + sum_{S_c} e^{s_n}) - s_c over its clicks (kind 'softmax'); impressions without a click or a non-click add 0."""
    h, emb = np.asarray(h, np.float64), np.asarray(emb, np.float64)
    out = np.zeros(len(pos_indptr) - 1)
    for p in range(len(out)):
        for q in range(pos_indptr[p], pos_indptr[p + 1]):
            it, c = items[indptr[q]:indptr[q + 1]], clicked[indptr[q]:indptr[q + 1]].astype(bool)
            if c.all() or not c.any():
                continue
            s = emb[it] @ h[p]
            if kind == 'pairwise':
                out[p] += _softplus(s[~c][None] - s[c][:, None]).mean()
            else:
                for cp, S in negative_sets(c, int(ids[q]), K, seed, epoch):
                    a = s[np.concatenate([[cp], S]).astype(np.int64)]
                    out[p] += np.logaddexp.reduce(a) - a[0]
    return out
