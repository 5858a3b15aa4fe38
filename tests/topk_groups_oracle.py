"""Host references for the grouped top-k (top_k_similar(groups=...), recommend(groups=...), dae_*_topk_groups*).

grouped_top_k: the contract directly -- candidates in (score desc, index asc) order, the first member of each group kept, the k
best of those.  brute_force_grouped: the same answer a different way (best member of every group, then sort), for the host test.
streamed_grouped: a model of the kernels -- per-part streaming lists of KMAX slots of which the first k count, and the merge that
skips taken groups -- so that the two facts the design rests on are checked on the host.
"""
import numpy as np


def grouped_top_k(s, groups, k, allowed=None):
    """s [Nq, Nc] scores (exactly what the kernel computes, any float dtype), groups int [Nc], allowed: optional bool [Nq, Nc]
    mask of the candidates.  Returns (index int32 [Nq, k], score float32 [Nq, k]) padded with -1 / -inf."""
    s = np.asarray(s)
    groups = np.asarray(groups)
    nq, nc = s.shape
    idx = np.full((nq, k), -1, np.int32)
    val = np.full((nq, k), -np.inf, np.float32)
    cols = np.arange(nc)
    for r in range(nq):
        c = cols if allowed is None else cols[allowed[r]]
        order = c[np.lexsort((c, -s[r, c].astype(np.float64)))]
        _, first = np.unique(groups[order], return_index=True)
        sel = order[np.sort(first)[:k]]
        idx[r, :sel.size] = sel
        val[r, :sel.size] = s[r, sel]
    return idx, val


def brute_force_grouped(s, groups, k, allowed=None):
    """The same answer by another route: every group's best candidate (max score, then min index), then the k best of those."""
    nq, nc = s.shape
    idx = np.full((nq, k), -1, np.int32)
    val = np.full((nq, k), -np.inf, np.float32)
    for r in range(nq):
        best = {}
        for c in range(nc):
            if allowed is not None and not allowed[r, c]:
                continue
            g, v = int(groups[c]), float(s[r, c])
            if g not in best or v > best[g][0]:   # columns in increasing order: an equal score keeps the lower index
                best[g] = (v, c)
        reps = sorted(best.values(), key=lambda t: (-t[0], t[1]))[:k]
        for j, (v, c) in enumerate(reps):
            idx[r, j], val[r, j] = c, v
    return idx, val


def _stream(row, cols, groups, k, kmax, all_slots=False):
    """One partial list as the dense epilogue keeps it: KMAX slots, the first k hold distinct groups.  all_slots: look for the
    candidate's group in every slot, not only the first k."""
    sv = [-np.inf] * kmax
    si = [-1] * kmax
    for c in cols:
        v, g = float(row[c]), int(groups[c])
        if not v > sv[k - 1]:
            continue
        gp = kmax - 1
        for j in range(kmax if all_slots else k):
            if si[j] >= 0 and int(groups[si[j]]) == g:
                gp = j
        if not v > sv[gp]:
            continue
        pos = next(j for j in range(gp + 1) if v > sv[j])
        sv[pos + 1:gp + 1], si[pos + 1:gp + 1] = sv[pos:gp], si[pos:gp]
        sv[pos], si[pos] = v, c
    return list(zip(sv[:k], si[:k]))


def _merge(lists, groups, k):
    heads = [entry for lst in lists for entry in lst if entry[1] >= 0]
    heads.sort(key=lambda t: (-t[0], t[1]))
    out, taken = [], set()
    for v, c in heads:
        if int(groups[c]) in taken:
            continue
        taken.add(int(groups[c]))
        out.append((v, c))
        if len(out) == k:
            break
    return out


def streamed_grouped(s, groups, k, parts, kmax=32, allowed=None, all_slots=False):
    """The kernels' route: the candidate columns cut into `parts` contiguous ranges, one streaming list per range, then the merge."""
    nq, nc = s.shape
    idx = np.full((nq, k), -1, np.int32)
    val = np.full((nq, k), -np.inf, np.float32)
    bounds = np.linspace(0, nc, parts + 1).astype(int)
    for r in range(nq):
        lists = []
        for p in range(parts):
            cols = range(bounds[p], bounds[p + 1])
            if allowed is not None:
                cols = [c for c in cols if allowed[r, c]]
            lists.append(_stream(s[r], cols, groups, k, kmax, all_slots))
        for j, (v, c) in enumerate(_merge(lists, groups, k)):
            idx[r, j], val[r, j] = c, v
    return idx, val
