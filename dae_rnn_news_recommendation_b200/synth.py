"""Synthetic bag-of-words generators for the BASELINE.json configs (there is no network for datasets).

Rows look like CountVectorizer / TfidfTransformer output (reference datasets/articles.py:131-174): ~Poisson(mean_nnz)
distinct words per article, word ids Zipf-distributed (frequent words shared across articles), values 1 (binary) or
row-L2-normalised positive weights (tf-idf like).  Deterministic in `seed`.
"""
import numpy as np
import scipy.sparse as sp


def make_sparse(n_rows, n_features, mean_nnz=100, kind='binary', seed=0, zipf_s=1.1, chunk=32768):
    rng = np.random.default_rng(seed)
    if zipf_s > 0:
        p = 1.0 / np.arange(1, n_features + 1, dtype=np.float64) ** zipf_s
    else:
        p = np.ones(n_features)
    cdf = np.cumsum(p / p.sum())
    cdf[-1] = 1.0
    colperm = rng.permutation(n_features).astype(np.int32)
    indptr = [np.zeros(1, dtype=np.int64)]
    idx_parts, val_parts = [], []
    base = 0
    for r0 in range(0, n_rows, chunk):
        m = min(chunk, n_rows - r0)
        k = np.clip(rng.poisson(mean_nnz, m), 1, n_features)
        kmax = int(k.max())
        D = 3 * kmax + 8  # candidates per row; the first k DISTINCT ones are kept (sampling without replacement)
        cand = colperm[np.searchsorted(cdf, rng.random((m, D)), side='left')].astype(np.int64)
        order = np.argsort(cand, axis=1, kind='stable')
        srt = np.take_along_axis(cand, order, axis=1)
        first_sorted = np.ones_like(srt, dtype=bool)
        first_sorted[:, 1:] = srt[:, 1:] != srt[:, :-1]
        is_first = np.zeros_like(first_sorted)
        np.put_along_axis(is_first, order, first_sorted, axis=1)
        rank = np.cumsum(is_first, axis=1)
        sel = is_first & (rank <= k[:, None])
        cols = np.where(sel, cand, n_features)  # sentinel: not selected
        cols.sort(axis=1)
        keep = cols < n_features
        cnt = keep.sum(1)
        idx = cols[keep].astype(np.int32)
        if kind == 'binary':
            val = np.ones(idx.shape[0], dtype=np.float32)
        else:
            val = (1.0 - rng.random(idx.shape[0])).astype(np.float32)  # (0,1]
            rows = np.repeat(np.arange(m), cnt)
            nrm = np.sqrt(np.bincount(rows, weights=val.astype(np.float64) ** 2, minlength=m))
            val = (val / nrm[rows]).astype(np.float32)
        ip = base + np.cumsum(cnt)
        base = int(ip[-1])
        indptr.append(ip.astype(np.int64))
        idx_parts.append(idx)
        val_parts.append(val)
    m = sp.csr_matrix((np.concatenate(val_parts), np.concatenate(idx_parts), np.concatenate(indptr)),
                      shape=(n_rows, n_features))
    m.has_sorted_indices = True
    return m


def make_histories(n_users, labels, mean_len=20, seed=0, max_len=2000, holdout=True, second_class=0.5, primary_share=0.7):
    """Synthetic reading histories over articles labelled `labels` (class ids >= 0; -1 articles are never read).
    Each user prefers one class, or with probability `second_class` two (a share `primary_share` of the reads from the first);
    inside a class, article popularity follows a Zipf law (rank r drawn log-uniformly, P ~ 1 / r, over a random order of the
    class); history lengths are geometric with mean `mean_len`, at least 1 and capped at `max_len`.  A repeated draw counts once.
    holdout: one more read per user drawn the same way is held out as the target (and removed from the history if already there).
    Returns (histories, targets): scipy CSR float32 [n_users, N] with weight 1 per read; targets is None without holdout."""
    rng = np.random.default_rng(seed)
    labels = np.asarray(labels).reshape(-1)
    n = labels.shape[0]
    valid = np.flatnonzero(labels >= 0)
    classes, inv = np.unique(labels[valid], return_inverse=True)
    if classes.size == 0:
        raise ValueError('make_histories: no labelled article')
    order = valid[np.lexsort((rng.random(valid.size), inv))]   # articles grouped by class, random popularity order inside
    size = np.bincount(inv, minlength=classes.size)
    start = np.concatenate([[0], np.cumsum(size)[:-1]])
    c1 = rng.integers(0, classes.size, n_users)
    two = rng.random(n_users) < second_class
    c2 = np.where(two, rng.integers(0, classes.size, n_users), c1)
    lens = np.minimum(rng.geometric(1.0 / max(mean_len, 1.0), n_users), max_len)
    draws = lens + (1 if holdout else 0)
    user = np.repeat(np.arange(n_users), draws)
    cls = np.where(rng.random(user.size) < primary_share, c1[user], c2[user])
    rank = np.minimum(np.floor(np.exp(rng.random(user.size) * np.log(size[cls] + 1.0))).astype(np.int64) - 1, size[cls] - 1)
    art = order[start[cls] + rank]
    ends = np.cumsum(draws)
    is_target = np.zeros(user.size, dtype=bool)
    if holdout:
        is_target[ends - 1] = True
    hist = sp.csr_matrix((np.ones(int((~is_target).sum()), np.float32), (user[~is_target], art[~is_target])), shape=(n_users, n))
    hist.sum_duplicates()
    hist.data[:] = 1.0
    targets = None
    if holdout:
        targets = sp.csr_matrix((np.ones(n_users, np.float32), (user[is_target], art[is_target])), shape=(n_users, n))
        hist = (hist - hist.multiply(targets)).tocsr()   # a held-out read is not in the history
        hist.eliminate_zeros()
        hist.sort_indices()
    return hist.astype(np.float32), targets


def make_sequences(n_users, labels, mean_len=20, session_len=5, seed=0, max_len=2000, holdout=True, tries=20):
    """Synthetic ordered reading sequences over articles labelled `labels` (class ids >= 0; -1 articles are never read).
    Each user prefers 2 or 3 classes.  Reads come in sessions (geometric lengths, mean `session_len`); each session picks one of the
    user's classes uniformly and reads Zipf-popular articles of it (as make_histories).  Sequence lengths are geometric with mean
    `mean_len`, at least 1 and capped at `max_len`.  So the next read follows the current session's class, which the order of the
    reads shows and their mean does not.
    holdout: the target is the user's next read, drawn in the last session, redrawn up to `tries` times while it is an article the
    user already read (-1 when every draw was).
    Returns (indptr int64 [U + 1], items int32, targets int64 [U] or None)."""
    rng = np.random.default_rng(seed)
    labels = np.asarray(labels).reshape(-1)
    valid = np.flatnonzero(labels >= 0)
    classes, inv = np.unique(labels[valid], return_inverse=True)
    if classes.size == 0:
        raise ValueError('make_sequences: no labelled article')
    nc = classes.size
    order = valid[np.lexsort((rng.random(valid.size), inv))]
    size = np.bincount(inv, minlength=nc)
    start = np.concatenate([[0], np.cumsum(size)[:-1]])
    prefs = np.argsort(rng.random((n_users, nc)), axis=1)[:, :3]
    n_pref = np.minimum(rng.integers(2, 4, n_users), nc)
    lens = np.minimum(rng.geometric(1.0 / max(mean_len, 1.0), n_users), max_len)
    user = np.repeat(np.arange(n_users), lens)
    first = np.zeros(user.size, dtype=bool)
    first[np.cumsum(lens) - lens] = True
    new = first | (rng.random(user.size) < 1.0 / max(session_len, 1.0))
    sess = np.cumsum(new) - 1
    sess_cls = prefs[user[new], (rng.random(int(new.sum())) * n_pref[user[new]]).astype(np.int64)]

    def draw(cls):
        rank = np.minimum(np.floor(np.exp(rng.random(cls.size) * np.log(size[cls] + 1.0))).astype(np.int64) - 1, size[cls] - 1)
        return order[start[cls] + rank]

    items = draw(sess_cls[sess]).astype(np.int32)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    targets = None
    if holdout:
        last_cls = sess_cls[sess[indptr[1:] - 1]]
        targets = np.full(n_users, -1, np.int64)
        read = sp.csr_matrix((np.ones(items.size), (user, items)), shape=(n_users, labels.shape[0]))
        todo = np.arange(n_users)
        for _ in range(tries):
            t = draw(last_cls[todo])
            ok = np.asarray(read[todo, t]).ravel() == 0
            targets[todo[ok]] = t[ok]
            todo = todo[~ok]
            if todo.size == 0:
                break
    return indptr, items, targets


def make_impressions(indptr, items, labels, targets=None, shown=20, seed=0, tries=20):
    """Synthetic impression logs for make_sequences' users (user_model.check_impressions' keys).  Returns (train, test):
    train has one impression per user and time t = 1 .. len - 1 that clicks read t + 1; test (with targets) has one per user
    with a target, at time = len, that clicks the target.  Each shows the click and shown - 1 distinct other articles in a
    random order: (shown - 1) // 2 from the classes of the user's reads before the impression other than the click's class (a
    class drawn through a random earlier read; from the whole catalogue when there is none within `tries` draws) and the rest
    from the whole catalogue.  Every distractor is a random read of all users' reads in its class, so articles are shown as
    often as they are read (make_sequences' Zipf popularity) and popularity does not give the click away.  A distractor that
    repeats the click or another distractor is redrawn up to `tries` times and dropped after that."""
    rng = np.random.default_rng(seed)
    indptr, items = np.asarray(indptr, np.int64), np.asarray(items, np.int64)
    labels = np.asarray(labels).reshape(-1)
    cls_of = labels[items].astype(np.int64)
    pool = items[np.argsort(cls_of, kind='stable')]
    classes = np.sort(cls_of)
    ids = np.arange(int(classes.max(initial=0)) + 1)
    c_lo, c_hi = np.searchsorted(classes, ids, 'left'), np.searchsorted(classes, ids, 'right')   # class c's reads: pool[c_lo:c_hi]
    lens = np.diff(indptr)
    k_user = (shown - 1) // 2

    def impressions(user, time, click):
        n = user.size
        # the class of each user-side distractor: a random earlier read's class other than the click's
        src_cls = np.full((n, k_user), -1, np.int64)
        todo = np.ones((n, k_user), bool)
        for _ in range(tries):
            r, c = np.nonzero(todo)
            if r.size == 0:
                break
            pick = indptr[user[r]] + (rng.random(r.size) * time[r]).astype(np.int64)
            cl = cls_of[pick]
            ok = cl != labels[click[r]]
            src_cls[r[ok], c[ok]] = cl[ok]
            todo[r[ok], c[ok]] = False

        def draw(cl):   # a random read of class cl (a random read of all when cl < 0)
            glob = cl < 0
            lo = np.where(glob, 0, c_lo[np.maximum(cl, 0)])
            hi = np.where(glob, pool.size, c_hi[np.maximum(cl, 0)])
            return pool[lo + (rng.random(cl.size) * (hi - lo)).astype(np.int64)]

        cls = np.concatenate([src_cls, np.full((n, shown - 1 - k_user), -1, np.int64)], 1).reshape(-1)
        dis = draw(cls).reshape(n, shown - 1)
        for _ in range(tries + 1):
            full = np.concatenate([click[:, None], dis], 1)
            o = np.argsort(full, axis=1, kind='stable')
            srt = np.take_along_axis(full, o, 1)
            dup = np.zeros_like(full, dtype=bool)
            rep = np.zeros_like(srt, dtype=bool)
            rep[:, 1:] = srt[:, 1:] == srt[:, :-1]
            np.put_along_axis(dup, o, rep, 1)   # the stable sort keeps the click (column 0) first among equal articles
            bad = dup[:, 1:]
            if not bad.any():
                break
            r, c = np.nonzero(bad)
            if _ < tries:
                dis[r, c] = draw(cls.reshape(n, -1)[r, c])
        keep = ~bad
        m = 1 + keep.sum(1)
        ind = np.concatenate([[0], np.cumsum(m)]).astype(np.int64)
        rows = np.concatenate([click[:, None], dis], 1)[np.concatenate([np.ones((n, 1), bool), keep], 1)]
        clicked = np.zeros(rows.size, np.uint8)
        clicked[ind[:-1]] = 1
        # a random order within each impression
        key = np.repeat(np.arange(n), m) + rng.random(rows.size)
        o = np.argsort(key, kind='stable')
        return {'user': user.astype(np.int64), 'time': time.astype(np.int64), 'indptr': ind, 'items': rows[o].astype(np.int32),
                'clicked': clicked[o]}

    n_u = lens.size
    t_user = np.repeat(np.arange(n_u), np.maximum(lens - 1, 0))
    t_time = np.arange(t_user.size) - np.repeat(np.cumsum(np.maximum(lens - 1, 0)) - np.maximum(lens - 1, 0), np.maximum(lens - 1, 0)) + 1
    train = impressions(t_user, t_time, items[indptr[t_user] + t_time])
    test = None
    if targets is not None:
        targets = np.asarray(targets, np.int64)
        u = np.flatnonzero((targets >= 0) & (lens > 0))
        test = impressions(u, lens[u], targets[u])
    return train, test


def make_long_term_impressions(n_users, labels, window=5, history=(20, 40), shown=5, home_share=0.7, seed=0):
    """Reading sequences whose signal lies before the last `window` reads, and one training and one test impression per user
    (user_model.check_impressions' keys): the learning check of the long-term user vectors (DESIGN 4.18).  labels: class ids of
    the articles (at least 3 classes).  Each user has a home class.  The first h reads (h uniform in `history`) come in sessions
    of 2 to 5 reads, each from the home class with probability home_share and from another class otherwise; the last `window`
    reads are one session of a noise class, never home.  Both impressions are at time = len, so an encoder that sees only the
    last `window` reads has seen only the noise session: each clicks one home-class article and shows shown - 1 non-clicks,
    (shown - 1) // 2 from the noise class and the rest from the classes that are neither.  Returns (indptr, items, train, test)."""
    rng = np.random.default_rng(seed)
    labels = np.asarray(labels).astype(np.int64)
    C = int(labels.max()) + 1
    pools = [np.flatnonzero(labels == c) for c in range(C)]
    seqs = []
    imps = ([], [])
    n_noise = (shown - 1) // 2
    for u in range(n_users):
        home = int(rng.integers(C))
        others = [c for c in range(C) if c != home]
        h = int(rng.integers(history[0], history[1] + 1))
        s = []
        while len(s) < h:
            c = home if rng.random() < home_share else others[int(rng.integers(len(others)))]
            s.extend(rng.choice(pools[c], int(rng.integers(2, 6))))
        noise = others[int(rng.integers(len(others)))]
        s = np.concatenate([np.asarray(s[:h]), rng.choice(pools[noise], window)])
        seqs.append(s)
        rest = np.concatenate([pools[c] for c in others if c != noise])
        for imp in imps:
            shown_items = np.concatenate([rng.choice(pools[home], 1), rng.choice(pools[noise], n_noise, replace=False),
                                          rng.choice(rest, shown - 1 - n_noise, replace=False)])
            clicked = np.zeros(shown, np.uint8)
            clicked[0] = 1
            o = rng.permutation(shown)
            imp.append((u, s.size, shown_items[o], clicked[o]))
    indptr = np.concatenate([[0], np.cumsum([s.size for s in seqs])]).astype(np.int64)
    items = np.concatenate(seqs).astype(np.int32)

    def pack(imp):
        return {'user': np.array([x[0] for x in imp], np.int64), 'time': np.array([x[1] for x in imp], np.int64),
                'indptr': np.arange(len(imp) + 1, dtype=np.int64) * shown, 'items': np.concatenate([x[2] for x in imp]).astype(np.int32),
                'clicked': np.concatenate([x[3] for x in imp])}
    return indptr, items, pack(imps[0]), pack(imps[1])


def make_labels(n_rows, n_classes=4, seed=0):
    return np.random.default_rng(seed + 7919).integers(0, n_classes, n_rows).astype(np.float32)


def perturb_rows(m, frac=0.3, seed=1, zipf_s=1.1):
    """'pos' rows for the explicit-triplet config: the anchor with ~frac of its entries resampled."""
    rng = np.random.default_rng(seed)
    coo = m.tocoo()
    keep = rng.random(coo.nnz) >= frac
    extra = make_sparse(m.shape[0], m.shape[1], mean_nnz=max(1, int(frac * m.nnz / m.shape[0])), kind='binary',
                        seed=seed + 1, zipf_s=zipf_s)
    base = sp.coo_matrix((coo.data[keep], (coo.row[keep], coo.col[keep])), shape=m.shape).tocsr()
    out = (base + extra).tocsr()
    out.data[:] = 1.0
    out.sort_indices()
    return out.astype(np.float32)
