"""fp64 restatements for the impression-log path (user_model.UserGRU.fit(impressions=...), impression_states,
helpers.impression_metrics): the impression loss and its dh per packed position, the GRU batch gradient by autograd, the four
ranking metrics with the tie rule of dae_impression_metrics, and the evaluation windows.  Tests only."""
import numpy as np
import torch

from user_gru_oracle import gru_states


def _softplus(x):
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def impression_loss(h, emb, pos_indptr, indptr, items, clicked, scale):
    """(loss sum, dh [P, H]) of dae_impression_rank_loss in fp64: position p's impressions are [pos_indptr[p], pos_indptr[p + 1])."""
    h, emb = np.asarray(h, np.float64), np.asarray(emb, np.float64)
    dh = np.zeros_like(h)
    total = 0.0
    for p in range(h.shape[0]):
        for q in range(int(pos_indptr[p]), int(pos_indptr[p + 1])):
            it = items[indptr[q]:indptr[q + 1]]
            c = clicked[indptr[q]:indptr[q + 1]].astype(bool)
            if c.all() or not c.any():
                continue
            s = emb[it] @ h[p]
            x = s[~c][None, :] - s[c][:, None]          # [|C|, |N|]: s_n - s_c
            sig = 1.0 / (1.0 + np.exp(-x))
            inv = 1.0 / (c.sum() * (~c).sum())
            total += _softplus(x).sum() * inv
            w = np.zeros(it.size)
            w[~c] = sig.sum(0)
            w[c] = -sig.sum(1)
            dh[p] += scale * inv * (w @ emb[it])
    return total, dh


def impression_loss_and_grads(params_np, seqs, emb, imps):
    """Mean over the impressions of 1 / (|C| |N|) sum softplus(h_t . e_n - h_t . e_c) with h_t the state after read t' + 1 of a
    packed user's window.  seqs: per user the (truncated) reads; imps: list of (user index, t', items, clicked).  Returns
    (loss, {name: grad})."""
    params = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in params_np.items()}
    E = torch.as_tensor(np.asarray(emb, np.float64))
    hs = gru_states(params, seqs, emb)
    terms = []
    for i, t, it, c in imps:
        c = np.asarray(c).astype(bool)
        s = E[torch.as_tensor(np.asarray(it, np.int64))] @ hs[i][t]
        x = s[torch.from_numpy(~c)][None, :] - s[torch.from_numpy(c)][:, None]
        terms.append(torch.nn.functional.softplus(x).mean())
    loss = torch.stack(terms).mean()
    loss.backward()
    return float(loss), {k: v.grad.numpy() for k, v in params.items()}


def metrics(scores, indptr, clicked):
    """[I, 4] AUC, MRR, nDCG@5, nDCG@10 from the scores as given (fp32 scores compared as they are), ranks by score descending
    with ties to the earlier position; NaN rows for impressions without a click or without a non-click.  Also returns the
    integer parts: [I, 2] (2 x the AUC numerator, sum of the clicked ranks)."""
    n_imp = len(indptr) - 1
    out = np.full((n_imp, 4), np.nan)
    ints = np.zeros((n_imp, 2), np.int64)
    for i in range(n_imp):
        s = np.asarray(scores[indptr[i]:indptr[i + 1]])
        c = np.asarray(clicked[indptr[i]:indptr[i + 1]]).astype(bool)
        if c.all() or not c.any():
            continue
        m = s.size
        idx = np.arange(m)
        rank = np.array([(s > s[j]).sum() + ((s == s[j]) & (idx < j)).sum() for j in range(m)])
        sc, sn = s[c], s[~c]
        auc2 = int(2 * (sc[:, None] > sn[None, :]).sum() + (sc[:, None] == sn[None, :]).sum())
        rc = rank[c]
        ints[i] = auc2, int(rc.sum())
        out[i, 0] = auc2 / (2.0 * c.sum() * (~c).sum())
        out[i, 1] = np.mean(1.0 / (rc + 1.0))
        for col, k in ((2, 5), (3, 10)):
            dcg = (1.0 / np.log2(rc[rc < k] + 2.0)).sum()
            idcg = (1.0 / np.log2(np.arange(min(int(c.sum()), k)) + 2.0)).sum()
            out[i, col] = dcg / idcg
    return out, ints


def scores(q, emb, indptr, items, cosine):
    """fp64 scores of every shown article against its impression's query row."""
    q, emb = np.asarray(q, np.float64), np.asarray(emb, np.float64)
    row = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    e = emb[items]
    s = (q[row] * e).sum(1)
    if cosine:
        nq, ne = np.linalg.norm(q, axis=1)[row], np.linalg.norm(e, axis=1)
        s = np.where((nq > 0) & (ne > 0), s / np.where((nq > 0) & (ne > 0), nq * ne, 1.0), 0.0)
    return s


def window_states(params_np, indptr, items, user, time, emb, max_len):
    """[I, H]: the GRU state after the last min(time, max_len) reads before each impression; zero at time = 0."""
    params = {k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in params_np.items()}
    H = params['weight_hh_l0'].shape[1]
    out = np.zeros((len(user), H))
    seqs = [items[indptr[u] + max(0, t - max_len):indptr[u] + t] for u, t in zip(user, time)]
    for i, h in enumerate(gru_states(params, seqs, emb)):
        if len(h):
            out[i] = h[-1].detach().numpy()
    return out
