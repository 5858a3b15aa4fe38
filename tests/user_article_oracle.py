"""fp64 reference of the user encoders trained jointly with the article encoder (user_model.ArticleEncoder, DESIGN 4.19): the DAE
encoder e(x) = f(s x W + bh) - f(bh) with W and bh as autograd leaves, the GRU / LSTM / attention states over e(a) of each read,
and the random-negative, pairwise-impression and sampled-softmax losses.  Tests only."""
import numpy as np
import scipy.sparse as sp
import torch

import user_attention_oracle as uo

RNN_NAMES = ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')
KINDS = ('random', 'pairwise', 'softmax')


def act(name, x):
    return torch.sigmoid(x) if name == 'sigmoid' else torch.tanh(x) if name == 'tanh' else x


def vectors(X, W, bh, act_name, in_scale):
    """e(X) [N, H] and the pre-activation A (fp64 tensors, differentiable in W and bh); X: scipy sparse or dense [N, F]."""
    Xd = torch.as_tensor(np.asarray(X.todense() if sp.issparse(X) else X, np.float64))
    A = in_scale * Xd @ W + bh
    return act(act_name, A) - act(act_name, bh), A


def rnn_states(cell, params, xs, h0=None):
    """States [L_u, H] of each user from the inputs xs (list of [L_u, H] tensors), h_0 = h0[i] or 0 (c_0 = 0)."""
    Wi, Wh, bi, bh = (params[n] for n in RNN_NAMES)
    H = Wh.shape[1]
    out = []
    for i, x in enumerate(xs):
        h = torch.zeros(H, dtype=torch.float64) if h0 is None else h0[i]
        c = torch.zeros(H, dtype=torch.float64)
        hs = []
        for t in range(x.shape[0]):
            xg = Wi @ x[t] + bi
            hg = Wh @ h + bh
            if cell == 'gru':
                r = torch.sigmoid(xg[:H] + hg[:H])
                z = torch.sigmoid(xg[H:2 * H] + hg[H:2 * H])
                n = torch.tanh(xg[2 * H:] + r * hg[2 * H:])
                h = (1 - z) * n + z * h
            else:
                g = xg + hg
                i_, f_, g_, o_ = torch.sigmoid(g[:H]), torch.sigmoid(g[H:2 * H]), torch.tanh(g[2 * H:3 * H]), torch.sigmoid(g[3 * H:])
                c = f_ * c + i_ * g_
                h = o_ * torch.tanh(c)
            hs.append(h)
        out.append(torch.stack(hs))
    return out


def states(cell, params, xs, heads=None, h0=None):
    if cell == 'attention':
        return [uo.encode(params, x, heads)[0] for x in xs]
    return rnn_states(cell, params, xs, h0)


def loss(kind, hs, E, seqs, data):
    """random: data = per user the L - 1 negatives, mean over the terms softplus(h_t.e(neg) - h_t.e(a_{t+1})); pairwise: data = list
    of (user, t, items, clicked), mean over impressions of 1 / (|C| |N|) sum softplus(s_n - s_c); softmax: data = list of (user, t,
    click item, negative items), mean over samples of log(e^{s_c} + sum e^{s_n}) - s_c."""
    idx = lambda a: torch.as_tensor(np.asarray(a, np.int64))   # noqa: E731
    terms = []
    if kind == 'random':
        for h, s, ng in zip(hs, seqs, data):
            if len(s) < 2:
                continue
            ht = h[:-1]
            terms.append(torch.nn.functional.softplus((ht * E[idx(ng)]).sum(1) - (ht * E[idx(s[1:])]).sum(1)))
        return torch.cat(terms).mean()
    for i, t, a, b in data:
        if kind == 'pairwise':
            c = np.asarray(b).astype(bool)
            s = E[idx(a)] @ hs[i][t]
            terms.append(torch.nn.functional.softplus(s[torch.from_numpy(~c)][None, :] - s[torch.from_numpy(c)][:, None]).mean())
        else:
            s = E[idx(np.concatenate([[a], np.asarray(b, np.int64)]))] @ hs[i][t]
            terms.append(torch.logsumexp(s, 0) - s[0])
    return torch.stack(terms).mean()


def joint(cell, params_np, W_np, bh_np, X, act_name, in_scale, seqs, kind, data, heads=None, h0=None, articles=True):
    """The joint loss of one batch and its gradients.  seqs: per user its (truncated) reads.  With articles=False W and bh are
    constants (the frozen-embedding loss).  Returns {'loss', 'grads' ({name: grad}), 'dW', 'dbh', 'E', 'dE' (dL/de of every
    article), 'dA' (dL/dA), 'dX' (per user [L_u, H]: dL/dx of each read's input), 'states'}."""
    params = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in params_np.items()}
    W = torch.tensor(np.asarray(W_np, np.float64), requires_grad=articles)
    bh = torch.tensor(np.asarray(bh_np, np.float64), requires_grad=articles)
    E, A = vectors(X, W, bh, act_name, in_scale)
    if not articles:
        E, A = E.detach().requires_grad_(True), A.detach()
    E.retain_grad()
    if A.requires_grad:
        A.retain_grad()
    xs = [E[torch.as_tensor(np.asarray(s, np.int64))] for s in seqs]
    for x in xs:
        x.retain_grad()
    hs = states(cell, params, xs, heads, h0)
    L = loss(kind, hs, E, seqs, data)
    L.backward()
    return {'loss': float(L.detach()), 'grads': {k: v.grad.numpy() for k, v in params.items()},
            'dW': W.grad.numpy() if articles else None, 'dbh': bh.grad.numpy() if articles else None,
            'E': E.detach().numpy(), 'dE': E.grad.numpy(), 'dA': A.grad.numpy() if articles else None,
            'dX': [np.zeros(tuple(x.shape)) if x.grad is None else x.grad.numpy() for x in xs], 'states': [h.detach().numpy() for h in hs]}


def compact(ids):
    """dae_touch_compact restated: (rows, slots) -- the distinct ids >= 0 in the order of their first occurrence, and each id's
    index in rows (-1 for ids < 0)."""
    ids = np.asarray(ids, np.int64)
    valid = np.flatnonzero(ids >= 0)
    _, first = np.unique(ids[valid], return_index=True)
    rows = ids[valid[np.sort(first)]]
    slot_of = {int(a): k for k, a in enumerate(rows)}
    slots = np.array([slot_of[int(a)] if a >= 0 else -1 for a in ids], np.int32)
    return rows.astype(np.int32), slots
