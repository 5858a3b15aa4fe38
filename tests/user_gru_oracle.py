"""fp64 reference of the GRU user encoder (user_model.UserGRU): the torch.nn.GRU cell written out in torch, the ranking loss and
autograd, plus TF-1.12 Adam.  Tests only."""
import numpy as np
import torch

NAMES = ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')


def gru_states(params, seqs, emb):
    """States of every user: list of [L_u, H] tensors (fp64, differentiable in params).  seqs: list of item arrays (already
    truncated); params: dict of fp64 tensors with torch.nn.GRU's names."""
    Wi, Wh, bi, bh = (params[n] for n in NAMES)
    H = Wh.shape[1]
    E = torch.as_tensor(np.asarray(emb, np.float64))
    out = []
    for s in seqs:
        h = torch.zeros(H, dtype=torch.float64)
        hs = []
        for a in s:
            xg = Wi @ E[int(a)] + bi
            hg = Wh @ h + bh
            r = torch.sigmoid(xg[:H] + hg[:H])
            z = torch.sigmoid(xg[H:2 * H] + hg[H:2 * H])
            n = torch.tanh(xg[2 * H:] + r * hg[2 * H:])
            h = (1 - z) * n + z * h
            hs.append(h)
        out.append(torch.stack(hs) if hs else torch.zeros(0, H, dtype=torch.float64))
    return out


def loss_and_grads(params_np, seqs, negs, emb):
    """Mean over every (user, t < L - 1) of softplus(h_t . e(neg) - h_t . e(a_{t+1})).  negs: per user an array of L - 1
    negatives.  Returns (loss, {name: grad}, states)."""
    params = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in params_np.items()}
    E = torch.as_tensor(np.asarray(emb, np.float64))
    hs = gru_states(params, seqs, emb)
    terms = []
    for h, s, ng in zip(hs, seqs, negs):
        if len(s) < 2:
            continue
        ht = h[:-1]
        sp_ = (ht * E[torch.as_tensor(np.asarray(s[1:], np.int64))]).sum(1)
        sn = (ht * E[torch.as_tensor(np.asarray(ng, np.int64))]).sum(1)
        terms.append(torch.nn.functional.softplus(sn - sp_))
    loss = torch.cat(terms).mean()
    loss.backward()
    return float(loss), {k: v.grad.numpy() for k, v in params.items()}, [h.detach().numpy() for h in hs]


def adam_tf(p, g, m, v, t, lr):
    """TF-1.12 Adam (beta1 .9, beta2 .999, eps 1e-8), in place; t is the 1-based step."""
    m[:] = 0.9 * m + 0.1 * g
    v[:] = 0.999 * v + 0.001 * g * g
    lr_t = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
    p -= lr_t * m / (np.sqrt(v) + 1e-8)
