"""fp64 references of the attention user encoder (user_model.UserAttention, csrc/user_attention.cu).  Tests only.

Whole batches: the causal multi-head self-attention and additive pooling written out in torch (attention_states), the three losses
with their gradients by autograd (loss_and_grads, impression_loss_and_grads, softmax_loss_and_grads) and the evaluation windows
of impression_states (window_states).

Kernels: each reference returns (value, scale) per output and a kernel passes when |got - want| <= C_FP32 scale + tiny for every
element (C_FP32 = 2^-20, 16 units of fp32 rounding u = 2^-24; gru_kernel_oracle.check), from the kernel's own fp32 inputs taken
exact.  The scales count the roundings of the kernels' fp32 operation order:
  score s_ts = c q_t . k_s (c = 1 / sqrt d): d fmas, an absolute error of d u E_ts with E_ts = c sum |q_t k_s|; the row's weights
    p_ts = e^{s_ts - lse_t} then carry 2 d u max_s E_ts relatively, and the online softmax adds one rounding per key tile and
    per key of l_t: O_t[j] within (2 d E_t + L + 8) u sum_s p_ts |v_s[j]|; lse_t within (d E_t + L + 8 + |lse_t|) u.
  dS_ts = p_ts (dO_t . v_s - D_t) with D_t = dO_t . O_t: p's error as above, the two d-term dots each within (d + 4) u of their
    absolute sums; dQ_t = c sum_s dS_ts k_s and dK_s = c sum_t dS_ts q_t add (L + 4) u of sum |dS k| (|dS q|);
    dV_s = sum_{t >= s} p_ts dO_t: (2 d E + L + 8) u sum p |dO|.
  pooling: a_s = q . tanh Z_s: tanhf within 2 u of |T| + (1 - T^2) |Z| u for the rounded input, A fmas: (A + 8) u sum_k |q_k|
    (|T| + (1 - T^2) |Z|) = scale_a; the prefix weights w_ts = e^{a_s - lse_t} carry (2 max scale_a + t + 16) u relatively, so
    u_t[j] within that times sum_s w_ts |M_s[j]|.
  pooling backward (from the exact fp32 a and lse): w_ts = w_ss prod e_r carries (2 L + 16) u, so dM_s (value path) within
    (2 L + 16) u sum_t w_ts |dU_t|; da_s = w_ss (M_s . R_s - C_s) within (H + 2 L + 24) u w_ss (sum_j |M_s[j]| |R|_s[j] + |C|_s)
    (|R|, |C|: the same sums of absolute values); dZ = da q (1 - T^2) adds 8 u (|da q| (1 + T^2)); dq_k = sum_s da_s T_sk over
    at most L reads per user, B / 32 users per warp and 32 warps: (L + B / 32 + 40) u of sum |da| (|T| + 2) plus the da errors.
"""
import numpy as np
import torch

U = 2.0 ** -24


def _np64(a):
    return np.asarray(a, np.float64)


# ---------------------------------------------------------------------------------------------------------------------------
# whole batches
# ---------------------------------------------------------------------------------------------------------------------------
def encode(params, X, heads):
    """u [L, H] of one window X [L, H] (fp64 tensors, differentiable in params), and m [L, H] (the attention output)."""
    L, H = X.shape
    d = H // heads
    qkv = X @ params['self_attn.in_proj_weight'].T + params['self_attn.in_proj_bias']
    q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    mask = torch.triu(torch.ones(L, L, dtype=torch.bool), 1)
    outs = []
    for h in range(heads):
        sl = slice(h * d, (h + 1) * d)
        s = (q[:, sl] @ k[:, sl].T) / np.sqrt(d)
        outs.append(torch.softmax(s.masked_fill(mask, float('-inf')), 1) @ v[:, sl])
    m = torch.cat(outs, 1) @ params['self_attn.out_proj.weight'].T + params['self_attn.out_proj.bias']
    a = torch.tanh(m @ params['pool.weight'].T + params['pool.bias']) @ params['pool.query']
    w = torch.softmax(a[None, :].expand(L, L).masked_fill(mask, float('-inf')), 1)
    return w @ m, m


def attention_states(params, seqs, emb, heads):
    """u of every user: list of [L_u, H] tensors (fp64).  seqs: list of item arrays (already truncated)."""
    E = torch.as_tensor(_np64(emb))
    H = E.shape[1]
    return [encode(params, E[torch.as_tensor(np.asarray(s, np.int64))], heads)[0] if len(s) else torch.zeros(0, H, dtype=torch.float64)
            for s in seqs]


def _leaf(params_np):
    return {k: torch.tensor(_np64(v), requires_grad=True) for k, v in params_np.items()}


def loss_and_grads(params_np, seqs, negs, emb, heads):
    """The random-negative loss (user_lstm_oracle.rank_loss) of a batch: (loss, {name: grad}, states)."""
    from user_lstm_oracle import rank_loss
    params = _leaf(params_np)
    hs = attention_states(params, seqs, emb, heads)
    loss = rank_loss(hs, seqs, negs, emb)
    loss.backward()
    return float(loss.detach()), {k: v.grad.numpy() for k, v in params.items()}, [h.detach().numpy() for h in hs]


def impression_loss_and_grads(params_np, seqs, emb, imps, heads):
    """The pairwise impression loss: imps is a list of (user index, t, items, clicked).  (loss, {name: grad})."""
    params = _leaf(params_np)
    E = torch.as_tensor(_np64(emb))
    hs = attention_states(params, seqs, emb, heads)
    terms = []
    for i, t, it, c in imps:
        c = np.asarray(c).astype(bool)
        s = E[torch.as_tensor(np.asarray(it, np.int64))] @ hs[i][t]
        terms.append(torch.nn.functional.softplus(s[torch.from_numpy(~c)][None, :] - s[torch.from_numpy(c)][:, None]).mean())
    loss = torch.stack(terms).mean()
    loss.backward()
    return float(loss.detach()), {k: v.grad.numpy() for k, v in params.items()}


def softmax_loss_and_grads(params_np, seqs, emb, samples, heads):
    """The sampled-softmax impression loss: samples is a list of (user index, t, click item, negative items).  Mean over samples of
    log(e^{s_c} + sum_n e^{s_n}) - s_c.  (loss, {name: grad})."""
    params = _leaf(params_np)
    E = torch.as_tensor(_np64(emb))
    hs = attention_states(params, seqs, emb, heads)
    terms = []
    for i, t, c, negs in samples:
        it = torch.as_tensor(np.concatenate([[c], np.asarray(negs, np.int64)]).astype(np.int64))
        s = E[it] @ hs[i][t]
        terms.append(torch.logsumexp(s, 0) - s[0])
    loss = torch.stack(terms).mean()
    loss.backward()
    return float(loss.detach()), {k: v.grad.numpy() for k, v in params.items()}


def window_states(params_np, indptr, items, user, time, emb, max_len, heads):
    """[I, H]: u after the last min(time, max_len) reads before each impression; zero at time = 0."""
    params = {k: torch.as_tensor(_np64(v)) for k, v in params_np.items()}
    H = params['self_attn.out_proj.weight'].shape[0]
    out = np.zeros((len(user), H))
    seqs = [items[indptr[u] + max(0, t - max_len):indptr[u] + t] for u, t in zip(user, time)]
    for i, h in enumerate(attention_states(params, seqs, emb, heads)):
        if len(h):
            out[i] = h[-1].numpy()
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# kernels, per user in the packed layout: rows(off, i, L) are user i's positions
# ---------------------------------------------------------------------------------------------------------------------------
def rows(off, i, L):
    return np.asarray(off[:L], np.int64) + i


def attention_fwd(qkv, off, lens, H, heads):
    """dae_seq_attention_fwd: {'O': (value, scale) [P, H], 'lse': (value, scale) [P, heads]} over the positions of the users."""
    qkv = _np64(qkv)
    P, d = qkv.shape[0], H // heads
    c = 1.0 / np.sqrt(d)
    O, sO = np.zeros((P, H)), np.zeros((P, H))
    lse, sl = np.zeros((P, heads)), np.zeros((P, heads))
    for i, L in enumerate(lens):
        r = rows(off, i, int(L))
        mask = np.triu(np.ones((L, L), bool), 1)
        for h in range(heads):
            q, k, v = (qkv[r][:, g * H + h * d:g * H + (h + 1) * d] for g in range(3))
            s = np.where(mask, -np.inf, c * q @ k.T)
            E = np.where(mask, 0.0, c * np.abs(q) @ np.abs(k).T).max(1, keepdims=True)
            mx = s.max(1, keepdims=True)
            e = np.exp(s - mx)
            ls = mx + np.log(e.sum(1, keepdims=True))
            p = np.exp(s - ls)
            O[r, h * d:(h + 1) * d] = p @ v
            sO[r, h * d:(h + 1) * d] = (2 * d * E + L + 8) * (p @ np.abs(v))
            lse[r, h] = ls[:, 0]
            sl[r, h] = (d * E + L + 8 + np.abs(ls))[:, 0]
    return {'O': (O, sO / 16), 'lse': (lse, sl / 16)}


def attention_bwd(qkv, O, lse, dO, off, lens, H, heads):
    """dae_seq_attention_bwd from the kernel's inputs: {'dQKV': (value, scale) [P, 3H]}."""
    qkv, O, lse, dO = _np64(qkv), _np64(O), _np64(lse), _np64(dO)
    P, d = qkv.shape[0], H // heads
    c = 1.0 / np.sqrt(d)
    G, sG = np.zeros((P, 3 * H)), np.zeros((P, 3 * H))
    for i, L in enumerate(lens):
        r = rows(off, i, int(L))
        mask = np.triu(np.ones((L, L), bool), 1)
        for h in range(heads):
            sl = slice(h * d, (h + 1) * d)
            q, k, v = (qkv[r][:, g * H + h * d:g * H + (h + 1) * d] for g in range(3))
            go, o = dO[r][:, sl], O[r][:, sl]
            p = np.where(mask, 0.0, np.exp(c * q @ k.T - lse[r, h][:, None]))
            E = np.where(mask, 0.0, c * np.abs(q) @ np.abs(k).T).max(1, keepdims=True)
            D = (go * o).sum(1, keepdims=True)
            dP = go @ v.T
            dS = p * (dP - D)
            eS = p * (np.abs(dP - D) * (2 * d * E + 8) + (d + 4) * (np.abs(go) @ np.abs(v).T + (np.abs(go) * np.abs(o)).sum(1, keepdims=True)))
            G[r, sl] = c * dS @ k
            sG[r, sl] = c * (eS @ np.abs(k) + (L + 4) * np.abs(dS) @ np.abs(k))
            G[r, H + h * d:H + (h + 1) * d] = c * dS.T @ q
            sG[r, H + h * d:H + (h + 1) * d] = c * (eS.T @ np.abs(q) + (L + 4) * np.abs(dS).T @ np.abs(q))
            G[r, 2 * H + h * d:2 * H + (h + 1) * d] = p.T @ go
            sG[r, 2 * H + h * d:2 * H + (h + 1) * d] = (np.abs(p.T) * (2 * d * E.T + L + 8)) @ np.abs(go)
    return {'dQKV': (G, sG / 16)}


def pool_fwd(Z, q, M, off, lens, H, A):
    """dae_seq_pool_fwd: {'score', 'plse' [P], 'u' [P, H]} as (value, scale)."""
    Z, q, M = _np64(Z)[:, :A], _np64(q), _np64(M)[:, :H]
    P = Z.shape[0]
    T = np.tanh(Z)
    a = T @ q
    sa = (A + 8) * (np.abs(T) + (1 - T * T) * np.abs(Z)) @ np.abs(q)
    u, su, pl, spl = np.zeros((P, H)), np.zeros((P, H)), np.zeros(P), np.zeros(P)
    for i, L in enumerate(lens):
        r = rows(off, i, int(L))
        mask = np.triu(np.ones((L, L), bool), 1)
        x = np.where(mask, -np.inf, a[r][None, :])
        mx = x.max(1, keepdims=True)
        ls = mx + np.log(np.exp(x - mx).sum(1, keepdims=True))
        w = np.exp(x - ls)
        f = 2 * np.maximum.accumulate(sa[r]) + np.arange(L) + 16
        u[r] = w @ M[r]
        su[r] = f[:, None] * (w @ np.abs(M[r]))
        pl[r] = ls[:, 0]
        spl[r] = f - 8 + np.abs(ls[:, 0])
    return {'score': (a, sa / 16), 'plse': (pl, spl / 16), 'u': (u, su / 16)}


def pool_bwd(dU, u, M, Z, q, score, plse, off, lens, H, A):
    """dae_seq_pool_bwd from the kernel's inputs: {'dM' [P, H], 'dZ' [P, A], 'dq' [A]} as (value, scale)."""
    dU, u, M, Z, q, score, plse = (_np64(x) for x in (dU, u, M, Z, q, score, plse))
    dU, u, M, Z = dU[:, :H], u[:, :H], M[:, :H], Z[:, :A]
    P, B = Z.shape[0], len(lens)
    T = np.tanh(Z)
    dM, sdM, da, sda = np.zeros((P, H)), np.zeros((P, H)), np.zeros(P), np.zeros(P)
    for i, L in enumerate(lens):
        r = rows(off, i, int(L))
        mask = np.triu(np.ones((L, L), bool), 1)
        w = np.where(mask, 0.0, np.exp(score[r][None, :] - plse[r][:, None]))     # w[t, s]
        dM[r] = w.T @ dU[r]
        sdM[r] = (2 * L + 16) * (w.T @ np.abs(dU[r]))
        g = dU[r] @ M[r].T                                                        # g[t, s] = dU_t . M_s
        c = (dU[r] * u[r]).sum(1)
        da[r] = (w * (g - c[:, None])).sum(0)
        wss = np.exp(score[r] - plse[r])
        Rabs = np.where(mask, 0.0, np.exp(plse[r][None, :] - plse[r][:, None])).T @ np.abs(dU[r])   # sum_{t >= s} e^{lse_s - lse_t} |dU_t|
        Cabs = np.where(mask, 0.0, np.exp(plse[r][None, :] - plse[r][:, None])).T @ (np.abs(dU[r]) * np.abs(u[r])).sum(1)
        sda[r] = (H + 2 * L + 24) * wss * ((np.abs(M[r]) * Rabs).sum(1) + Cabs)
    dZ = da[:, None] * q[None, :] * (1 - T * T)
    sdZ = np.abs(q)[None, :] * (sda[:, None] * (1 - T * T) + 8 * np.abs(da)[:, None] * (1 + T * T))
    dq = T.T @ da
    Lmax = int(max(lens)) if len(lens) else 1
    sdq = np.abs(T).T @ sda + (Lmax + B / 32 + 40) * (np.abs(T) + 2).T @ np.abs(da)
    return {'dM': (dM, sdM / 16), 'dZ': (dZ, sdZ / 16), 'dq': (dq, sdq / 16)}
