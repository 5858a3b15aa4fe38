"""fp64 references of the LSTM user encoder (user_model.UserLSTM, csrc/user_lstm.cu).  Tests only.

Whole batches: the torch.nn.LSTM cell written out in torch (lstm_states), the random-negative loss and its four gradients by autograd
(loss_and_grads), the impression loss (impression_loss_and_grads) and the evaluation windows of impression_states (window_states).
Adam is user_gru_oracle.adam_tf.

Kernels: cell_fwd / cell_bwd return (value, scale) per output, and a kernel passes when |got - want| <= C_FP32 scale + tiny for
every element (C_FP32 = 2^-20, 16 units of fp32 rounding u = 2^-24), as in gru_kernel_oracle.py.  Every reference starts from the
kernel's own fp32 inputs, taken exact.  With s(a) = 1 / (1 + e^-a):

Cell forward, from XP = [x_i | x_f | x_g | x_o], HP = [h_i | h_f | h_g | h_o] and c_prev:
  i = s(x_i + h_i).  The sum rounds once (u (|x_i| + |h_i|)), which s' = i (1 - i) carries into i; expf, the add and the divide
    add a few u of i itself:                        scale_i = i (1 - i) (|x_i| + |h_i|) + i;  f and o alike.
  g = tanh(x_g + h_g).  The sum rounds once, tanh' = 1 - g^2 carries it, tanhf adds a few u of g:
                                                    scale_g = (1 - g^2) (|x_g| + |h_g|) + |g|.
  c = f c_prev + i g.  The errors of f, i and g enter through |c_prev|, |g| and i; each product and the sum round once:
                                                    scale_c = |c_prev| scale_f + |g| scale_i + i scale_g + |f c_prev| + |i g|.
  h = o tanh(c).  tanh(c) carries c's error through 1 - tanh^2 c and adds a few u of itself; o's error enters through |tanh c|;
    the product rounds once:                        scale_h = |tanh c| scale_o + o ((1 - tanh^2 c) scale_c + |tanh c|) + |h|.
  The stored gates [i | f | g | o] carry the scales of i, f, g, o.  The next step's operand is the bf16 split of the kernel's own
  fp32 h_out, bit for bit.

Cell backward, from the stored gates (i, f, g, o), c_t, c_{t-1}, the two carries and dh_in (all exact inputs).
  dh = carry_h + dh_in rounds once:                 D = |carry_h| + |dh_in|.
  T = tanhf(c_t) is within a few u of tanh(c_t), so 1 - T^2 has an ABSOLUTE error of a few u (1 + T^2) (it cancels near |T| = 1);
  dc = carry_c + dh o (1 - T^2):                    scale_dc = |carry_c| + D o (1 + T^2).
  do = dh T o (1 - o) (1 - o is exact for o >= 1/2 and rounds by u |1 - o| below):
                                                    scale_do = D |T| o (1 - o);
  di = dc g i (1 - i), dc's error included:         scale_di = scale_dc |g| i (1 - i);
  df = dc c_{t-1} f (1 - f):                        scale_df = scale_dc |c_{t-1}| f (1 - f);
  dg = dc i (1 - g^2), 1 - g^2 with an absolute error of a few u (1 + g^2):
                                                    scale_dg = scale_dc i (1 + g^2);
  carry_c <- dc f:                                  scale = scale_dc f.
  Each is a product of at most six correctly rounded factors and one inherited error: under 8 u of its scale.  dA = [di | df | dg |
  do] is compared as bf16 hi + lo, with gru_kernel_oracle.check_pair's extra 2^-17 |v| for the split and the hi = rn(hi + lo) check.
"""
import numpy as np
import torch

from gru_kernel_oracle import sigmoid
from user_gru_oracle import NAMES  # noqa: F401  (torch.nn.LSTM uses the same names)


# ---------------------------------------------------------------------------------------------------------------------------
# whole batches
# ---------------------------------------------------------------------------------------------------------------------------
def lstm_states(params, seqs, emb, cells=False):
    """h of every user: list of [L_u, H] tensors (fp64, differentiable in params); with cells=True also the list of c.  seqs: list
    of item arrays (already truncated); params: dict of fp64 tensors with torch.nn.LSTM's names."""
    Wi, Wh, bi, bh = (params[n] for n in NAMES)
    H = Wh.shape[1]
    E = torch.as_tensor(np.asarray(emb, np.float64))
    hs_all, cs_all = [], []
    for s in seqs:
        h = torch.zeros(H, dtype=torch.float64)
        c = torch.zeros(H, dtype=torch.float64)
        hs, cs = [], []
        for a in s:
            z = Wi @ E[int(a)] + bi + Wh @ h + bh
            i, f = torch.sigmoid(z[:H]), torch.sigmoid(z[H:2 * H])
            g, o = torch.tanh(z[2 * H:3 * H]), torch.sigmoid(z[3 * H:])
            c = f * c + i * g
            h = o * torch.tanh(c)
            hs.append(h)
            cs.append(c)
        empty = torch.zeros(0, H, dtype=torch.float64)
        hs_all.append(torch.stack(hs) if hs else empty)
        cs_all.append(torch.stack(cs) if cs else empty)
    return (hs_all, cs_all) if cells else hs_all


def _leaf(params_np):
    return {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in params_np.items()}


def rank_loss(hs, seqs, negs, emb):
    """Mean over every (user, t < L - 1) of softplus(h_t . e(neg) - h_t . e(a_{t+1})), from the states hs (any differentiable
    tensors)."""
    E = torch.as_tensor(np.asarray(emb, np.float64))
    terms = []
    for h, s, ng in zip(hs, seqs, negs):
        if len(s) < 2:
            continue
        ht = h[:-1]
        sp_ = (ht * E[torch.as_tensor(np.asarray(s[1:], np.int64))]).sum(1)
        sn = (ht * E[torch.as_tensor(np.asarray(ng, np.int64))]).sum(1)
        terms.append(torch.nn.functional.softplus(sn - sp_))
    return torch.cat(terms).mean()


def loss_and_grads(params_np, seqs, negs, emb):
    """The random-negative loss of UserLSTM's batch (negs: per user an array of L - 1 negatives).  Returns (loss, {name: grad},
    states)."""
    params = _leaf(params_np)
    hs = lstm_states(params, seqs, emb)
    loss = rank_loss(hs, seqs, negs, emb)
    loss.backward()
    return float(loss.detach()), {k: v.grad.numpy() for k, v in params.items()}, [h.detach().numpy() for h in hs]


def impression_loss_and_grads(params_np, seqs, emb, imps):
    """Mean over the impressions of 1 / (|C| |N|) sum softplus(h_t . e_n - h_t . e_c), h_t the state after read t + 1 of a packed
    user's window.  imps: list of (user index, t, items, clicked).  Returns (loss, {name: grad})."""
    params = _leaf(params_np)
    E = torch.as_tensor(np.asarray(emb, np.float64))
    hs = lstm_states(params, seqs, emb)
    terms = []
    for i, t, it, c in imps:
        c = np.asarray(c).astype(bool)
        s = E[torch.as_tensor(np.asarray(it, np.int64))] @ hs[i][t]
        x = s[torch.from_numpy(~c)][None, :] - s[torch.from_numpy(c)][:, None]
        terms.append(torch.nn.functional.softplus(x).mean())
    loss = torch.stack(terms).mean()
    loss.backward()
    return float(loss.detach()), {k: v.grad.numpy() for k, v in params.items()}


def window_states(params_np, indptr, items, user, time, emb, max_len):
    """[I, H]: h after the last min(time, max_len) reads before each impression; zero at time = 0."""
    params = {k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in params_np.items()}
    H = params['weight_hh_l0'].shape[1]
    out = np.zeros((len(user), H))
    seqs = [items[indptr[u] + max(0, t - max_len):indptr[u] + t] for u, t in zip(user, time)]
    for i, h in enumerate(lstm_states(params, seqs, emb)):
        if len(h):
            out[i] = h[-1].numpy()
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# cell kernels
# ---------------------------------------------------------------------------------------------------------------------------
def lstm_edge_inputs(rng, n, H):
    """fp32 XP, HP [n x 4H] and c_prev [n x H] reaching the cell's edges: pre-activations from -30 to 30 (row 0 sweeps them), g = +-1
    in fp32 (row 1), |c| large enough that tanh c = +-1 in fp32 (row 2), c_prev = 0 (row 3), f c_prev cancelling i g (row 4)."""
    f32 = np.float32
    xp = (rng.standard_normal((n, 4 * H)) * rng.choice([0.3, 3.0, 15.0], (n, 1))).astype(f32)
    hp = (rng.standard_normal((n, 4 * H)) * rng.choice([0.3, 3.0, 15.0], (n, 1))).astype(f32)
    cprev = (rng.standard_normal((n, H)) * rng.choice([0.1, 2.0, 20.0], (n, 1))).astype(f32)
    xp[0] = np.linspace(-30, 30, 4 * H, dtype=f32)
    hp[0] = 0
    if n > 1:
        xp[1, 2 * H:3 * H] = 30.0 * np.sign(rng.standard_normal(H)).astype(f32)
        hp[1, 2 * H:3 * H] = 0
    if n > 2:
        cprev[2] = 40.0 * np.sign(rng.standard_normal(H)).astype(f32)
        xp[2, H:2 * H], hp[2, H:2 * H] = 30.0, 0.0                      # f = 1
    if n > 3:
        cprev[3] = 0
    if n > 4:                                                           # i = f = 1 - tiny, g = -c_prev: c close to 0
        xp[4, :2 * H], hp[4, :2 * H] = 30.0, 0.0
        g = np.tanh(xp[4, 2 * H:3 * H].astype(np.float64) + hp[4, 2 * H:3 * H])
        cprev[4] = (-g).astype(f32)
    return np.clip(xp, -30, 30), np.clip(hp, -30, 30), cprev


def cell_fwd(xp, hp, c_prev, H):
    """One forward step for every row of xp / hp [n x >= 4H] and c_prev [n x H] (None: 0).  Returns {name: (value, scale)} for
    i, f, g, o, c and h."""
    xp = np.asarray(xp, np.float64)[:, :4 * H]
    hp = np.asarray(hp, np.float64)[:, :4 * H]
    cp = np.zeros((xp.shape[0], H)) if c_prev is None else np.asarray(c_prev, np.float64)[:, :H]
    out = {}
    for k, name in enumerate('ifgo'):
        x, a = xp[:, k * H:(k + 1) * H], hp[:, k * H:(k + 1) * H]
        if name == 'g':
            v = np.tanh(x + a)
            out[name] = (v, (1.0 - v * v) * (np.abs(x) + np.abs(a)) + np.abs(v))
        else:
            v = sigmoid(x + a)
            out[name] = (v, v * (1.0 - v) * (np.abs(x) + np.abs(a)) + v)
    (i, s_i), (f, s_f), (g, s_g), (o, s_o) = (out[k] for k in 'ifgo')
    c = f * cp + i * g
    s_c = np.abs(cp) * s_f + np.abs(g) * s_i + i * s_g + np.abs(f * cp) + np.abs(i * g)
    tc = np.tanh(c)
    h = o * tc
    s_h = np.abs(tc) * s_o + o * ((1.0 - tc * tc) * s_c + np.abs(tc)) + np.abs(h)
    out['c'], out['h'] = (c, s_c), (h, s_h)
    return out


def cell_bwd(dh_in, carry_h, carry_c, gates, c, c_prev, H):
    """One backward step from the stored gates [n x >= 4H] = [i | f | g | o], c_t, c_{t-1} (None: 0), the two carries and dh_in
    (None: 0).  Returns {name: (value, scale)} for di, df, dg, do, 'carry_c' (dc f) and 'dc'."""
    gt = np.asarray(gates, np.float64)
    i, f, g, o = (gt[:, k * H:(k + 1) * H] for k in range(4))
    ch = np.asarray(carry_h, np.float64)[:, :H]
    cc = np.asarray(carry_c, np.float64)[:, :H]
    di_ = np.zeros_like(ch) if dh_in is None else np.asarray(dh_in, np.float64)[:, :H]
    cp = np.zeros_like(ch) if c_prev is None else np.asarray(c_prev, np.float64)[:, :H]
    T = np.tanh(np.asarray(c, np.float64)[:, :H])
    dh, D = ch + di_, np.abs(ch) + np.abs(di_)
    dc = cc + dh * o * (1.0 - T * T)
    s_dc = np.abs(cc) + D * o * (1.0 + T * T)
    return {'di': (dc * g * i * (1.0 - i), s_dc * np.abs(g) * i * (1.0 - i)),
            'df': (dc * cp * f * (1.0 - f), s_dc * np.abs(cp) * f * (1.0 - f)),
            'dg': (dc * i * (1.0 - g * g), s_dc * i * (1.0 + g * g)),
            'do': (dh * T * o * (1.0 - o), D * np.abs(T) * o * (1.0 - o)),
            'carry_c': (dc * f, s_dc * f),
            'dc': (dc, s_dc)}
