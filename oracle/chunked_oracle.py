"""Chunked batch_all oracle (test infrastructure, NOT product code).

`dae_oracle.batch_all_triplet_loss` materialises the reference's B x B x B tensors, which stops at a few thousand rows.  The
function here has the same semantics (triplet_loss_utils.py:79-131) but never holds more than a block of anchors of one class at a
time: for each anchor i it forms only the |P| x |N| block of softplus(S_ik - S_ij) (P = same label, j != i; N = other labels),
and it takes G = dL/dS for those anchors by autograd on the block.  It runs in any dtype on any torch device -- the GPU tests run it in
fp64 with plain torch ops on the GPU; it does not call this project's kernels.

`ChunkedOracleDAE` is `dae_oracle.OracleDAE` on a torch device, with batch_all mined by the chunked function
(batch_all='chunked', the default) or by the materialising one (batch_all='materialise').
"""
import numpy as np
import scipy.sparse as sp
import torch

from oracle.dae_oracle import (EPS, OracleDAE, batch_all_triplet_loss, decode, encode, to_torch_sparse, weighted_loss,
                               _as_dense)


def batch_all_triplet_loss_chunked(labels, E, pos_triplets_only=False, device=None, block_elems=1 << 25, S=None):
    """-> (loss, w, fraction, num, G).  loss is a 0-d tensor that differentiates into E like the materialising oracle's (through
    S = E.E^T and G); w[B] are the data weights (mask sums over the three triplet axes), fraction = num / N_valid, num = number of
    positive triplets ((S_ik - S_ij) > 1e-16), G [B x B] = d loss / d S.  block_elems bounds anchors x |P| x |N| per block.
    S (optional): mine this similarity matrix instead of E.E^T (E may then be None; loss is a plain value)."""
    if S is None:
        dev = torch.device(device) if device is not None else E.device
        Ed = E.detach().to(dev)
        S = Ed @ Ed.t()
    else:
        dev = torch.device(device) if device is not None else S.device
        S = S.detach().to(dev)
        Ed = S
        E = None
    lab = torch.as_tensor(labels).reshape(-1).to(dev)
    B = S.shape[0]
    G = torch.zeros(B, B, dtype=Ed.dtype, device=dev)
    w = torch.zeros(B, dtype=torch.float64, device=dev)
    loss_sum = torch.zeros((), dtype=Ed.dtype, device=dev)
    n_valid = 0
    n_pos = 0
    for c in torch.unique(lab):
        P_all = torch.nonzero(lab == c).flatten()
        N = torch.nonzero(lab != c).flatten()
        npc, nn = P_all.numel(), N.numel()
        if npc < 2 or nn == 0:
            continue
        step = max(1, block_elems // (npc * nn))
        for a0 in range(0, npc, step):
            A = P_all[a0:a0 + step]
            na = A.numel()
            s_p = S[A][:, P_all].clone().requires_grad_(True)      # [na, |P|]   S_ij
            s_n = S[A][:, N].clone().requires_grad_(True)          # [na, |N|]   S_ik
            d = s_n[:, None, :] - s_p[:, :, None]                  # [na, |P|, |N|]   S_ik - S_ij
            not_self = (P_all[None, :] != A[:, None])              # j != i
            valid = not_self[:, :, None].expand(na, npc, nn)
            pos = valid & (d.detach() > 1e-16)
            n_valid += int(valid.sum())
            n_pos += int(pos.sum())
            mask = (pos if pos_triplets_only else valid).to(Ed.dtype)
            part = (torch.nn.functional.softplus(d) * mask).sum()
            gp, gn = torch.autograd.grad(part, (s_p, s_n))
            loss_sum = loss_sum + part.detach()
            G[A[:, None], P_all[None, :]] = gp
            G[A[:, None], N[None, :]] = gn
            m64 = mask.to(torch.float64)
            w.index_add_(0, A, m64.sum((1, 2)))                     # as anchor
            w.index_add_(0, P_all, m64.sum((0, 2)))                 # as positive
            w.index_add_(0, N, m64.sum((0, 1)))                     # as negative
            del d, mask, m64, valid, pos
    n = n_pos if pos_triplets_only else n_valid
    inv = 1.0 / (n + EPS)
    G = G * inv
    value = loss_sum * inv
    if E is not None and E.requires_grad:      # d loss / d E = (G + G^T) E through S = E.E^T, the value stays the chunked sum
        Sg = E.to(dev) @ E.to(dev).t()
        surrogate = (Sg * G).sum()
        loss = value + surrogate - surrogate.detach()
    else:
        loss = value
    frac = n_pos / (n_valid + EPS)
    return loss, w.to(Ed.dtype), frac, n_pos, G


class ChunkedOracleDAE(OracleDAE):
    """OracleDAE whose parameters, data and arithmetic live on `device`; batch_all='chunked' mines with the chunked function."""

    def __init__(self, W0, bh0=None, bv0=None, device='cpu', batch_all='chunked', dtype=torch.float64, **kw):
        super().__init__(W0, bh0, bv0, dtype=dtype, **kw)
        assert batch_all in ('chunked', 'materialise')
        self.device = torch.device(device)
        self.batch_all = batch_all
        self.W, self.bh, self.bv = [p.detach().to(self.device).requires_grad_(True) for p in (self.W, self.bh, self.bv)]
        self.slot1 = [s.to(self.device) for s in self.slot1]
        self.slot2 = [s.to(self.device) for s in self.slot2]

    def _sparse_or_dense(self, x):
        if sp.issparse(x):
            return to_torch_sparse(x, self.dtype).to(self.device)
        return _as_dense(x, self.dtype).to(self.device)

    def forward(self, x, xc, labels=None):
        xd = _as_dense(x, self.dtype).to(self.device)
        E = encode(self._sparse_or_dense(xc), self.W, self.bh, self.enc_act_func)
        D = decode(E, self.W, self.bv, self.dec_act_func)
        out = {'encode': E, 'decode': D}
        if self.triplet_strategy == 'none':
            ael = weighted_loss(xd, D, self.loss_func, torch.ones(xd.shape[0], dtype=D.dtype, device=self.device))
            out.update(autoencoder_loss=ael, cost=ael)
            return out
        lab = torch.from_numpy(np.asarray(labels, dtype=np.float32).reshape(-1)).to(self.device)
        if self.triplet_strategy == 'batch_all' and self.batch_all == 'chunked':
            tl, w, frac, num, _ = batch_all_triplet_loss_chunked(lab, E, device=self.device)
        elif self.triplet_strategy == 'batch_all':
            tl, w, frac, num = batch_all_triplet_loss(lab, E)
        else:
            tl, w, frac, num = _batch_hard_on(lab, E)
        w = w.detach()
        ael = weighted_loss(xd, D, self.loss_func, w)
        out.update(triplet_loss=tl, autoencoder_loss=ael, cost=ael + self.alpha * tl, fraction=frac, num=num, weight=w)
        return out

    def step(self, x, xc, labels=None):
        out = self.forward(x, xc, labels)
        g = self.grads(out)
        self.apply_gradients(g)
        res = {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}
        res['grads'] = [t.detach().cpu().numpy() for t in g]
        return res

    def transform(self, data):
        with torch.no_grad():
            return encode(self._sparse_or_dense(data), self.W, self.bh, self.enc_act_func).cpu().numpy()

    def get_parameters(self):
        return {'enc_w': self.W.detach().cpu().numpy().copy(), 'enc_b': self.bh.detach().cpu().numpy().copy(),
                'dec_b': self.bv.detach().cpu().numpy().copy()}


def _batch_hard_on(labels, E):
    """dae_oracle.batch_hard_triplet_loss on E's device (its masks are built on the CPU)."""
    dev = E.device
    S = E @ E.t()
    eye = torch.eye(E.shape[0], dtype=torch.bool, device=dev)
    same = labels[None, :] == labels[:, None]
    ap = ((~eye) & same).to(E.dtype)
    m = torch.amax(S, 1, keepdim=True)
    hp = torch.amin(S + m * (1.0 - ap), 1, keepdim=True)
    an = (~same).to(E.dtype)
    hn = torch.amax(an * S, 1, keepdim=True)
    td = torch.clamp(hn - hp, min=0.0)
    c = (td > 0.0).to(E.dtype)
    w = c.squeeze(1) + (c * (S == hp).to(E.dtype)).sum(0) + (c * (S == hn).to(E.dtype)).sum(0)
    loss = (torch.nn.functional.softplus(td) * c).sum() / (c.sum() + EPS)
    return loss, w, c.sum() / float(labels.shape[0]), c.sum()
