"""Block oracles for batch_all / batch_hard at batch sizes where no B x B tensor fits (test infrastructure, NOT product code).

`dae_oracle.batch_hard_triplet_loss` and `chunked_oracle._batch_hard_on` materialise several B x B tensors, and
`chunked_oracle.batch_all_triplet_loss_chunked` builds S = E.E^T and G as B x B.  The functions here have the same semantics
(triplet_loss_utils.py:79-131 and :202-259) but only ever hold one block of anchor rows of S.  Instead of G they return
C = dL/dE = (G + G^T) E, accumulated block by block, and their loss differentiates into E through the surrogate (E * C).sum().  They run
in any dtype on any torch device with plain torch ops; they do not call this project's kernels.

`BlockOracleDAE` is `chunked_oracle.ChunkedOracleDAE` with both strategies mined by these functions.
"""
import numpy as np
import torch

from oracle.chunked_oracle import ChunkedOracleDAE
from oracle.dae_oracle import EPS, decode, encode, weighted_loss, _as_dense


def _with_surrogate(value, E, C):
    """value (a plain number) that differentiates into E as C: d/dE (E * C).sum() = C."""
    if E is None or not E.requires_grad:
        return value
    s = (E * C).sum()
    return value + s - s.detach()


def batch_hard_triplet_loss_chunked(labels, E, block_rows=4096):
    """-> (loss, w, fraction, num, C).  Per anchor row a: m = max_c S_ac, hp = min_c (S_ac + m (1 - ap_ac)), hn = max_c an_ac S_ac,
    td = max(hn - hp, 0), active = td > 0; loss = sum softplus(td) over active rows / (num + eps).  dL/dS comes from torch.amin / amax
    autograd on each block's rows of S, so ties share the gradient as with TF's reduce_min / reduce_max.  w = the data weights
    (active + equality counts of S against each active row's hp / hn, summed over the rows), num = number of active rows."""
    dev, Ed = E.device, E.detach()
    lab = torch.as_tensor(labels).reshape(-1).to(dev)
    B = Ed.shape[0]
    cols = torch.arange(B, device=dev)
    w = torch.zeros(B, dtype=torch.float64, device=dev)
    C = torch.zeros_like(Ed)
    loss_sum = torch.zeros((), dtype=Ed.dtype, device=dev)
    num = 0.0
    for r0 in range(0, B, block_rows):
        A = cols[r0:r0 + block_rows]
        with torch.enable_grad():
            s = (Ed[A] @ Ed.t()).requires_grad_(True)                    # [n, B]: rows A of S
            same = lab[A][:, None] == lab[None, :]
            ap = ((A[:, None] != cols[None, :]) & same).to(Ed.dtype)
            an = (~same).to(Ed.dtype)
            m = torch.amax(s, 1, keepdim=True)
            hp = torch.amin(s + m * (1.0 - ap), 1, keepdim=True)
            hn = torch.amax(an * s, 1, keepdim=True)
            td = torch.clamp(hn - hp, min=0.0)
            c = (td > 0.0).to(Ed.dtype)
            part = (torch.nn.functional.softplus(td) * c).sum()
            g, = torch.autograd.grad(part, s)
        sd = s.detach()
        w[A] += c.squeeze(1).double()
        w += (c * (sd == hp.detach()).to(Ed.dtype)).sum(0).double() + (c * (sd == hn.detach()).to(Ed.dtype)).sum(0).double()
        C[A] += g @ Ed                 # G_blk . E       -> the block's rows
        C += g.t() @ Ed[A]             # G_blk^T . E_blk -> every row
        loss_sum = loss_sum + part.detach()
        num += float(c.sum())
        del s, sd, g, same, ap, an
    inv = 1.0 / (num + EPS)
    C = C * inv
    return _with_surrogate(loss_sum * inv, E, C), w.to(Ed.dtype), num / float(B), num, C


def batch_all_triplet_loss_block(labels, E, block_elems=1 << 25):
    """-> (loss, w, fraction, num, C), the values of chunked_oracle.batch_all_triplet_loss_chunked with C = (G + G^T) E in place of
    G: for each class and each block of its anchors only the |P| x |N| block of softplus(S_ik - S_ij) is formed, from the rows of E."""
    dev, Ed = E.device, E.detach()
    lab = torch.as_tensor(labels).reshape(-1).to(dev)
    B = Ed.shape[0]
    w = torch.zeros(B, dtype=torch.float64, device=dev)
    C = torch.zeros_like(Ed)
    loss_sum = torch.zeros((), dtype=Ed.dtype, device=dev)
    n_valid = n_pos = 0
    for cl in torch.unique(lab):
        P_all = torch.nonzero(lab == cl).flatten()
        N = torch.nonzero(lab != cl).flatten()
        npc, nn = P_all.numel(), N.numel()
        if npc < 2 or nn == 0:
            continue
        EP, EN = Ed[P_all], Ed[N]
        step = max(1, block_elems // (npc * nn))
        for a0 in range(0, npc, step):
            A = P_all[a0:a0 + step]
            na = A.numel()
            with torch.enable_grad():
                s_p = (Ed[A] @ EP.t()).requires_grad_(True)            # [na, |P|]   S_ij
                s_n = (Ed[A] @ EN.t()).requires_grad_(True)            # [na, |N|]   S_ik
                d = s_n[:, None, :] - s_p[:, :, None]
                valid = (P_all[None, :] != A[:, None])[:, :, None].expand(na, npc, nn)
                pos = valid & (d.detach() > 1e-16)
                mask = valid.to(Ed.dtype)
                part = (torch.nn.functional.softplus(d) * mask).sum()
                gp, gn = torch.autograd.grad(part, (s_p, s_n))
            n_valid += int(valid.sum())
            n_pos += int(pos.sum())
            loss_sum = loss_sum + part.detach()
            C[A] += gp @ EP + gn @ EN
            C.index_add_(0, P_all, gp.t() @ Ed[A])
            C.index_add_(0, N, gn.t() @ Ed[A])
            m64 = mask.to(torch.float64)
            w.index_add_(0, A, m64.sum((1, 2)))
            w.index_add_(0, P_all, m64.sum((0, 2)))
            w.index_add_(0, N, m64.sum((0, 1)))
            del d, mask, m64, valid, pos, s_p, s_n
    inv = 1.0 / (n_valid + EPS)
    C = C * inv
    return _with_surrogate(loss_sum * inv, E, C), w.to(Ed.dtype), n_pos / (n_valid + EPS), n_pos, C


class BlockOracleDAE(ChunkedOracleDAE):
    """ChunkedOracleDAE whose batch_all and batch_hard never hold a B x B tensor (block_rows: batch_hard's anchor rows per block)."""

    def __init__(self, W0, bh0=None, bv0=None, device='cpu', block_rows=4096, **kw):
        super().__init__(W0, bh0, bv0, device=device, **kw)
        self.block_rows = int(block_rows)

    def forward(self, x, xc, labels=None):
        if self.triplet_strategy == 'none':
            return super().forward(x, xc, labels)
        xd = _as_dense(x, self.dtype).to(self.device)
        E = encode(self._sparse_or_dense(xc), self.W, self.bh, self.enc_act_func)
        D = decode(E, self.W, self.bv, self.dec_act_func)
        lab = torch.from_numpy(np.asarray(labels, dtype=np.float32).reshape(-1)).to(self.device)
        if self.triplet_strategy == 'batch_all':
            tl, w, frac, num, _ = batch_all_triplet_loss_block(lab, E)
        else:
            tl, w, frac, num, _ = batch_hard_triplet_loss_chunked(lab, E, self.block_rows)
        w = w.detach()
        ael = weighted_loss(xd, D, self.loss_func, w)
        return {'encode': E, 'decode': D, 'triplet_loss': tl, 'autoencoder_loss': ael, 'cost': ael + self.alpha * tl,
                'fraction': frac, 'num': num, 'weight': w}
