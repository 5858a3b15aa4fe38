"""The DAE's article encoder as a trainable input of the user encoders (DESIGN 4.19): user_model.ArticleEncoder, its device copy of
the articles, its own [W | bh] and optimizer state, the per-batch compact table of touched articles and the encoder's forward and
backward over it."""
import numpy as np
import torch

from . import _cabi
from ._cabi import call


def _stream():
    return torch.cuda.current_stream().cuda_stream


ARTICLE_LEARNING_RATE = 1e-3   # ArticleEncoder's default learning rate (Adam): the smallest of 1e-4, 1e-3, 1e-2 at the best AUC (DESIGN 4.19)
ARTICLE_ENCODE_GROUPS = 1       # thread groups per row of every ArticleEncoder encode, training batches and vectors() alike


class ArticleEncoder:
    """The DAE's encoder e(x) = f(in_scale x W + bh) - f(bh) over a fixed set of articles, as a trainable input of the user encoders
    (DESIGN 4.19).  X: the articles' bag-of-words rows [N, F] (scipy sparse or dense; a device copy is kept); params: the DAE's
    parameters (get_model_parameters(): 'enc_w' [F, H] and 'enc_b' [H], or state_dict()'s 'enc-w' / 'hidden-bias'); enc_act_func:
    the DAE's f ('sigmoid', 'tanh', anything else the identity); in_scale: the input scaling, 1 - corr_frac for a masking-noise
    DAE, as decay_noise before transform.  The encoder keeps its own fp32 [W | bh], gradient and optimizer slots (opt, learning_rate:
    None for ARTICLE_LEARNING_RATE, momentum, steps): the DAE object is never modified; its decoder is not part of this.

    UserGRU / UserLSTM / UserAttention.fit(sequences, art, ...) trains theta and [W | bh] on the same loss; every other entry point
    (transform, impression_states, recommend, helpers.impression_metrics) takes art where it takes embeddings and reads
    art.vectors()."""

    def __init__(self, X, params, enc_act_func='tanh', in_scale=1.0, opt='adam', learning_rate=None, momentum=0.5, device='cuda:0'):
        import scipy.sparse as sp
        from .engine import DeviceCSR, canonical_csr
        m = canonical_csr(X if sp.issparse(X) else np.asarray(X, dtype=np.float32)).astype(np.float32)
        N, F = m.shape
        W = params['enc-w'] if 'enc-w' in params else params.get('enc_w')
        bh = params['hidden-bias'] if 'hidden-bias' in params else params.get('enc_b')
        if W is None or bh is None:
            raise ValueError("ArticleEncoder: params must hold 'enc_w' and 'enc_b' (or 'enc-w' and 'hidden-bias')")
        W = W.detach().cpu().numpy() if isinstance(W, torch.Tensor) else np.asarray(W)
        bh = bh.detach().cpu().numpy() if isinstance(bh, torch.Tensor) else np.asarray(bh)
        if W.ndim != 2 or W.shape[0] != F or W.shape[1] < 1:
            raise ValueError('ArticleEncoder: W has shape %s, [F = %d, H] expected for the articles\' %d features' % (W.shape, F, F))
        H = int(W.shape[1])
        if bh.shape != (H,):
            raise ValueError('ArticleEncoder: the hidden bias has shape %s, (%d,) expected' % (bh.shape, H))
        if N < 2:
            raise ValueError('ArticleEncoder: at least 2 articles are needed')
        if opt not in _cabi.OPT:
            raise ValueError('ArticleEncoder: opt = %r, one of %s' % (opt, sorted(_cabi.OPT)))
        lr = ARTICLE_LEARNING_RATE if learning_rate is None else float(learning_rate)
        if not lr >= 0.0:
            raise ValueError('ArticleEncoder: learning_rate = %r must be >= 0' % (learning_rate,))
        self.n, self.F, self.dim = int(N), int(F), H
        self.enc_act_func, self.in_scale = enc_act_func, float(in_scale)
        self.opt, self.learning_rate, self.momentum = opt, lr, float(momentum)
        self.device = torch.device(device)
        self.steps = 0
        self.csr = DeviceCSR(m, self.device)
        self.theta = torch.from_numpy(np.concatenate([W.astype(np.float32).ravel(), bh.astype(np.float32)])).to(self.device)
        self.grad = torch.zeros_like(self.theta)
        self.slot1 = torch.full_like(self.theta, 0.1 if opt == 'ada_grad' else 0.0)
        self.slot2 = torch.zeros_like(self.theta)
        self._tag = torch.zeros(N, dtype=torch.int64, device=self.device)    # dae_touch_compact's stamps
        self._slot_of = torch.empty(N, dtype=torch.int32, device=self.device)
        self._stamp = 0

    @property
    def W(self):
        """W [F, H] fp32 on the device (a view: writing it changes the encoder)."""
        return self.theta[:self.F * self.dim].view(self.F, self.dim)

    @property
    def bh(self):
        return self.theta[self.F * self.dim:]

    def state_dict(self):
        """{'enc-w': [F, H], 'hidden-bias': [H]} (CPU fp32 tensors): the reference checkpoint's names."""
        return {'enc-w': self.W.cpu().clone(), 'hidden-bias': self.bh.cpu().clone()}

    def save(self, path):
        np.savez(path, **{k: v.numpy() for k, v in self.state_dict().items()}, enc_act_func=self.enc_act_func, in_scale=self.in_scale,
                 opt=self.opt, learning_rate=self.learning_rate, momentum=self.momentum)

    @classmethod
    def load(cls, path, X, **kw):
        """An encoder over the articles X from save()'s .npz; keyword arguments as the constructor's override the file's."""
        z = np.load(path)
        for k in ('enc_act_func', 'opt'):
            kw.setdefault(k, str(z[k]))
        for k in ('in_scale', 'learning_rate', 'momentum'):
            kw.setdefault(k, float(z[k]))
        return cls(X, {'enc-w': z['enc-w'], 'hidden-bias': z['hidden-bias']}, **kw)

    def _encode(self, csr, rows, n, E, col_count=None):
        call('dae_encode_csr_fwd_groups', csr.indptr.data_ptr(), csr.indices.data_ptr(), csr.values.data_ptr(),
             None if rows is None else rows.data_ptr(), n, self.F, self.dim, self.in_scale, self.W.data_ptr(), self.bh.data_ptr(),
             _cabi.act_code(self.enc_act_func), E.data_ptr(), E.stride(0), None if col_count is None else col_count.data_ptr(), None,
             None, 0, ARTICLE_ENCODE_GROUPS, _stream())

    def vectors(self, X=None, to_host=True):
        """Article vectors [N, H] fp32 with the current W and bh: of the encoder's own articles, or of X (any rows with the same F:
        articles never seen in training included).  A row's vector is bit-identical to its row of a training batch's table."""
        from .engine import DeviceCSR
        csr = self.csr
        if X is not None:
            csr = DeviceCSR(X, self.device)
            if csr.shape[1] != self.F:
                raise ValueError('ArticleEncoder.vectors: X has %d features, the encoder %d' % (csr.shape[1], self.F))
        out = torch.empty(csr.shape[0], self.dim, dtype=torch.float32, device=self.device)
        self._encode(csr, None, csr.shape[0], out)
        return out.cpu().numpy() if to_host else out

    # ---- one joint training batch -----------------------------------------------------------------------------------------
    def touch(self, ids):
        """The batch's compact table: ids (int32 device, article ids, -1: none) -> (rows int32 [T], slots int32 like ids, T)."""
        n = ids.numel()
        self._stamp += 1
        rows = torch.empty(n, dtype=torch.int32, device=self.device)
        slots = torch.empty_like(ids)
        ws = torch.empty(int(_cabi.query('dae_touch_compact_workspace', n)), dtype=torch.int32, device=self.device)
        call('dae_touch_compact', ids.data_ptr(), n, self._stamp, self._tag.data_ptr(), self._slot_of.data_ptr(), rows.data_ptr(),
             slots.data_ptr(), ws.data_ptr(), _stream())
        T = int(ws[0].item())   # sizes the encode launch: one device-to-host read per batch
        return rows[:T], slots, T

    def encode_rows(self, rows, T):
        """E_t [T, H] of the listed articles and the per-column entry counts the backward needs."""
        E = torch.empty(T, self.dim, dtype=torch.float32, device=self.device)
        col_count = torch.empty(self.F, dtype=torch.int32, device=self.device)
        self._encode(self.csr, rows, T, E, col_count)
        return E, col_count

    def backward(self, rows, T, E, dE, col_count, deterministic=False):
        """grad = [dW | dbh] of the listed articles' gradient dE [T, H] (overwritten with dA), by dae_encode_csr_bwd_gather, or with
        deterministic=True by dae_encode_csr_bwd_det and dae_encode_sparse_dw_add onto a zeroed dW (DESIGN 4.21); the latter's
        workspace size is kept in det_workspace_bytes."""
        F, H, i32 = self.F, self.dim, dict(dtype=torch.int32, device=self.device)
        cap = max(1, min(self.csr.nnz, T * self.csr.max_row_nnz))
        if deterministic:
            nb = _cabi.query('dae_encode_csr_bwd_det_workspace', T, F, H, cap)
            self.det_workspace_bytes = nb
            ws = torch.empty(nb, dtype=torch.uint8, device=self.device)
            call('dae_encode_csr_bwd_det', self.csr.indptr.data_ptr(), self.csr.indices.data_ptr(), self.csr.values.data_ptr(),
                 rows.data_ptr(), T, F, H, self.in_scale, E.data_ptr(), self.bh.data_ptr(), _cabi.act_code(self.enc_act_func),
                 dE.data_ptr(), None, H, self.grad[F * H:].data_ptr(), col_count.data_ptr(), cap, ws.data_ptr(), nb, _stream())
            self.grad[:F * H].zero_()
            call('dae_encode_sparse_dw_add', T, F, H, cap, ws.data_ptr(), nb, self.grad.data_ptr(), _stream())
            return
        col_start, col_cursor = torch.empty(F + 1, **i32), torch.empty(F, **i32)
        ent_col, ent_row = torch.empty(cap, **i32), torch.empty(cap, **i32)
        ent_val = torch.empty(cap, dtype=torch.float32, device=self.device)
        self.grad[:F * H].zero_()
        call('dae_encode_csr_bwd_gather', self.csr.indptr.data_ptr(), self.csr.indices.data_ptr(), self.csr.values.data_ptr(),
             rows.data_ptr(), T, F, H, self.in_scale, E.data_ptr(), self.bh.data_ptr(), _cabi.act_code(self.enc_act_func), dE.data_ptr(),
             None, H, self.grad.data_ptr(), self.grad[F * H:].data_ptr(), 0, col_count.data_ptr(), col_start.data_ptr(),
             col_cursor.data_ptr(), ent_col.data_ptr(), ent_row.data_ptr(), ent_val.data_ptr(), _stream())

    def scatter_rows(self, src, slots, dE):
        """dE[slots[p]] += src[p] for every row p of src (dae_rows_scatter_add)."""
        call('dae_rows_scatter_add', src.data_ptr(), src.stride(0), slots.data_ptr(), src.shape[0], self.dim, dE.data_ptr(), dE.stride(0),
             _stream())

    def ordered_rows(self, trip, src, dX, slots, T, dE):
        """dE [T, H] (stored) = per slot, the loss kernels' triples trip = (slot, row, coefficient) over the rows of src in triple
        order, then dX[p] for every p with slots[p] = the slot, in p order (dae_ordered_rows)."""
        t_slot, t_row, t_coef = trip
        n_a, n_b = t_slot.numel(), dX.shape[0]
        ws = torch.empty(max(1, _cabi.query('dae_ordered_rows_workspace', n_a, n_b, T)), dtype=torch.uint8, device=self.device)
        call('dae_ordered_rows', t_slot.data_ptr(), t_row.data_ptr(), t_coef.data_ptr(), n_a, src.data_ptr(), src.stride(0),
             slots.data_ptr(), n_b, dX.data_ptr(), dX.stride(0), T, self.dim, dE.data_ptr(), dE.stride(0), ws.data_ptr(), ws.numel(),
             _stream())

    def step(self):
        """One dense dae_optimizer_step of [W | bh] (torch.optim semantics)."""
        self.steps += 1
        call('dae_optimizer_step', self.theta.data_ptr(), self.grad.data_ptr(), self.slot1.data_ptr(), self.slot2.data_ptr(),
             self.theta.numel(), _cabi.OPT[self.opt], self.learning_rate, self.momentum, 1.0, self.steps, None, None, None, 0, 0, 0,
             _stream())
