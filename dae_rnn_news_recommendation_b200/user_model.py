"""Learned user vectors: a GRU over each user's reading sequence, trained on the H100 to score the next read above a random
article (DESIGN 4.10).

    m = UserGRU(dim=H, max_len=50, batch_users=1024, num_epochs=5)
    m.fit((indptr, items), embeddings)        # embeddings: [N, H] article vectors (transform()'s output), kept frozen
    U = m.transform((indptr, items), embeddings)            # [U, H] user vectors, score articles by inner product
    idx, score = m.recommend((indptr, items), embeddings, k=10)

Sequences are (indptr int64 [U + 1], items int32 [nnz]): user u read items[indptr[u]:indptr[u + 1]] in that order
(helpers.sequences_from_csr builds them from a matrix of read times).  Only the last max_len reads of a user are used.

The cell is torch.nn.GRU's (one layer, input size = hidden size = H, gate order r, z, n); state_dict() uses its names and shapes, so
a CPU torch.nn.GRU(H, H) loads the parameters.  For a user with reads a_1..a_L and states h_1..h_L the loss has one term per
t < L, softplus(h_t . e(neg_t) - h_t . e(a_{t+1})), averaged over the batch's terms; neg_t is uniform over the other articles
(dae_seq_negatives).  The user vector is the state after the last (truncated) read; a user without reads gets a zero row.

Device path per training batch (users ordered by length, descending, so the users active at step t are rows [0, n_t)):
  dae_seq_negatives; dae_gather_split_bf16 ([X | 1] of every position) and one GEMM for the input projection XP;
  per step a GEMM for HP_t = [h_{t-1} | 1].[W_hh | b_hh]^T and dae_gru_cell_fwd; dae_seq_rank_loss;
  per step in reverse dae_gru_cell_bwd and the carry GEMM dh_{t-1} += dHP_t . W_hh;
  [dW_hh | db_hh] = dHP^T.[h_prev | 1] and [dW_ih | db_ih] = dXP^T.[X | 1] over all positions; dae_optimizer_step.
Parameters: one flat fp32 buffer theta = [W~_hh (3H x (H+1)) | W~_ih (3H x (H+1))] with W~ = [W | b].
"""
import numpy as np
import torch

from . import _cabi
from ._cabi import call

_NAMES = ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _upload(a, device):
    """Host array -> device without waiting: staged through pinned memory, which the caching host allocator keeps until the copy
    has run (an asynchronous copy straight from the NumPy array could read it after it is freed)."""
    return torch.from_numpy(a).pin_memory().to(device, non_blocking=True)


def _ld8(n):
    return (n + 7) // 8 * 8


def check_sequences(sequences, n_items, fn):
    """(indptr, items) as (int64 ndarray, int32 ndarray), or ValueError: indptr must start at 0, never decrease and end at
    len(items); every item must lie in [0, n_items)."""
    try:
        indptr, items = sequences
    except (TypeError, ValueError):
        raise ValueError('%s: sequences must be a pair (indptr, items)' % fn)
    indptr, items = np.asarray(indptr), np.asarray(items)
    if indptr.ndim != 1 or indptr.size < 1 or not np.issubdtype(indptr.dtype, np.integer):
        raise ValueError('%s: indptr must be a 1-D integer array of U + 1 offsets' % fn)
    if items.ndim != 1 or not (np.issubdtype(items.dtype, np.integer) or items.size == 0):
        raise ValueError('%s: items must be a 1-D integer array' % fn)
    if indptr[0] != 0 or indptr[-1] != items.size or (np.diff(indptr) < 0).any():
        raise ValueError('%s: indptr must start at 0, never decrease and end at len(items) = %d' % (fn, items.size))
    if items.size and (items.min() < 0 or items.max() >= n_items):
        raise ValueError('%s: items hold an article outside [0, %d)' % (fn, n_items))
    return indptr.astype(np.int64), items.astype(np.int32)


class Packed:
    """One batch in the PackedSequence layout.  order: the batch's users (ids) by truncated length L, descending (stable), users with
    L = 0 left out; n[t] = users with L > t; off[t] = first position of step t; position off[t] + i is user order[i]'s read t.
    items[p]: the article read at position p; nxt[p]: the article read next (-1 at a user's last position)."""

    def __init__(self, indptr, items, users, max_len):
        users = np.asarray(users, dtype=np.int64)
        L = np.minimum(indptr[users + 1] - indptr[users], max_len)
        keep = L > 0
        users, L = users[keep], L[keep]
        s = np.argsort(-L, kind='stable')
        self.order, self.L = users[s], L[s]
        self.B = int(self.order.size)
        T = int(self.L[0]) if self.B else 0
        self.n = np.searchsorted(-self.L, -np.arange(T), side='left').astype(np.int64)   # #{i: L_i > t}
        self.off = np.concatenate([[0], np.cumsum(self.n)]).astype(np.int64)
        self.P = int(self.off[-1])
        i_all = np.repeat(np.arange(self.B), self.L)
        t_all = np.arange(self.P) - np.repeat(np.cumsum(self.L) - self.L, self.L)
        src = (indptr[self.order + 1] - self.L)[i_all] + t_all
        p = self.off[t_all] + i_all
        self.items = np.empty(self.P, np.int32)
        self.items[p] = items[src]
        self.nxt = np.full(self.P, -1, np.int32)
        more = t_all + 1 < self.L[i_all]
        self.nxt[p[more]] = items[src[more] + 1]
        self.terms = int(more.sum())

    def position(self, i, t):
        return int(self.off[t] + i)


class UserGRU:
    """GRU user encoder over reading sequences; see the module docstring."""

    def __init__(self, dim, max_len=50, batch_users=1024, num_epochs=5, opt='adam', learning_rate=1e-3, seed=0, device='cuda:0',
                 momentum=0.5):
        if dim < 1 or max_len < 1 or batch_users < 1 or num_epochs < 0:
            raise ValueError('UserGRU: dim, max_len and batch_users must be >= 1 and num_epochs >= 0')
        if opt not in _cabi.OPT:
            raise ValueError('UserGRU: opt = %r, one of %s' % (opt, sorted(_cabi.OPT)))
        self.dim, self.max_len, self.batch_users, self.num_epochs = int(dim), int(max_len), int(batch_users), int(num_epochs)
        self.opt, self.learning_rate, self.momentum, self.seed = opt, float(learning_rate), float(momentum), int(seed)
        self.device = torch.device(device)
        self.train_loss = []
        self.steps = 0
        self.epochs_done = 0
        H = self.dim
        self.nW = 3 * H * (H + 1)
        self.ldx, self.ldg = _ld8(H + 1), _ld8(3 * H)
        # torch.nn.GRU's initialisation: every parameter uniform in [-1/sqrt(H), 1/sqrt(H)]
        rng = np.random.default_rng(self.seed)
        k = 1.0 / np.sqrt(H)
        self.theta = torch.from_numpy(rng.uniform(-k, k, 2 * self.nW).astype(np.float32)).to(self.device)
        self.grad = torch.zeros_like(self.theta)
        self.slot1 = torch.full_like(self.theta, 0.1 if opt == 'ada_grad' else 0.0)
        self.slot2 = torch.zeros_like(self.theta)
        bf = dict(dtype=torch.bfloat16, device=self.device)
        self.W_hl = {g: (torch.zeros(3 * H, self.ldx, **bf), torch.zeros(3 * H, self.ldx, **bf)) for g in ('hh', 'ih')}
        self._hh_valid = False
        self._buf = {}
        self._cap = (0, 0)
        self.stats = torch.zeros(1, dtype=torch.float64, device=self.device)
        self.phase_events = None   # a list to record (phase name, CUDA event) pairs into (tools/bench_user_model.py)

    # ---- parameters -------------------------------------------------------------------------------------------------------
    def _theta(self, g):
        """W~_g = [W_g | b_g] as a [3H, H+1] view of theta (g = 'hh' or 'ih')."""
        o = 0 if g == 'hh' else self.nW
        return self.theta[o:o + self.nW].view(3 * self.dim, self.dim + 1)

    def state_dict(self):
        """torch.nn.GRU(H, H)'s parameter names and shapes (CPU fp32 tensors)."""
        ih, hh = self._theta('ih').cpu(), self._theta('hh').cpu()
        H = self.dim
        return {'weight_ih_l0': ih[:, :H].clone(), 'weight_hh_l0': hh[:, :H].clone(), 'bias_ih_l0': ih[:, H].clone(),
                'bias_hh_l0': hh[:, H].clone()}

    def load_state_dict(self, sd):
        H = self.dim
        want = {'weight_ih_l0': (3 * H, H), 'weight_hh_l0': (3 * H, H), 'bias_ih_l0': (3 * H,), 'bias_hh_l0': (3 * H,)}
        missing = set(want) - set(sd)
        if missing:
            raise ValueError('UserGRU.load_state_dict: missing %s' % sorted(missing))
        a = {}
        for name, shape in want.items():
            v = sd[name]
            v = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
            if tuple(v.shape) != shape:
                raise ValueError('UserGRU.load_state_dict: %s has shape %s, %s expected (H = %d)' % (name, tuple(v.shape), shape, H))
            a[name] = v.astype(np.float32)
        for g in ('ih', 'hh'):
            t = np.concatenate([a['weight_%s_l0' % g], a['bias_%s_l0' % g][:, None]], 1)
            self._theta(g).copy_(torch.from_numpy(t))
        self.slot1.fill_(0.1 if self.opt == 'ada_grad' else 0.0)
        self.slot2.zero_()
        self.steps = 0
        self._hh_valid = False

    def save(self, path):
        sd = self.state_dict()
        np.savez(path, max_len=self.max_len, **{k: v.numpy() for k, v in sd.items()})

    @classmethod
    def load(cls, path, **kw):
        """A model from save()'s .npz; keyword arguments as the constructor's (dim and max_len come from the file)."""
        z = np.load(path)
        kw.setdefault('max_len', int(z['max_len']))
        m = cls(int(z['weight_hh_l0'].shape[1]), **kw)
        m.load_state_dict({k: z[k] for k in _NAMES})
        return m

    # ---- device helpers ---------------------------------------------------------------------------------------------------
    def _embeddings(self, embeddings, fn):
        from .helpers import _dense_embeddings
        emb = _dense_embeddings(embeddings, self.device, fn)
        if emb.shape[1] != self.dim:
            raise ValueError('%s: embeddings are %d wide, the model has H = %d' % (fn, emb.shape[1], self.dim))
        if emb.shape[0] < 2:
            raise ValueError('%s: at least 2 articles are needed' % fn)
        return emb

    def _gemm(self, M, N, K, A, a_mn, Bm, b_mn, C, ldc, accumulate=0, k_splits=1):
        (a_hi, a_lo), (b_hi, b_lo) = A, Bm
        call('dae_gemm_bf16x3', M, N, K, 1.0, a_hi.data_ptr(), a_lo.data_ptr(), a_hi.stride(0), a_mn, b_hi.data_ptr(), b_lo.data_ptr(),
             b_hi.stride(0), b_mn, C.data_ptr(), ldc, 0, -1, None, k_splits, accumulate, _stream())

    def _split(self, g):
        hi, lo = self.W_hl[g]
        call('dae_split_bf16', self._theta(g).data_ptr(), 3 * self.dim, self.dim + 1, self.dim + 1, hi.data_ptr(), lo.data_ptr(),
             self.ldx, -1, 1.0, _stream())

    def _mark(self, name):
        if self.phase_events is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.phase_events.append((name, e))

    def _buffers(self, P, B):
        """Training buffers for P positions and B users (grown, never shrunk)."""
        if P <= self._cap[0] and B <= self._cap[1]:
            return self._buf
        P, B = max(P, self._cap[0]), max(B, self._cap[1])
        H, d = self.dim, self.device
        f32, bf, i32 = dict(dtype=torch.float32, device=d), dict(dtype=torch.bfloat16, device=d), dict(dtype=torch.int32, device=d)
        self._buf = None
        torch.cuda.empty_cache()
        b = {'neg': torch.empty(P, **i32),
             'X_hl': (torch.empty(P, self.ldx, **bf), torch.empty(P, self.ldx, **bf)),
             'XP': torch.empty(P, 3 * H, **f32),
             'Hp_hl': (torch.zeros(P, self.ldx, **bf), torch.zeros(P, self.ldx, **bf)),   # [h_{t-1} | 1] of every position
             'HP': torch.empty(B, 3 * H, **f32),
             'Hs': torch.empty(P, H, **f32),
             'gates': torch.empty(P, 4 * H, **f32),
             'dH': torch.empty(P, H, **f32),
             'carry': torch.empty(B, H, **f32),
             'dXP_hl': (torch.empty(P, self.ldg, **bf), torch.empty(P, self.ldg, **bf)),
             'dHP_hl': (torch.empty(P, self.ldg, **bf), torch.empty(P, self.ldg, **bf))}
        b['Hp_hl'][0][:, H] = 1.0
        self._buf, self._cap = b, (P, B)
        return b

    # ---- training ---------------------------------------------------------------------------------------------------------
    def _forward_backward(self, pk, emb, epoch, batch):
        """Loss (added to self.stats) and the gradient (self.grad) of one packed batch with pk.terms > 0."""
        H, P, T = self.dim, pk.P, len(pk.n)
        b = self._buffers(P, pk.B)
        st = _stream()
        items, nxt = _upload(pk.items, self.device), _upload(pk.nxt, self.device)
        if not self._hh_valid:
            self._split('hh')
            self._hh_valid = True
        self._mark('start')
        call('dae_seq_negatives', nxt.data_ptr(), P, emb.shape[0], self.seed, epoch, batch, b['neg'].data_ptr(), st)
        X_hi, X_lo = b['X_hl']
        call('dae_gather_split_bf16', emb.data_ptr(), emb.stride(0), items.data_ptr(), P, H, X_hi.data_ptr(), X_lo.data_ptr(), self.ldx,
             H, st)
        self._split('ih')
        self._gemm(P, 3 * H, H + 1, b['X_hl'], 0, self.W_hl['ih'], 0, b['XP'], 3 * H)
        self._mark('input_projection')
        Hp_hi, Hp_lo = b['Hp_hl']
        n0 = int(pk.n[0])
        Hp_hi[:n0, :H].zero_()
        Hp_lo[:n0].zero_()
        Hs, XP, HP, G = b['Hs'], b['XP'], b['HP'], b['gates']
        for t in range(T):
            o, n = int(pk.off[t]), int(pk.n[t])
            n_next = int(pk.n[t + 1]) if t + 1 < T else 0
            self._gemm(n, 3 * H, H + 1, (Hp_hi[o:], Hp_lo[o:]), 0, self.W_hl['hh'], 0, HP, 3 * H)
            hprev = Hs[int(pk.off[t - 1]):].data_ptr() if t else None
            nx = int(pk.off[t + 1])
            call('dae_gru_cell_fwd', n, H, XP[o:].data_ptr(), 3 * H, HP.data_ptr(), 3 * H, hprev, H, Hs[o:].data_ptr(), H, n_next,
                 Hp_hi[nx:].data_ptr() if n_next else None, Hp_lo[nx:].data_ptr() if n_next else None, self.ldx, G[o:].data_ptr(),
                 4 * H, st)
        self._mark('forward_recurrence')
        call('dae_seq_rank_loss', Hs.data_ptr(), H, emb.data_ptr(), emb.stride(0), H, nxt.data_ptr(), b['neg'].data_ptr(), P,
             1.0 / pk.terms, b['dH'].data_ptr(), H, self.stats.data_ptr(), st)
        self._mark('loss')
        carry, dH = b['carry'], b['dH']
        carry[:n0].zero_()
        (dX_hi, dX_lo), (dP_hi, dP_lo) = b['dXP_hl'], b['dHP_hl']
        for t in range(T - 1, -1, -1):
            o, n = int(pk.off[t]), int(pk.n[t])
            hprev = Hs[int(pk.off[t - 1]):].data_ptr() if t else None
            call('dae_gru_cell_bwd', n, H, dH[o:].data_ptr(), H, carry.data_ptr(), H, G[o:].data_ptr(), 4 * H, hprev, H,
                 dX_hi[o:].data_ptr(), dX_lo[o:].data_ptr(), dP_hi[o:].data_ptr(), dP_lo[o:].data_ptr(), self.ldg, st)
            if t:   # h_{-1} = 0 is a constant: no carry below step 0
                self._gemm(n, H, 3 * H, (dP_hi[o:], dP_lo[o:]), 0, self.W_hl['hh'], 1, carry, H, accumulate=1)
        self._mark('backward_recurrence')
        g_hh, g_ih = self.grad[:self.nW], self.grad[self.nW:]
        self._gemm(3 * H, H + 1, P, b['dHP_hl'], 1, b['Hp_hl'], 1, g_hh, H + 1, k_splits=-1)
        self._gemm(3 * H, H + 1, P, b['dXP_hl'], 1, b['X_hl'], 1, g_ih, H + 1, k_splits=-1)
        self._mark('weight_gradients')

    def _optimizer_step(self):
        self.steps += 1
        hi, lo = self.W_hl['hh']
        call('dae_optimizer_step', self.theta.data_ptr(), self.grad.data_ptr(), self.slot1.data_ptr(), self.slot2.data_ptr(),
             2 * self.nW, _cabi.OPT[self.opt], self.learning_rate, self.momentum, 1.0, self.steps, None, hi.data_ptr(), lo.data_ptr(),
             3 * self.dim, self.dim + 1, self.ldx, _stream())
        self._hh_valid = True
        self._mark('optimizer')

    def batches(self, indptr, epoch):
        """The epoch's batches of user ids: a permutation (seeded by seed and epoch) of the users with at least 2 reads -- the
        others have no loss term -- cut into batch_users."""
        active = np.flatnonzero(np.diff(indptr) >= 2)
        perm = active[np.random.default_rng([self.seed, epoch]).permutation(active.size)]
        return [perm[i:i + self.batch_users] for i in range(0, perm.size, self.batch_users)]

    def fit(self, sequences, embeddings):
        """num_epochs epochs over the users; train_loss gets each epoch's mean loss term.  The article embeddings stay fixed."""
        emb = self._embeddings(embeddings, 'UserGRU.fit')
        indptr, items = check_sequences(sequences, emb.shape[0], 'UserGRU.fit')
        for _ in range(self.num_epochs):
            epoch = self.epochs_done
            self.stats.zero_()
            terms = 0
            for bi, users in enumerate(self.batches(indptr, epoch)):
                pk = Packed(indptr, items, users, self.max_len)
                if pk.terms == 0:   # max_len = 1
                    continue
                self._forward_backward(pk, emb, epoch, bi)
                self._optimizer_step()
                terms += pk.terms
            self.train_loss.append(float(self.stats.item()) / max(terms, 1))
            self.epochs_done += 1
        return self

    # ---- inference --------------------------------------------------------------------------------------------------------
    def transform(self, sequences, embeddings, to_host=True):
        """User vectors [U, H] fp32: the state after each user's last (truncated) read; zero rows for users without reads.  Projects
        step by step, so device memory per batch is O(batch_users x 3H), not O(positions x 3H)."""
        emb = self._embeddings(embeddings, 'UserGRU.transform')
        indptr, items = check_sequences(sequences, emb.shape[0], 'UserGRU.transform')
        H, U, B, d, st = self.dim, len(indptr) - 1, self.batch_users, self.device, _stream()
        out = torch.zeros(U, H, dtype=torch.float32, device=d)
        if not self._hh_valid:
            self._split('hh')
            self._hh_valid = True
        self._split('ih')
        bf = dict(dtype=torch.bfloat16, device=d)
        X_hi, X_lo = torch.zeros(B, self.ldx, **bf), torch.zeros(B, self.ldx, **bf)
        h_hi, h_lo = torch.zeros(B, self.ldx, **bf), torch.zeros(B, self.ldx, **bf)
        XP = torch.empty(B, 3 * H, dtype=torch.float32, device=d)
        HP = torch.empty_like(XP)
        h = torch.empty(B, H, dtype=torch.float32, device=d)
        for u0 in range(0, U, B):
            pk = Packed(indptr, items, np.arange(u0, min(U, u0 + B)), self.max_len)
            if pk.B == 0:
                continue
            it = _upload(pk.items, d)
            h_hi.zero_()
            h_lo.zero_()
            h_hi[:, H] = 1.0
            h[:pk.B].zero_()
            for t in range(len(pk.n)):
                o, n = int(pk.off[t]), int(pk.n[t])
                call('dae_gather_split_bf16', emb.data_ptr(), emb.stride(0), it[o:].data_ptr(), n, H, X_hi.data_ptr(), X_lo.data_ptr(),
                     self.ldx, H, st)
                self._gemm(n, 3 * H, H + 1, (X_hi, X_lo), 0, self.W_hl['ih'], 0, XP, 3 * H)
                self._gemm(n, 3 * H, H + 1, (h_hi, h_lo), 0, self.W_hl['hh'], 0, HP, 3 * H)
                call('dae_gru_cell_fwd', n, H, XP.data_ptr(), 3 * H, HP.data_ptr(), 3 * H, h.data_ptr(), H, h.data_ptr(), H, n,
                     h_hi.data_ptr(), h_lo.data_ptr(), self.ldx, None, 0, st)
            out.index_copy_(0, torch.from_numpy(pk.order).to(d), h[:pk.B])
        return out.cpu().numpy() if to_host else out

    def recommend(self, sequences, embeddings, k=10, candidates=None, exclude_read=True, metric='linear kernel', to_host=True,
                  groups=None):
        """The k best articles per user for the GRU user vectors (helpers.recommend with profiles=transform(...)): every read
        article (the whole history, not only the last max_len) is excluded with exclude_read, users without reads get padding.
        groups: the articles' group labels, passed to helpers.recommend (at most one article per group, read groups excluded)."""
        from .helpers import recommend
        emb = self._embeddings(embeddings, 'UserGRU.recommend')
        indptr, items = check_sequences(sequences, emb.shape[0], 'UserGRU.recommend')
        hist = history_matrix(indptr, items, emb.shape[0])
        prof = self.transform((indptr, items), emb, to_host=False)
        return recommend(hist, emb, k=k, candidates=candidates, metric=metric, exclude_read=exclude_read, device=self.device,
                         to_host=to_host, profiles=prof, groups=groups)


def history_matrix(indptr, items, n_items):
    """The users' read articles as a scipy CSR [U, n_items] with 1 per article read (helpers.recommend's histories).  Built on
    copies: scipy sorts the arrays it is given in place."""
    import scipy.sparse as sp
    m = sp.csr_matrix((np.ones(len(items), np.float32), np.array(items), np.array(indptr)), shape=(len(indptr) - 1, n_items))
    m.sum_duplicates()
    m.data[:] = 1.0
    return m


def negatives_from_draws(pos, c, n_items):
    """dae_seq_negatives' map from the 32-bit Philox draw c to the negative of positive `pos`: (pos + 1 + floor(c (N - 1) / 2^32)) mod N."""
    pos, c = np.asarray(pos, np.int64), np.asarray(c, np.uint64)
    return ((pos + 1 + ((c * np.uint64(n_items - 1)) >> np.uint64(32)).astype(np.int64)) % n_items).astype(np.int32)
