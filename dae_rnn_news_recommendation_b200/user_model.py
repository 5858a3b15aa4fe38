"""Learned user vectors: a GRU over each user's reading sequence, trained on the H100 to score the next read above a random
article (DESIGN 4.10).

    m = UserGRU(dim=H, max_len=50, batch_users=1024, num_epochs=5)
    m.fit((indptr, items), embeddings)        # embeddings: [N, H] article vectors (transform()'s output), kept frozen, or an
                                              # ArticleEncoder, trained with the model (DESIGN 4.19)
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

Impression logs (DESIGN 4.13): fit(..., impressions=...) trains on the shown-but-not-clicked articles of each impression
(dae_impression_rank_loss in place of the two random-negative kernels), impression_states gives the query vector before each
impression and prefix_histories the reads before it for the mean-profile baseline.

Sampled softmax (DESIGN 4.16): with impression_loss='softmax' each click of an impression is one sample, scored against
impression_negatives = K non-clicks of the same impression drawn per click (all of them with K = 0 or K >= |N|) under a
(K + 1)-way softmax cross-entropy, the objective of MIND's NRMS / NAML / LSTUR trainers (npratio = 4).  The draws depend only on
(seed, epoch, impression id, the click's ordinal); dae_impression_softmax_loss replaces dae_impression_rank_loss.  Unlike MIND's
code, an impression with fewer than K non-clicks is not padded: its clicks are scored against all of them.

UserLSTM (DESIGN 4.15) is the same encoder with torch.nn.LSTM's cell (gate order i, f, g, o; state_dict loads into a CPU
torch.nn.LSTM(H, H)): the same constructor, losses, negatives, batches and methods, with 4H-wide projections and
dae_lstm_cell_fwd / dae_lstm_cell_bwd in place of the GRU's cell kernels.  Both derive from _UserRNN, which holds everything
that does not depend on the cell.

Long-term user vectors (DESIGN 4.18, LSTUR-ini): UserGRU / UserLSTM(..., long_term_users=U) learn a vector P[u] per user (the
long_term attribute, [U, H] fp32, zero at first) and start u's window from h_0 = P[u] instead of 0, so that what a user read
before the last max_len reads still shapes the state.  Training masks each batch user with probability long_term_mask (LSTUR's
training: a masked user starts from 0) and updates only the rows of the unmasked batch users, by dae_rows_optimizer_step
(long_term_learning_rate).  transform, impression_states and recommend start every user from its row, with no mask; users at or
beyond row U (cold-start users) start from 0.  save() / load() keep the table; state_dict() keeps torch's four keys.

Fine-tuned article encoder (DESIGN 4.19): fit(sequences, art) with an ArticleEncoder art in place of the embeddings trains the user
encoder and the DAE encoder e(x) = f(s x W + bh) - f(bh) of art on the same loss, with e(a) in place of the frozen row a.  Each
batch encodes only the T articles it touches (dae_touch_compact, dae_encode_csr_fwd_groups), runs every user-encoder kernel on that
compact table with slot ids, takes the article gradient from the loss (the *_loss_grad exports) and from the input projection
(dX = dXP . W_in, dae_rows_scatter_add), backpropagates it into [W | bh] (dae_encode_csr_bwd_gather) and steps [W | bh] after
theta.  art.vectors(X) encodes any bag of words with the learned W and bh, articles never seen in training included.

Deterministic training (DESIGN 4.21): with deterministic=True, two fits with the same seed, inputs, build and GPU model give the same
bits: theta, its slots, steps, train_loss, the long-term table, an ArticleEncoder's [W | bh] and slots, and everything computed from
them.  The stream-K weight GEMMs run as dae_gemm_bf16x3_det, the loss kernels store one fp64 term per position that
dae_loss_slots_sum adds in a fixed order, and with an ArticleEncoder the loss kernels emit the article gradient as (slot, row,
coefficient) triples that dae_ordered_rows sums per slot in a fixed order together with dX, before dae_encode_csr_bwd_det.  It is a
run option: save() does not store it.
"""
import numpy as np
import torch

from . import _cabi, sparse_optim
from ._cabi import call
from .article_encoder import ARTICLE_ENCODE_GROUPS, ARTICLE_LEARNING_RATE, ArticleEncoder  # noqa: F401

_NAMES = ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')
_LOSS_SLOTS_SUM = 'dae_loss_slots_sum'   # the deterministic mode's fixed-order loss sum (DESIGN 4.21)
LONG_TERM_LEARNING_RATE = 0.1    # the long-term table's default learning rate: the best of 0.01, 0.03 and 0.1 (DESIGN 4.18)


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


IMPRESSION_KEYS = ('user', 'time', 'indptr', 'items', 'clicked')
IMPRESSION_LOSSES = ('pairwise', 'softmax')
MAX_IMPRESSION_NEGATIVES = 32   # dae_impression_softmax_loss draws one negative per lane


def check_impressions(impressions, n_items, fn, seq_indptr=None):
    """An impression set as a dict of fresh arrays {'user' int64 [I], 'time' int64 [I], 'indptr' int64 [I + 1], 'items' int32,
    'clicked' uint8}, or ValueError before any device work.  impressions: a mapping with those keys (a dict, or np.load of the CLI's
    .npz).  indptr must start at 0, never decrease and end at len(items); items lie in [0, n_items) and are distinct within one
    impression; clicked has one 0 / 1 flag per shown article.  With seq_indptr (the sequences' offsets) user must be a row of the
    sequences and 0 <= time <= that user's read count; without it user and time are not read.  The caller's arrays are not
    modified."""
    try:
        got = {k: np.asarray(impressions[k]) for k in IMPRESSION_KEYS if seq_indptr is not None or k in ('indptr', 'items', 'clicked')}
    except (KeyError, TypeError, IndexError, ValueError):
        raise ValueError('%s: impressions must map %s to arrays' % (fn, ', '.join(IMPRESSION_KEYS)))
    indptr, items, clicked = got['indptr'], got['items'], got['clicked']
    if indptr.ndim != 1 or indptr.size < 1 or not np.issubdtype(indptr.dtype, np.integer):
        raise ValueError('%s: impressions indptr must be a 1-D integer array of I + 1 offsets' % fn)
    if items.ndim != 1 or not (np.issubdtype(items.dtype, np.integer) or items.size == 0):
        raise ValueError('%s: impressions items must be a 1-D integer array' % fn)
    if indptr[0] != 0 or indptr[-1] != items.size or (np.diff(indptr) < 0).any():
        raise ValueError('%s: impressions indptr must start at 0, never decrease and end at len(items) = %d' % (fn, items.size))
    if clicked.shape != items.shape or not (clicked.dtype == np.bool_ or np.issubdtype(clicked.dtype, np.integer)) or \
            (clicked.size and not np.isin(clicked, (0, 1)).all()):
        raise ValueError('%s: clicked must hold one 0 / 1 flag per shown article (%d)' % (fn, items.size))
    if items.size and (items.min() < 0 or items.max() >= n_items):
        raise ValueError('%s: impressions show an article outside [0, %d)' % (fn, n_items))
    n_imp = indptr.size - 1
    row = np.repeat(np.arange(n_imp, dtype=np.int64), np.diff(indptr))
    key = row * max(int(n_items), 1) + items.astype(np.int64)
    if key.size > 1 and (np.diff(np.sort(key)) == 0).any():
        raise ValueError('%s: an impression shows the same article twice' % fn)
    out = {'indptr': indptr.astype(np.int64), 'items': items.astype(np.int32), 'clicked': clicked.astype(np.uint8)}
    if seq_indptr is not None:
        user, time = got['user'], got['time']
        for k, v in (('user', user), ('time', time)):
            if v.shape != (n_imp,) or not (np.issubdtype(v.dtype, np.integer) or v.size == 0):
                raise ValueError('%s: impressions %s must be an integer array of one entry per impression (%d)' % (fn, k, n_imp))
        n_u = len(seq_indptr) - 1
        if user.size and (user.min() < 0 or user.max() >= n_u):
            raise ValueError('%s: impressions user outside [0, %d)' % (fn, n_u))
        lens = np.diff(seq_indptr)
        if time.size and ((time < 0).any() or (time > lens[user]).any()):
            raise ValueError("%s: impressions time must lie in [0, the user's read count]" % fn)
        out['user'], out['time'] = user.astype(np.int64), time.astype(np.int64)
    return out


def usable_impressions(imp, seq_indptr, max_len):
    """Boolean [I]: the impressions the impression loss uses -- at least one click and one non-click, and a state inside the
    user's trained window of the last max_len reads (time > len - min(len, max_len), so never time = 0)."""
    lens = np.diff(seq_indptr)[imp['user']]
    L = np.minimum(lens, max_len)
    n = np.diff(imp['indptr'])
    cs = np.concatenate([[0], np.cumsum(imp['clicked'], dtype=np.int64)])
    nc = cs[imp['indptr'][1:]] - cs[imp['indptr'][:-1]]
    return (nc > 0) & (nc < n) & (imp['time'] > lens - L) & (imp['time'] >= 1)


def _count(impressions):
    """The impression count len(indptr) - 1 without reading the arrays (0 when malformed: check_impressions reports that)."""
    try:
        return len(impressions['indptr']) - 1
    except (KeyError, TypeError, IndexError, ValueError):
        return 0


class ImpressionBatch:
    """The impressions of one packed training batch (pk: Packed), grouped by packed position.  An impression of user order[i] at
    time t has its state at position off[t'] + i with t' = t - 1 - (len - L).  pos_indptr [P + 1]: position p's impressions are
    [pos_indptr[p], pos_indptr[p + 1]) of this batch's own (indptr, items, clicked), in increasing impression id.  ids: the
    impression ids in that order; clicks: their click count.  `buffer` packs the four arrays (and with ids=True the ids) into one
    byte buffer for a single upload; `views` cuts the uploaded copy back into typed device tensors."""

    def __init__(self, pk, imp, use, seq_indptr):
        slot = np.full(int(seq_indptr.size - 1), -1, np.int64)
        slot[pk.order] = np.arange(pk.B)
        ids = np.flatnonzero(use & (slot[imp['user']] >= 0))
        u = imp['user'][ids]
        i = slot[u]
        lens = seq_indptr[u + 1] - seq_indptr[u]
        t = imp['time'][ids] - 1 - (lens - pk.L[i])
        p = pk.off[t] + i
        o = np.argsort(p, kind='stable')
        self.ids, self.p = ids[o], p[o]
        self.n = int(self.ids.size)
        self.pos_indptr = np.zeros(pk.P + 1, np.int64)
        np.cumsum(np.bincount(self.p, minlength=pk.P), out=self.pos_indptr[1:])
        lo, hi = imp['indptr'][self.ids], imp['indptr'][self.ids + 1]
        m = hi - lo
        self.indptr = np.concatenate([[0], np.cumsum(m)]).astype(np.int64)
        src = np.repeat(lo - self.indptr[:-1], m) + np.arange(int(self.indptr[-1]))
        self.items, self.clicked = imp['items'][src], imp['clicked'][src]
        self.clicks = int(np.count_nonzero(self.clicked))

    def buffer(self, ids=False):
        parts = [self.pos_indptr.view(np.uint8), self.indptr.view(np.uint8), self.items.view(np.uint8), self.clicked]
        if ids:
            parts.append(self.ids.astype(np.int64).view(np.uint8))
        self._sizes = [a.size for a in parts]
        pad = [(-s) % 8 for s in self._sizes]
        return np.concatenate([np.concatenate([a, np.zeros(q, np.uint8)]) for a, q in zip(parts, pad)])

    def views(self, dev):
        out, o = [], 0
        for s, dt in zip(self._sizes, (torch.int64, torch.int64, torch.int32, torch.uint8, torch.int64)):
            out.append(dev[o:o + s].view(dt))
            o += s + (-s) % 8
        return out


class Packed:
    """One batch in the PackedSequence layout.  order: the batch's users (ids) by truncated length L, descending (stable), users with
    L = 0 left out; n[t] = users with L > t; off[t] = first position of step t; position off[t] + i is user order[i]'s read t.
    items[p]: the article read at position p; nxt[p]: the article read next (-1 at a user's last position).  users: the user each
    row belongs to, order itself unless the rows are impression_states' runs (which set it)."""

    def __init__(self, indptr, items, users, max_len):
        users = np.asarray(users, dtype=np.int64)
        L = np.minimum(indptr[users + 1] - indptr[users], max_len)
        keep = L > 0
        users, L = users[keep], L[keep]
        s = np.argsort(-L, kind='stable')
        self.order, self.L = users[s], L[s]
        self.users = self.order
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


class _UserEncoder:
    """What every user encoder shares (UserGRU, UserLSTM, UserAttention): the constructor's checks, the flat fp32 parameters theta
    and their optimizer slots, the loss dispatch of a packed training batch, the fit loop, batches, the optimizer step, the
    impression runs of impression_states, transform's batch loop, recommend, save and load.  An encoder class supplies the
    parameters and their files (state_dict, load_state_dict, _CONFIG / _PARAMS / _dim_of), its training buffers, _refresh (the
    bf16 weight operands before a forward), _forward (the states Hs of every packed position) and _backward (theta's gradient from
    dH), and for inference _infer_buffers, _last_states and _run_capture."""
    _CONFIG = ()                     # constructor arguments save() stores next to max_len
    _PARAMS = ()                     # state_dict names

    def __init__(self, dim, max_len=50, batch_users=1024, num_epochs=5, opt='adam', learning_rate=1e-3, seed=0, device='cuda:0',
                 momentum=0.5, impression_loss='pairwise', impression_negatives=4, deterministic=False):
        name = type(self).__name__
        if type(deterministic) is not bool:
            raise ValueError('%s: deterministic = %r, True or False' % (name, deterministic))
        if dim < 1 or max_len < 1 or batch_users < 1 or num_epochs < 0:
            raise ValueError('%s: dim, max_len and batch_users must be >= 1 and num_epochs >= 0' % name)
        if opt not in _cabi.OPT:
            raise ValueError('%s: opt = %r, one of %s' % (name, opt, sorted(_cabi.OPT)))
        if impression_loss not in IMPRESSION_LOSSES:
            raise ValueError('%s: impression_loss = %r, one of %s' % (name, impression_loss, list(IMPRESSION_LOSSES)))
        if isinstance(impression_negatives, bool) or not isinstance(impression_negatives, (int, np.integer)) or \
                not 0 <= impression_negatives <= MAX_IMPRESSION_NEGATIVES:
            raise ValueError('%s: impression_negatives = %r, an integer in [0, %d] (0: every non-click)'
                             % (name, impression_negatives, MAX_IMPRESSION_NEGATIVES))
        self.impression_loss, self.impression_negatives = impression_loss, int(impression_negatives)
        self.deterministic = deterministic
        self._gemm_ws = None      # dae_gemm_bf16x3_det's workspace (deterministic mode; the user path runs on one stream)
        self.dim, self.max_len, self.batch_users, self.num_epochs = int(dim), int(max_len), int(batch_users), int(num_epochs)
        self.opt, self.learning_rate, self.momentum, self.seed = opt, float(learning_rate), float(momentum), int(seed)
        self.device = torch.device(device)
        self.train_loss = []
        self.steps = 0
        self.epochs_done = 0
        self._buf = {}
        self._cap = (0, 0)
        self.stats = torch.zeros(1, dtype=torch.float64, device=self.device)
        self.phase_events = None   # a list to record (phase name, CUDA event) pairs into (tools/bench_user_model.py)

    def _set_theta(self, theta):
        """theta (fp32 NumPy) on the device, its gradient and the optimizer slots."""
        self.theta = torch.from_numpy(theta).to(self.device)
        self.grad = torch.zeros_like(self.theta)
        self.slot1 = torch.full_like(self.theta, 0.1 if self.opt == 'ada_grad' else 0.0)
        self.slot2 = torch.zeros_like(self.theta)

    def _reset_slots(self):
        self.slot1.fill_(0.1 if self.opt == 'ada_grad' else 0.0)
        self.slot2.zero_()
        self.steps = 0

    def _load_arrays(self, sd, want):
        """{name: fp32 NumPy array} from a state dict, or ValueError naming the missing keys or a wrong shape."""
        name = type(self).__name__
        missing = set(want) - set(sd)
        if missing:
            raise ValueError('%s.load_state_dict: missing %s' % (name, sorted(missing)))
        a = {}
        for k, shape in want.items():
            v = sd[k]
            v = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
            if tuple(v.shape) != shape:
                raise ValueError('%s.load_state_dict: %s has shape %s, %s expected (H = %d)' % (name, k, tuple(v.shape), shape,
                                                                                              self.dim))
            a[k] = v.astype(np.float32)
        return a

    def _files(self):
        """save()'s arrays: max_len, the encoder's _CONFIG and the state dict."""
        sd = self.state_dict()
        return dict(max_len=self.max_len, **{k: getattr(self, k) for k in self._CONFIG}, **{k: v.numpy() for k, v in sd.items()})

    def save(self, path):
        np.savez(path, **self._files())

    @classmethod
    def load(cls, path, **kw):
        """A model from save()'s .npz; keyword arguments as the constructor's (dim, max_len and the encoder's _CONFIG come from the
        file).  A file without this encoder's keys -- another encoder's -- raises ValueError naming them; another recurrent cell's
        file fails load_state_dict's shape check."""
        z = np.load(path)
        missing = sorted(set(('max_len',) + cls._CONFIG + cls._PARAMS) - set(z.files))
        if missing:
            raise ValueError('%s.load: %s is not a %s file: it lacks %s' % (cls.__name__, path, cls.__name__, missing))
        for k in ('max_len',) + cls._CONFIG:
            kw.setdefault(k, int(z[k]))
        m = cls(cls._dim_of(z), **kw)
        m.load_state_dict({k: z[k] for k in cls._PARAMS})
        return m

    # ---- device helpers ---------------------------------------------------------------------------------------------------
    def _check_articles(self, art, fn):
        if art.dim != self.dim:
            raise ValueError('%s: the article encoder has H = %d, the model %d' % (fn, art.dim, self.dim))

    def _embeddings(self, embeddings, fn):
        from .helpers import _dense_embeddings
        if isinstance(embeddings, ArticleEncoder):
            self._check_articles(embeddings, fn)
            return embeddings.vectors(to_host=False)
        emb = _dense_embeddings(embeddings, self.device, fn)
        if emb.shape[1] != self.dim:
            raise ValueError('%s: embeddings are %d wide, the model has H = %d' % (fn, emb.shape[1], self.dim))
        if emb.shape[0] < 2:
            raise ValueError('%s: at least 2 articles are needed' % fn)
        return emb

    def _gemm(self, M, N, K, A, a_mn, Bm, b_mn, C, ldc, accumulate=0, k_splits=1):
        """C (+)= A . B^T on the bf16x3 tensor cores.  The stream-K calls (k_splits = -1) add split tiles by fp32 atomics; in the
        deterministic mode they run as dae_gemm_bf16x3_det.  Calls with k_splits = 1 have one writer per element in both modes."""
        (a_hi, a_lo), (b_hi, b_lo) = A, Bm
        args = (M, N, K, 1.0, a_hi.data_ptr(), a_lo.data_ptr(), a_hi.stride(0), a_mn, b_hi.data_ptr(), b_lo.data_ptr(), b_hi.stride(0),
                b_mn, C.data_ptr(), ldc, 0, -1, None, k_splits, accumulate)
        name, ws = 'dae_gemm_bf16x3', ()
        if self.deterministic and k_splits != 1:
            if self._gemm_ws is None:
                self._gemm_ws = torch.empty(_cabi.query('dae_gemm_det_workspace'), dtype=torch.uint8, device=self.device)
            name, ws = name + '_det', (self._gemm_ws.data_ptr(), self._gemm_ws.numel())
        call(name, *args, *ws, _stream())

    def _mark(self, name):
        if self.phase_events is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.phase_events.append((name, e))

    # ---- training ---------------------------------------------------------------------------------------------------------
    def _forward_backward(self, pk, emb, epoch, batch, ib=None, art=None):
        """Loss (added to self.stats) and the gradient (self.grad) of one packed batch with pk.terms > 0, or with ib (an
        ImpressionBatch with ib.n > 0) the impression loss of its impressions in place of the random negatives: pairwise, or with
        impression_loss='softmax' the sampled softmax over its ib.clicks samples.  With art (an ArticleEncoder; emb is then None)
        the batch runs on the compact table of the articles it touches and art.grad gets [dW | dbh] (DESIGN 4.19)."""
        H, P = self.dim, pk.P
        b = self._buffers(P, pk.B)
        st = _stream()
        neg = b['neg']
        if art is None:
            items = _upload(pk.items, self.device)
        elif ib is None:   # one upload of every id the batch touches: [items | nxt | neg (drawn below)] or [items | shown items]
            ids = _upload(np.concatenate([pk.items, pk.nxt, np.full(P, -1, np.int32)]), self.device)
        else:
            ids = _upload(np.concatenate([pk.items, ib.items]), self.device)
        if ib is None:
            nxt = _upload(pk.nxt, self.device) if art is None else ids[P:2 * P]
        elif self.impression_loss == 'softmax':
            pos_indptr, imp_indptr, imp_items, imp_clicked, imp_ids = ib.views(_upload(ib.buffer(ids=True), self.device))
        else:
            pos_indptr, imp_indptr, imp_items, imp_clicked = ib.views(_upload(ib.buffer(), self.device))
        self._refresh()
        self._mark('start')
        if ib is None:   # in article-id space: the same negatives as a run on frozen embeddings
            if art is not None:
                neg = ids[2 * P:]
            call('dae_seq_negatives', nxt.data_ptr(), P, emb.shape[0] if art is None else art.n, self.seed, epoch, batch, neg.data_ptr(),
                 st)
        grad = ()
        if art is not None:
            rows, slots, T = art.touch(ids)
            items = slots[:P]
            if ib is None:
                nxt, neg = slots[P:2 * P], slots[2 * P:]
            else:
                imp_items = slots[P:]
            self._mark('compact')
            emb, col_count = art.encode_rows(rows, T)
            self._mark('encode')
        det = self.deterministic
        if det:   # one fp64 loss slot per position; with art the article gradient as triples (slot, row of Hs, coefficient)
            loss = torch.empty(P, dtype=torch.float64, device=self.device)
            if art is not None:
                n_trip = 2 * P if ib is None else int(ib.items.size)
                trip = (torch.empty(n_trip, dtype=torch.int32, device=self.device), torch.empty(n_trip, dtype=torch.int32, device=self.device),
                        torch.empty(n_trip, dtype=torch.float32, device=self.device))
                grad = tuple(t.data_ptr() for t in trip)
        else:
            loss = self.stats
            if art is not None:
                dE = torch.zeros_like(emb)
                grad = (dE.data_ptr(), H)
        sfx = ('' if art is None else '_grad') + ('_det' if det else '')
        self._forward(b, pk, emb, items, st)
        Hs = b['Hs']
        if ib is None:
            call('dae_seq_rank_loss' + sfx, Hs.data_ptr(), H, emb.data_ptr(), emb.stride(0), H, nxt.data_ptr(), neg.data_ptr(), P,
                 1.0 / pk.terms, b['dH'].data_ptr(), H, loss.data_ptr(), *grad, st)
        elif self.impression_loss == 'softmax':
            ws = torch.empty(2 * ib.items.size, dtype=torch.int32, device=self.device)   # 8 bytes per shown article
            call('dae_impression_softmax_loss' + sfx, Hs.data_ptr(), H, emb.data_ptr(), emb.stride(0), H, pos_indptr.data_ptr(), P,
                 imp_indptr.data_ptr(), imp_items.data_ptr(), imp_clicked.data_ptr(), imp_ids.data_ptr(), self.impression_negatives,
                 self.seed, epoch, 1.0 / ib.clicks, b['dH'].data_ptr(), H, loss.data_ptr(), ws.data_ptr(), *grad, st)
        else:
            call('dae_impression_rank_loss' + sfx, Hs.data_ptr(), H, emb.data_ptr(), emb.stride(0), H, pos_indptr.data_ptr(), P,
                 imp_indptr.data_ptr(), imp_items.data_ptr(), imp_clicked.data_ptr(), 1.0 / ib.n, b['dH'].data_ptr(), H,
                 loss.data_ptr(), *grad, st)
        if det:   # stats[0] += the slots in dae_loss_slots_sum's fixed order
            call(_LOSS_SLOTS_SUM, loss.data_ptr(), P, self.stats.data_ptr(), st)
        self._mark('loss')
        self._backward(b, pk, st)
        if art is not None:
            # dX = dXP . W_in[:, :H] with the forward's bf16 copy of W_in, added into the rows of the positions' articles
            dgrad, W_in, K = self._input_grad(b)
            dX = torch.empty(P, H, dtype=torch.float32, device=self.device)
            self._gemm(P, H, K, dgrad, 0, W_in, 1, dX, H)
            if det:   # dE = the loss triples over Hs, then the dX rows, per slot in that order
                dE = torch.empty_like(emb)
                art.ordered_rows(trip, Hs, dX, items, T, dE)
            else:
                art.scatter_rows(dX, items, dE)
            self._mark('input_gradient')
            art.backward(rows, T, emb, dE, col_count, deterministic=det)
            self._mark('article_backward')
            self.article_batch = {'rows': rows, 'slots': slots, 'E': emb, 'dE': dE, 'dX': dX}   # the last batch's tables, for inspection

    def _optimizer_step(self):
        """One dae_optimizer_step over all of theta; _step_split() names the bf16 hi / lo copy of theta's leading block that the
        step also writes (or None)."""
        self.steps += 1
        hi, lo, rows, cols, ld = self._step_split()
        call('dae_optimizer_step', self.theta.data_ptr(), self.grad.data_ptr(), self.slot1.data_ptr(), self.slot2.data_ptr(),
             self.theta.numel(), _cabi.OPT[self.opt], self.learning_rate, self.momentum, 1.0, self.steps, None, hi, lo, rows, cols,
             ld, _stream())
        self._mark('optimizer')

    def batches(self, indptr, epoch, active=None):
        """The epoch's batches of user ids: a permutation (seeded by seed and epoch) of the users with at least 2 reads -- the
        others have no loss term -- cut into batch_users.  active: the user ids to permute instead (sorted)."""
        if active is None:
            active = np.flatnonzero(np.diff(indptr) >= 2)
        perm = active[np.random.default_rng([self.seed, epoch]).permutation(active.size)]
        return [perm[i:i + self.batch_users] for i in range(0, perm.size, self.batch_users)]

    def fit(self, sequences, embeddings, impressions=None):
        """num_epochs epochs over the users; train_loss gets each epoch's mean loss term.  embeddings: the article vectors [N, H],
        which stay fixed, or an ArticleEncoder, whose [W | bh] is trained on the same loss (DESIGN 4.19): after theta's step (and the
        long-term rows') one optimizer step of [W | bh] with the encoder's own opt and learning rate.

        impressions (check_impressions' keys): train on them instead of random negatives.  Impression i of user u at time t
        scores its shown articles with h, the packed training state after u's first t reads, and its loss is
        1 / (|C| |N|) sum_{c clicked, n not} softplus(h.e_n - h.e_c); a batch's loss is the mean over its impressions.  An
        impression counts when it has a click and a non-click and its state lies in the trained window of the user's last
        max_len reads (time > len - min(len, max_len)); impression_counts gets {'used', 'skipped'}.  The batches permute the
        users with a usable impression as batches() does; one impression with one click at time t on read t + 1 and one
        non-click is exactly the random-negative term at position t.

        With impression_loss='softmax' (DESIGN 4.16) each click c of a usable impression is one sample: its loss is
        log(e^{s_c} + sum_{n in S_c} e^{s_n}) - s_c with S_c = impression_negatives non-clicks of the same impression drawn for
        that click (every non-click when impression_negatives = 0 or the impression has no more), a batch's loss is the mean
        over its clicks, train_loss the epoch mean over clicks, and impression_counts also gets 'clicks'.  The log must hold
        fewer than 2^32 impressions (the draws are keyed by the impression id)."""
        fn = '%s.fit' % type(self).__name__
        art = embeddings if isinstance(embeddings, ArticleEncoder) else None
        if art is not None:
            self._check_articles(art, fn)
            emb, n_items = None, art.n
        else:
            emb = self._embeddings(embeddings, fn)
            n_items = emb.shape[0]
        indptr, items = check_sequences(sequences, n_items, fn)
        imp = active = use = None
        if impressions is not None:
            softmax = self.impression_loss == 'softmax'
            if softmax and _count(impressions) >= 2 ** 32:
                raise ValueError('%s: impression_loss=\'softmax\' keys its draws by a 32-bit impression id: at most 2^32 - 1 '
                                 'impressions' % fn)
            imp = check_impressions(impressions, n_items, fn, indptr)
            use = usable_impressions(imp, indptr, self.max_len)
            active = np.unique(imp['user'][use])
            self.impression_counts = {'used': int(use.sum()), 'skipped': int(use.size - use.sum())}
            if softmax:
                ends = imp['indptr']
                cs = np.concatenate([[0], np.cumsum(imp['clicked'], dtype=np.int64)])
                self.impression_counts['clicks'] = int((cs[ends[1:]] - cs[ends[:-1]])[use].sum())
        for _ in range(self.num_epochs):
            epoch = self.epochs_done
            self.stats.zero_()
            terms = 0
            for bi, users in enumerate(self.batches(indptr, epoch, active)):
                pk = Packed(indptr, items, users, self.max_len)
                ib = None
                if imp is not None:
                    ib = ImpressionBatch(pk, imp, use, indptr)
                    n = ib.clicks if self.impression_loss == 'softmax' else ib.n
                else:
                    n = pk.terms
                if n == 0:   # max_len = 1
                    continue
                self._forward_backward(pk, emb, epoch, bi, ib, art)
                self._optimizer_step()
                if art is not None:
                    art.step()
                    self._mark('article_step')
                terms += n
            self.train_loss.append(float(self.stats.item()) / max(terms, 1))
            self.epochs_done += 1
        return self

    # ---- inference --------------------------------------------------------------------------------------------------------
    def transform(self, sequences, embeddings, to_host=True):
        """User vectors [U, H] fp32: the state after each user's last (truncated) read; zero rows for users without reads.  With a
        long-term table (UserGRU / UserLSTM) user u's window starts from P[u], and users at or beyond long_term_users (cold-start
        users, whom training never saw) from 0, as without the table.  Device
        memory per batch: O(batch_users x GATES H) for the recurrent cells, which project step by step; O(batch positions x (3H + A))
        for UserAttention, which runs each batch in one pass."""
        fn = '%s.transform' % type(self).__name__
        emb = self._embeddings(embeddings, fn)
        indptr, items = check_sequences(sequences, emb.shape[0], fn)
        H, U, B, d = self.dim, len(indptr) - 1, self.batch_users, self.device
        out = torch.zeros(U, H, dtype=torch.float32, device=d)
        s = self._infer_buffers(B)
        for u0 in range(0, U, B):
            pk = Packed(indptr, items, np.arange(u0, min(U, u0 + B)), self.max_len)
            if pk.B == 0:
                continue
            out.index_copy_(0, torch.from_numpy(pk.order).to(d), self._last_states(pk, emb, s))
        return out.cpu().numpy() if to_host else out

    def impression_states(self, sequences, embeddings, impressions, to_host=True):
        """Query vectors [I, H] fp32 for impressions (check_impressions' keys): row i is the state after the last min(time, max_len)
        reads of its user before the impression, a zero row at time = 0.  At time = len this is transform's row.

        Training (fit(impressions=...)) takes the state from the packed window of the user's LAST max_len reads, which starts at
        read len - max_len whatever the impression's time; here the window ENDS at the impression.  The two agree at time = len
        and for users with at most max_len reads.  Each (user, window start) pair is one run of a packed batch, whose states are
        copied out at the steps that impressions ask for: a user whose impressions all lie within the first max_len reads costs
        one run.  With a long-term table every run starts from P[its user] (a cold-start user at or beyond long_term_users from 0),
        whatever the window's start.  Device memory per batch is transform's."""
        fn = '%s.impression_states' % type(self).__name__
        emb = self._embeddings(embeddings, fn)
        indptr, items = check_sequences(sequences, emb.shape[0], fn)
        imp = check_impressions(impressions, emb.shape[0], fn, indptr)
        H, d = self.dim, self.device
        n_imp = imp['user'].size
        out = torch.zeros(n_imp, H, dtype=torch.float32, device=d)
        ids = np.flatnonzero(imp['time'] > 0)
        if ids.size == 0:
            return out.cpu().numpy() if to_host else out
        u, t = imp['user'][ids], imp['time'][ids]
        start = np.maximum(t - self.max_len, 0)
        # runs: one per distinct (user, window start), each as long as its latest impression needs (<= max_len steps)
        key = u * (int(indptr[-1]) + 1) + start
        run_key, run_of = np.unique(key, return_inverse=True)
        n_run = run_key.size
        run_len = np.zeros(n_run, np.int64)
        np.maximum.at(run_len, run_of, t - start)
        first = np.zeros(n_run, np.int64)
        first[run_of] = np.arange(ids.size)   # any impression of the run gives its user and start
        r_src = indptr[u[first]] + start[first]
        r_indptr = np.concatenate([[0], np.cumsum(run_len)]).astype(np.int64)
        r_items = items[np.repeat(r_src - r_indptr[:-1], run_len) + np.arange(int(r_indptr[-1]))]
        step = t - start - 1   # the step after which impression ids[j] reads its run's state
        B = self.batch_users
        s = self._infer_buffers(B)
        order = np.argsort(run_of, kind='stable')
        run_user = u[first]
        for r0 in range(0, n_run, B):
            pk = Packed(r_indptr, r_items, np.arange(r0, min(n_run, r0 + B)), self.max_len)
            pk.users = run_user[pk.order]
            row = np.empty(n_run, np.int64)
            row[pk.order] = np.arange(pk.B)
            lo, hi = np.searchsorted(run_of[order], [r0, r0 + B])
            sel = order[lo:hi]
            self._run_capture(pk, emb, s, step[sel], row[run_of[sel]], ids[sel], out)
        return out.cpu().numpy() if to_host else out

    def recommend(self, sequences, embeddings, k=10, candidates=None, exclude_read=True, metric='linear kernel', to_host=True,
                  groups=None, long_lists=False):
        """The k best articles per user for the learned user vectors (helpers.recommend with profiles=transform(...)): every read
        article (the whole history, not only the last max_len) is excluded with exclude_read, users without reads get padding.
        groups: the articles' group labels, passed to helpers.recommend (at most one article per group, read groups excluded).
        long_lists: passed to helpers.recommend (k up to 1024)."""
        from .helpers import recommend
        fn = '%s.recommend' % type(self).__name__
        emb = self._embeddings(embeddings, fn)
        indptr, items = check_sequences(sequences, emb.shape[0], fn)
        hist = history_matrix(indptr, items, emb.shape[0])
        prof = self.transform((indptr, items), emb, to_host=False)
        return recommend(hist, emb, k=k, candidates=candidates, metric=metric, exclude_read=exclude_read, device=self.device,
                         to_host=to_host, profiles=prof, groups=groups, long_lists=long_lists)


class _UserRNN(_UserEncoder):
    """What the recurrent user encoders share (UserGRU, UserLSTM): the flat parameters theta = [W~_hh | W~_ih] of GATES H rows each,
    their torch.nn.GRU / torch.nn.LSTM names, the packed training batch's step loops and the step loop of transform and
    impression_states.  A cell class supplies GATES, its extra buffers, the carries its backward zeroes, the packed gradient
    operands of the two weight GEMMs and its two kernel calls (_cell_fwd / _cell_bwd for training, _step for inference).

    Long-term user vectors (LSTUR-ini, DESIGN 4.18): with long_term_users = U the encoder keeps a table P [U, H] fp32 (the
    long_term attribute), zero at first, and user u's window starts from h_0 = P[u] (the LSTM's c_0 stays 0) in fit, transform,
    impression_states and recommend; users at or beyond row U (cold-start users) start from 0.  In training each batch user is
    masked with probability long_term_mask, drawn per (seed, epoch, user id): a masked user starts from 0 and its row is not
    updated.  dL/dh_0 of the unmasked users updates their rows after theta's step by dae_rows_optimizer_step (the encoder's opt
    and momentum, learning rate long_term_learning_rate, Adam's bias correction counted per row); other rows and their slots are
    not touched.  The table holds one more row, index U, that stays zero: masked and cold-start users gather it."""
    GATES = 0
    _STATES = ('h',)                 # [B x H] inference states, zero at a batch's first step (h: P[u] with the long-term table)
    _CARRIES = ('carry',)            # [B x H] backward carries zeroed for the rows of step 0
    _DGRAD = ('dHP_hl', 'dXP_hl')    # packed gradient operands of [dW_hh | db_hh] and [dW_ih | db_ih]
    _CARRY_ACCUMULATE = 1            # the carry GEMM dh_{t-1} (+)= dHP_t . W_hh accumulates onto the cell's carry, or stores
    _PARAMS = _NAMES

    def __init__(self, dim, *args, long_term_users=None, long_term_mask=0.5, long_term_learning_rate=None, **kw):
        super().__init__(dim, *args, **kw)
        name = type(self).__name__
        if long_term_users is not None and (isinstance(long_term_users, bool) or not isinstance(long_term_users, (int, np.integer))
                                            or long_term_users < 1):
            raise ValueError('%s: long_term_users = %r, None or an integer >= 1' % (name, long_term_users))
        if not 0.0 <= long_term_mask <= 1.0:
            raise ValueError('%s: long_term_mask = %r must lie in [0, 1]' % (name, long_term_mask))
        lr = LONG_TERM_LEARNING_RATE if long_term_learning_rate is None else float(long_term_learning_rate)
        if not lr > 0.0:
            raise ValueError('%s: long_term_learning_rate = %r must be > 0' % (name, long_term_learning_rate))
        self.long_term_users = None if long_term_users is None else int(long_term_users)
        self.long_term_mask, self.long_term_learning_rate = float(long_term_mask), lr
        H, G = self.dim, self.GATES
        self.nW = G * H * (H + 1)
        self.ldx, self.ldg = _ld8(H + 1), _ld8(G * H)
        # torch.nn.GRU's and torch.nn.LSTM's initialisation: every parameter uniform in [-1/sqrt(H), 1/sqrt(H)]
        rng = np.random.default_rng(self.seed)
        k = 1.0 / np.sqrt(H)
        self._set_theta(rng.uniform(-k, k, 2 * self.nW).astype(np.float32))
        bf = dict(dtype=torch.bfloat16, device=self.device)
        self.W_hl = {g: (torch.zeros(G * H, self.ldx, **bf), torch.zeros(G * H, self.ldx, **bf)) for g in ('hh', 'ih')}
        self._hh_valid = False
        self._lt = self._lt_slot1 = self._lt_slot2 = self._lt_count = self._lt_batch = self._lt_kept = None
        if self.long_term_users is not None:
            shape, f32 = (self.long_term_users + 1, H), dict(dtype=torch.float32, device=self.device)
            self._lt = torch.zeros(shape, **f32)
            if self.opt != 'gradient_descent':
                self._lt_slot1 = torch.full(shape, 0.1 if self.opt == 'ada_grad' else 0.0, **f32)
            if self.opt == 'adam':
                self._lt_slot2 = torch.zeros(shape, **f32)
            self._lt_count = torch.zeros(shape[0], dtype=torch.int32, device=self.device)

    @property
    def long_term(self):
        """The long-term user vectors P [long_term_users, H] fp32 on the device (a view: writing it changes the model), or None."""
        return None if self._lt is None else self._lt[:self.long_term_users]

    def long_term_kept(self, epoch):
        """Boolean [long_term_users]: the users that start from their row of P in the training batches of this epoch, each kept
        with probability 1 - long_term_mask by a draw keyed by (seed, epoch, user id), so the set does not depend on batch_users or
        on the batch order."""
        if self._lt_kept is None or self._lt_kept[0] != epoch:
            u = np.random.default_rng([self.seed, epoch, 1]).random(self.long_term_users)
            self._lt_kept = (epoch, u >= self.long_term_mask)
        return self._lt_kept[1]

    def _table_rows(self, users):
        """The row of P each user starts from: its own below long_term_users, else the zero row."""
        return np.where(users < self.long_term_users, users, self.long_term_users).astype(np.int32)

    def _initial_states(self, rows, n, hi, lo, h, st):
        """h_0 of rows [0, n): [P[rows] | 1] as the recurrent GEMM's bf16 hi / lo operand, and P[rows] in fp32 into h."""
        H = self.dim
        call('dae_gather_split_bf16', self._lt.data_ptr(), H, rows.data_ptr(), n, H, hi.data_ptr(), lo.data_ptr(), self.ldx, H, st)
        torch.index_select(self._lt, 0, rows[:n], out=h[:n])

    def _h0(self, b):
        """The training cell's h_prev at step 0: the gathered P rows with the long-term table, else NULL (h_{-1} = 0)."""
        return None if self._lt is None else b['h0'].data_ptr()

    # ---- parameters -------------------------------------------------------------------------------------------------------
    def _theta(self, g):
        """W~_g = [W_g | b_g] as a [GATES H, H+1] view of theta (g = 'hh' or 'ih')."""
        o = 0 if g == 'hh' else self.nW
        return self.theta[o:o + self.nW].view(self.GATES * self.dim, self.dim + 1)

    def state_dict(self):
        """torch.nn.GRU(H, H)'s / torch.nn.LSTM(H, H)'s parameter names and shapes (CPU fp32 tensors)."""
        ih, hh = self._theta('ih').cpu(), self._theta('hh').cpu()
        H = self.dim
        return {'weight_ih_l0': ih[:, :H].clone(), 'weight_hh_l0': hh[:, :H].clone(), 'bias_ih_l0': ih[:, H].clone(),
                'bias_hh_l0': hh[:, H].clone()}

    def load_state_dict(self, sd):
        H, GH = self.dim, self.GATES * self.dim
        a = self._load_arrays(sd, {'weight_ih_l0': (GH, H), 'weight_hh_l0': (GH, H), 'bias_ih_l0': (GH,), 'bias_hh_l0': (GH,)})
        for g in ('ih', 'hh'):
            t = np.concatenate([a['weight_%s_l0' % g], a['bias_%s_l0' % g][:, None]], 1)
            self._theta(g).copy_(torch.from_numpy(t))
        self._reset_slots()
        self._hh_valid = False

    @staticmethod
    def _dim_of(z):
        return int(z['weight_hh_l0'].shape[1])

    def _files(self):
        f = super()._files()
        if self._lt is not None:
            f.update(long_term_users=self.long_term_users, long_term=self.long_term.cpu().numpy())
        return f

    @classmethod
    def load(cls, path, **kw):
        """As _UserEncoder.load; a file with a long-term table (long_term_users and long_term) restores it."""
        z = np.load(path)
        if 'long_term_users' in z.files:
            kw.setdefault('long_term_users', int(z['long_term_users']))
        m = super().load(path, **kw)
        if m._lt is not None and 'long_term' in z.files:
            P = z['long_term']
            if P.shape != tuple(m.long_term.shape):
                raise ValueError('%s.load: %s holds a long-term table of shape %s, the model has %s' % (
                    cls.__name__, path, P.shape, tuple(m.long_term.shape)))
            m.long_term.copy_(torch.from_numpy(P.astype(np.float32)))
        return m

    def fit(self, sequences, embeddings, impressions=None):
        """_UserEncoder.fit; with the long-term table the sequences may hold at most long_term_users rows (ValueError before any
        device work otherwise)."""
        if self._lt is not None:
            try:
                n_u = len(sequences[0]) - 1
            except (TypeError, IndexError, KeyError):
                n_u = 0      # malformed: check_sequences reports it
            if n_u > self.long_term_users:
                raise ValueError('%s.fit: the sequences hold %d users, the long-term table %d rows (long_term_users)' % (
                    type(self).__name__, n_u, self.long_term_users))
        return super().fit(sequences, embeddings, impressions)

    # ---- device helpers ---------------------------------------------------------------------------------------------------
    def _split(self, g):
        hi, lo = self.W_hl[g]
        call('dae_split_bf16', self._theta(g).data_ptr(), self.GATES * self.dim, self.dim + 1, self.dim + 1, hi.data_ptr(), lo.data_ptr(),
             self.ldx, -1, 1.0, _stream())

    def _buffers(self, P, B):
        """Training buffers for P positions and B users (grown, never shrunk)."""
        if P <= self._cap[0] and B <= self._cap[1]:
            return self._buf
        P, B = max(P, self._cap[0]), max(B, self._cap[1])
        H, GH, d = self.dim, self.GATES * self.dim, self.device
        f32, bf, i32 = dict(dtype=torch.float32, device=d), dict(dtype=torch.bfloat16, device=d), dict(dtype=torch.int32, device=d)
        self._buf = None
        torch.cuda.empty_cache()
        b = {'neg': torch.empty(P, **i32),
             'X_hl': (torch.empty(P, self.ldx, **bf), torch.empty(P, self.ldx, **bf)),
             'XP': torch.empty(P, GH, **f32),
             'Hp_hl': (torch.zeros(P, self.ldx, **bf), torch.zeros(P, self.ldx, **bf)),   # [h_{t-1} | 1] of every position
             'HP': torch.empty(B, GH, **f32),
             'Hs': torch.empty(P, H, **f32),
             'gates': torch.empty(P, 4 * H, **f32),
             'dH': torch.empty(P, H, **f32),
             'carry': torch.empty(B, H, **f32)}
        b.update(self._cell_buffers(P, B))
        if self._lt is not None:
            b['h0'] = torch.empty(B, H, **f32)     # fp32 h_0 of the batch's users
        b['Hp_hl'][0][:, H] = 1.0
        self._buf, self._cap = b, (P, B)
        return b

    # ---- training ---------------------------------------------------------------------------------------------------------
    def _refresh(self):
        if not self._hh_valid:
            self._split('hh')
            self._hh_valid = True

    def _forward_backward(self, pk, emb, epoch, batch, ib=None, art=None):
        if self._lt is not None:   # per user of the batch: the row h_0 comes from (masked: the zero row) and the row to update (-1)
            keep = self.long_term_kept(epoch)[pk.order]
            rows = np.stack([np.where(keep, pk.order, self.long_term_users), np.where(keep, pk.order, -1)]).astype(np.int32)
            self._lt_batch = (_upload(rows, self.device), pk.B)
        super()._forward_backward(pk, emb, epoch, batch, ib, art)

    def _optimizer_step(self):
        """theta's step, then with the long-term table the row step of the batch's unmasked users from dL/dh_0 (the carry)."""
        super()._optimizer_step()
        if self._lt is not None:
            rows, n = self._lt_batch
            sparse_optim.rows_step(self._lt, self._lt_slot1, self._lt_slot2, self._lt_count, rows[1], n, self._buf['carry'], self.opt,
                                   self.long_term_learning_rate, self.momentum, _stream())
            self._mark('long_term')

    def _forward(self, b, pk, emb, items, st):
        """The input projection of every position, then per step the recurrent GEMM and the cell: b['Hs']."""
        H, GH, P, T = self.dim, self.GATES * self.dim, pk.P, len(pk.n)
        X_hi, X_lo = b['X_hl']
        call('dae_gather_split_bf16', emb.data_ptr(), emb.stride(0), items.data_ptr(), P, H, X_hi.data_ptr(), X_lo.data_ptr(), self.ldx,
             H, st)
        self._split('ih')
        self._gemm(P, GH, H + 1, b['X_hl'], 0, self.W_hl['ih'], 0, b['XP'], GH)
        self._mark('input_projection')
        Hp_hi, Hp_lo = b['Hp_hl']
        n0 = int(pk.n[0])
        if self._lt is None:
            Hp_hi[:n0, :H].zero_()
            Hp_lo[:n0].zero_()
        else:
            self._initial_states(self._lt_batch[0][0], n0, Hp_hi, Hp_lo, b['h0'], st)
        Hs, HP = b['Hs'], b['HP']
        for t in range(T):
            o, n = int(pk.off[t]), int(pk.n[t])
            n_next = int(pk.n[t + 1]) if t + 1 < T else 0
            self._gemm(n, GH, H + 1, (Hp_hi[o:], Hp_lo[o:]), 0, self.W_hl['hh'], 0, HP, GH)
            self._cell_fwd(b, pk, t, n_next, st)
        self._mark('forward_recurrence')

    def _backward(self, b, pk, st):
        """Backpropagation through time from b['dH'], then the two weight GEMMs into self.grad."""
        H, GH, P, T = self.dim, self.GATES * self.dim, pk.P, len(pk.n)
        n0 = int(pk.n[0])
        # rows [n_t, n_{t-1}) of the carries belong to users whose last read is at t - 1: nothing flows into them from later steps,
        # and no later step writes them (step t' > t - 1 writes rows [0, n_t') only), so zeroing rows [0, n_0) once keeps them zero
        for k in self._CARRIES:
            b[k][:n0].zero_()
        carry = b['carry']
        dP_hi, dP_lo = b[self._DGRAD[0]]
        for t in range(T - 1, -1, -1):
            o, n = int(pk.off[t]), int(pk.n[t])
            self._cell_bwd(b, pk, t, st)
            # without the long-term table h_{-1} = 0 is a constant: no carry below step 0; with it the carry leaves dL/dh_0 in carry[:n0]
            if t or self._lt is not None:
                self._gemm(n, H, GH, (dP_hi[o:], dP_lo[o:]), 0, self.W_hl['hh'], 1, carry, H, accumulate=self._CARRY_ACCUMULATE)
        self._mark('backward_recurrence')
        g_hh, g_ih = self.grad[:self.nW], self.grad[self.nW:]
        self._gemm(GH, H + 1, P, b[self._DGRAD[0]], 1, b['Hp_hl'], 1, g_hh, H + 1, k_splits=-1)
        self._gemm(GH, H + 1, P, b[self._DGRAD[1]], 1, b['X_hl'], 1, g_ih, H + 1, k_splits=-1)
        self._mark('weight_gradients')

    def _input_grad(self, b):
        """The input projection's packed gradient, W~_ih's bf16 copy and their inner width: dX = dXP . W_ih."""
        return b[self._DGRAD[1]], self.W_hl['ih'], self.GATES * self.dim

    def _step_split(self):
        hi, lo = self.W_hl['hh']
        self._hh_valid = True
        return hi.data_ptr(), lo.data_ptr(), self.GATES * self.dim, self.dim + 1, self.ldx

    # ---- inference --------------------------------------------------------------------------------------------------------
    def _step_buffers(self, B):
        """transform / impression_states' buffers for batches of up to B users: O(B x GATES H) device memory.  Also refreshes the
        bf16 hi / lo copies of W~_hh (when stale) and W~_ih that the steps read."""
        H, GH, d = self.dim, self.GATES * self.dim, self.device
        if not self._hh_valid:
            self._split('hh')
            self._hh_valid = True
        self._split('ih')
        bf = dict(dtype=torch.bfloat16, device=d)
        s = {'X_hl': (torch.zeros(B, self.ldx, **bf), torch.zeros(B, self.ldx, **bf)),
             'h_hl': (torch.zeros(B, self.ldx, **bf), torch.zeros(B, self.ldx, **bf)),
             'XP': torch.empty(B, GH, dtype=torch.float32, device=d),
             'HP': torch.empty(B, GH, dtype=torch.float32, device=d),
             'h': torch.empty(B, H, dtype=torch.float32, device=d)}
        s.update(self._cell_step_buffers(B))
        return s

    _infer_buffers = _step_buffers

    def _last_states(self, pk, emb, s):
        self._steps(pk, emb, s)
        return s['h'][:pk.B]

    def _run_capture(self, pk, emb, s, cap_step, cap_row, cap_imp, out):
        """Run pk step by step; after step cap_step[j], row cap_row[j] of the states is impression cap_imp[j]'s row of out."""
        o = np.argsort(cap_step, kind='stable')
        cap_step, cap = cap_step[o], np.stack([cap_row[o], cap_imp[o]])
        bounds = np.searchsorted(cap_step, np.arange(len(pk.n) + 1))
        cap_d = _upload(np.ascontiguousarray(cap), self.device)
        h = s['h']

        def capture(tt):
            a, b = int(bounds[tt]), int(bounds[tt + 1])
            if b > a:
                out.index_copy_(0, cap_d[1, a:b], h.index_select(0, cap_d[0, a:b]))
        self._steps(pk, emb, s, capture)

    def _steps(self, pk, emb, s, after=None):
        """Run one packed batch from zero states (h_0 = P[pk.users] with the long-term table), step by step: the input projection of
        the step's reads, the recurrent GEMM and the cell, which updates s['h'] (and the cell's other states) in place.  after(t), if
        given, runs after step t."""
        H, GH, st = self.dim, self.GATES * self.dim, _stream()
        it = _upload(pk.items, self.device)
        h_hi, h_lo = s['h_hl']
        if self._lt is None:
            h_hi.zero_()
            h_lo.zero_()
            h_hi[:, H] = 1.0
        for k in self._STATES:
            s[k][:pk.B].zero_()
        if self._lt is not None:
            self._initial_states(_upload(self._table_rows(pk.users), self.device), pk.B, h_hi, h_lo, s['h'], st)
        X_hi, X_lo = s['X_hl']
        for t in range(len(pk.n)):
            o, n = int(pk.off[t]), int(pk.n[t])
            call('dae_gather_split_bf16', emb.data_ptr(), emb.stride(0), it[o:].data_ptr(), n, H, X_hi.data_ptr(), X_lo.data_ptr(),
                 self.ldx, H, st)
            self._gemm(n, GH, H + 1, (X_hi, X_lo), 0, self.W_hl['ih'], 0, s['XP'], GH)
            self._gemm(n, GH, H + 1, (h_hi, h_lo), 0, self.W_hl['hh'], 0, s['HP'], GH)
            self._step(s, n, st)
            if after is not None:
                after(t)


class UserGRU(_UserRNN):
    """GRU user encoder over reading sequences (torch.nn.GRU's cell, gate order r, z, n); see the module docstring.  Its backward
    writes dXP = [dr^, dz^, dn^] and dHP = [dr^, dz^, r dn^] separately (dHP's n-third differs), and carry <- dh z, onto which the
    carry GEMM accumulates dHP . W_hh."""
    GATES = 3

    def _cell_buffers(self, P, B):
        bf = dict(dtype=torch.bfloat16, device=self.device)
        return {'dXP_hl': (torch.empty(P, self.ldg, **bf), torch.empty(P, self.ldg, **bf)),
                'dHP_hl': (torch.empty(P, self.ldg, **bf), torch.empty(P, self.ldg, **bf))}

    def _cell_fwd(self, b, pk, t, n_next, st):
        H, o, n = self.dim, int(pk.off[t]), int(pk.n[t])
        Hs, XP, HP, G = b['Hs'], b['XP'], b['HP'], b['gates']
        Hp_hi, Hp_lo = b['Hp_hl']
        hprev = Hs[int(pk.off[t - 1]):].data_ptr() if t else self._h0(b)
        nx = int(pk.off[t + 1])
        call('dae_gru_cell_fwd', n, H, XP[o:].data_ptr(), 3 * H, HP.data_ptr(), 3 * H, hprev, H, Hs[o:].data_ptr(), H, n_next,
             Hp_hi[nx:].data_ptr() if n_next else None, Hp_lo[nx:].data_ptr() if n_next else None, self.ldx, G[o:].data_ptr(),
             4 * H, st)

    def _cell_bwd(self, b, pk, t, st):
        H, o, n = self.dim, int(pk.off[t]), int(pk.n[t])
        Hs, dH, G, carry = b['Hs'], b['dH'], b['gates'], b['carry']
        (dX_hi, dX_lo), (dP_hi, dP_lo) = b['dXP_hl'], b['dHP_hl']
        hprev = Hs[int(pk.off[t - 1]):].data_ptr() if t else self._h0(b)
        call('dae_gru_cell_bwd', n, H, dH[o:].data_ptr(), H, carry.data_ptr(), H, G[o:].data_ptr(), 4 * H, hprev, H,
             dX_hi[o:].data_ptr(), dX_lo[o:].data_ptr(), dP_hi[o:].data_ptr(), dP_lo[o:].data_ptr(), self.ldg, st)

    def _cell_step_buffers(self, B):
        return {}

    def _step(self, s, n, st):
        H, h = self.dim, s['h']
        h_hi, h_lo = s['h_hl']
        call('dae_gru_cell_fwd', n, H, s['XP'].data_ptr(), 3 * H, s['HP'].data_ptr(), 3 * H, h.data_ptr(), H, h.data_ptr(), H, n,
             h_hi.data_ptr(), h_lo.data_ptr(), self.ldx, None, 0, st)


class UserLSTM(_UserRNN):
    """LSTM user encoder over reading sequences (DESIGN 4.15): torch.nn.LSTM(H, H)'s cell (one layer, bias, no projection, gate
    order i, f, g, o), h_0 = c_0 = 0 (h_0 = P[u] with the long-term table); the user vector is h after the last (truncated) read.  Everything else -- the constructor,
    the losses and negatives, fit, transform, impression_states, recommend, save / load -- is UserGRU's; theta =
    [W~_hh (4H x (H+1)) | W~_ih (4H x (H+1))].

    Training keeps c_t of every position (Cs) next to h_t, and the gates [i | f | g | o].  The backward writes one packed gradient
    dA = [di | df | dg | do]: the pre-activation is XP + HP, so dXP = dHP = dA feeds both weight GEMMs and the carry GEMM.  The cell
    kernel reads the h carry and the carry GEMM then STORES dh_{t-1}[0, n_t) = dA_t . W_hh over it instead of accumulating: h_{t-1}
    reaches step t only through HP_t (there is no direct h -> h term, unlike the GRU's z h_{t-1}), so once the cell has read the
    carry nothing else contributes to it.  The c carry (carry_c <- dc f) is the cell kernel's own."""
    GATES = 4
    _STATES = ('h', 'c')
    _CARRIES = ('carry', 'carry_c')
    _DGRAD = ('dA_hl', 'dA_hl')
    _CARRY_ACCUMULATE = 0

    def _cell_buffers(self, P, B):
        f32, bf = dict(dtype=torch.float32, device=self.device), dict(dtype=torch.bfloat16, device=self.device)
        return {'Cs': torch.empty(P, self.dim, **f32),
                'carry_c': torch.empty(B, self.dim, **f32),
                'dA_hl': (torch.empty(P, self.ldg, **bf), torch.empty(P, self.ldg, **bf))}

    def _cell_fwd(self, b, pk, t, n_next, st):
        H, o, n = self.dim, int(pk.off[t]), int(pk.n[t])
        Cs = b['Cs']
        Hp_hi, Hp_lo = b['Hp_hl']
        cprev = Cs[int(pk.off[t - 1]):].data_ptr() if t else None
        nx = int(pk.off[t + 1])
        call('dae_lstm_cell_fwd', n, H, b['XP'][o:].data_ptr(), 4 * H, b['HP'].data_ptr(), 4 * H, cprev, H, Cs[o:].data_ptr(), H,
             b['Hs'][o:].data_ptr(), H, n_next, Hp_hi[nx:].data_ptr() if n_next else None, Hp_lo[nx:].data_ptr() if n_next else None,
             self.ldx, b['gates'][o:].data_ptr(), 4 * H, st)

    def _cell_bwd(self, b, pk, t, st):
        H, o, n = self.dim, int(pk.off[t]), int(pk.n[t])
        Cs = b['Cs']
        dA_hi, dA_lo = b['dA_hl']
        cprev = Cs[int(pk.off[t - 1]):].data_ptr() if t else None
        call('dae_lstm_cell_bwd', n, H, b['dH'][o:].data_ptr(), H, b['carry'].data_ptr(), H, b['carry_c'].data_ptr(), H,
             b['gates'][o:].data_ptr(), 4 * H, Cs[o:].data_ptr(), H, cprev, H, dA_hi[o:].data_ptr(), dA_lo[o:].data_ptr(), self.ldg, st)

    def _cell_step_buffers(self, B):
        return {'c': torch.empty(B, self.dim, dtype=torch.float32, device=self.device)}

    def _step(self, s, n, st):
        H, h, c = self.dim, s['h'], s['c']
        h_hi, h_lo = s['h_hl']
        call('dae_lstm_cell_fwd', n, H, s['XP'].data_ptr(), 4 * H, s['HP'].data_ptr(), 4 * H, c.data_ptr(), H, c.data_ptr(), H,
             h.data_ptr(), H, n, h_hi.data_ptr(), h_lo.data_ptr(), self.ldx, None, 0, st)


MAX_ATTENTION_LEN = 1024     # dae_seq_attention_* / dae_seq_pool_*: reads per window
MAX_HEAD_DIM = 128           # dae_seq_attention_*: H / heads
ATTENTION_NAMES = ('self_attn.in_proj_weight', 'self_attn.in_proj_bias', 'self_attn.out_proj.weight', 'self_attn.out_proj.bias',
                   'pool.weight', 'pool.bias', 'pool.query')


def default_heads(dim):
    """The largest divisor of dim that is at most 20 (NRMS's head count): 20 at H = 500, 1 at H = 37."""
    return max(k for k in range(1, min(int(dim), 20) + 1) if dim % k == 0)


class UserAttention(_UserEncoder):
    """NRMS's user encoder over reading sequences, made causal (DESIGN 4.17): for a window of reads with article vectors x_1..x_L,
    m = torch.nn.MultiheadAttention(H, heads, batch_first=True)(x, x, x) with a causal mask (read t attends to reads s <= t), then
    additive pooling a_s = q . tanh(W_a m_s + b_a) and u_t = sum_{s <= t} softmax_{s <= t}(a)_s m_s.  u_t depends only on the
    reads up to t, like an RNN's h_t, so the losses, fit, transform (u_L), impression_states and recommend are the recurrent
    encoders'.  NRMS concatenates the heads without an output projection; this encoder keeps torch's out_proj so that a CPU
    torch.nn.MultiheadAttention loads the self_attn.* parameters.

    heads: None for default_heads(dim); H / heads <= 128.  attention_dim: A >= 1, the pooling width.  max_len <= 1024.
    theta = [W~_in (3H x (H+1)) | W~_out (H x (H+1)) | W~_a (A x (H+1)) | q (A)] with W~ = [W | b], updated by one optimizer step.

    Device path per batch (one pass over every packed position, no step loop): [X | 1] and QKV = [X | 1].W~_in^T;
    dae_seq_attention_fwd (O, its bf16 split and the row log-sum-exps); M = [O | 1].W~_out^T; Z = [M | 1].W~_a^T; dae_seq_pool_fwd
    (Hs).  Backward: dae_seq_pool_bwd (dM's value path, dZ, dq); dM += dZ.W_a; dO = dM.W_out; dae_seq_attention_bwd (dQKV); the
    three weight GEMMs.  Device memory per batch is O(batch positions x (3H + A)), in training and in inference."""
    _CONFIG = ('heads', 'attention_dim')
    _PARAMS = ATTENTION_NAMES

    def __init__(self, dim, heads=None, attention_dim=200, **kw):
        super().__init__(dim, **kw)
        name = type(self).__name__
        H = self.dim
        if heads is None:
            heads = default_heads(H)
        if isinstance(heads, bool) or not isinstance(heads, (int, np.integer)) or heads < 1 or H % heads:
            raise ValueError('%s: heads = %r must be a positive divisor of dim = %d' % (name, heads, H))
        if H // heads > MAX_HEAD_DIM:
            raise ValueError('%s: head dim H / heads = %d exceeds %d' % (name, H // heads, MAX_HEAD_DIM))
        if isinstance(attention_dim, bool) or not isinstance(attention_dim, (int, np.integer)) or attention_dim < 1:
            raise ValueError('%s: attention_dim = %r must be an integer >= 1' % (name, attention_dim))
        if self.max_len > MAX_ATTENTION_LEN:
            raise ValueError('%s: max_len = %d exceeds %d' % (name, self.max_len, MAX_ATTENTION_LEN))
        self.heads, self.attention_dim = int(heads), int(attention_dim)
        A = self.attention_dim
        self.ldx, self.ld3, self.lda = _ld8(H + 1), _ld8(3 * H), _ld8(A)
        self._rows = {'in': 3 * H, 'out': H, 'pool': A}
        self._off = {'in': 0, 'out': 3 * H * (H + 1), 'pool': 4 * H * (H + 1), 'query': (4 * H + A) * (H + 1)}
        # torch.nn.MultiheadAttention's initialisation (Xavier-uniform in_proj, out_proj uniform +-1/sqrt(H), zero biases) and NRMS's
        # pooling layer's (Glorot-uniform W_a [A x H] and q [A x 1], zero b_a), drawn in that order
        rng = np.random.default_rng(self.seed)
        w_in = rng.uniform(-1.0, 1.0, (3 * H, H)) * np.sqrt(6.0 / (4 * H))
        w_out = rng.uniform(-1.0, 1.0, (H, H)) / np.sqrt(H)
        w_a = rng.uniform(-1.0, 1.0, (A, H)) * np.sqrt(6.0 / (A + H))
        q = rng.uniform(-1.0, 1.0, A) * np.sqrt(6.0 / (A + 1))
        pad = lambda w: np.concatenate([w, np.zeros((w.shape[0], 1))], 1).ravel()   # noqa: E731
        self._set_theta(np.concatenate([pad(w_in), pad(w_out), pad(w_a), q]).astype(np.float32))
        bf = dict(dtype=torch.bfloat16, device=self.device)
        self.W_hl = {g: (torch.zeros(r, self.ldx, **bf), torch.zeros(r, self.ldx, **bf)) for g, r in self._rows.items()}

    # ---- parameters -------------------------------------------------------------------------------------------------------
    def _theta(self, g, t=None):
        """W~_g = [W_g | b_g] as a [rows, H+1] view of theta (g = 'in', 'out' or 'pool'), or q [A] (g = 'query'); t: theta or grad."""
        t = self.theta if t is None else t
        o = self._off[g]
        if g == 'query':
            return t[o:o + self.attention_dim]
        return t[o:o + self._rows[g] * (self.dim + 1)].view(self._rows[g], self.dim + 1)

    def state_dict(self):
        """torch.nn.MultiheadAttention's names under 'self_attn.' and the pooling layer's under 'pool.' (CPU fp32 tensors)."""
        H = self.dim
        w = {g: self._theta(g).cpu() for g in ('in', 'out', 'pool')}
        return {'self_attn.in_proj_weight': w['in'][:, :H].clone(), 'self_attn.in_proj_bias': w['in'][:, H].clone(),
                'self_attn.out_proj.weight': w['out'][:, :H].clone(), 'self_attn.out_proj.bias': w['out'][:, H].clone(),
                'pool.weight': w['pool'][:, :H].clone(), 'pool.bias': w['pool'][:, H].clone(),
                'pool.query': self._theta('query').cpu().clone()}

    def load_state_dict(self, sd):
        H, A = self.dim, self.attention_dim
        a = self._load_arrays(sd, {'self_attn.in_proj_weight': (3 * H, H), 'self_attn.in_proj_bias': (3 * H,),
                                   'self_attn.out_proj.weight': (H, H), 'self_attn.out_proj.bias': (H,), 'pool.weight': (A, H),
                                   'pool.bias': (A,), 'pool.query': (A,)})
        for g, (wk, bk) in (('in', ('self_attn.in_proj_weight', 'self_attn.in_proj_bias')),
                            ('out', ('self_attn.out_proj.weight', 'self_attn.out_proj.bias')), ('pool', ('pool.weight', 'pool.bias'))):
            self._theta(g).copy_(torch.from_numpy(np.concatenate([a[wk], a[bk][:, None]], 1)))
        self._theta('query').copy_(torch.from_numpy(a['pool.query']))
        self._reset_slots()

    @staticmethod
    def _dim_of(z):
        return int(z['self_attn.out_proj.weight'].shape[0])

    # ---- device helpers ---------------------------------------------------------------------------------------------------
    def _buffers(self, P, B):
        """Buffers for P positions and B users (grown, never shrunk): O(P x (3H + A))."""
        if P <= self._cap[0] and B <= self._cap[1]:
            return self._buf
        P, B = max(P, self._cap[0]), max(B, self._cap[1])
        H, A, d = self.dim, self.attention_dim, self.device
        f32, bf, i32 = dict(dtype=torch.float32, device=d), dict(dtype=torch.bfloat16, device=d), dict(dtype=torch.int32, device=d)
        pair = lambda ld: (torch.zeros(P, ld, **bf), torch.zeros(P, ld, **bf))   # noqa: E731
        self._buf = None
        torch.cuda.empty_cache()
        b = {'neg': torch.empty(P, **i32), 'X_hl': pair(self.ldx), 'QKV': torch.empty(P, 3 * H, **f32), 'O': torch.empty(P, H, **f32),
             'O_hl': pair(self.ldx), 'lse': torch.empty(P, self.heads, **f32), 'M': torch.empty(P, H, **f32), 'M_hl': pair(self.ldx),
             'Z': torch.empty(P, A, **f32), 'score': torch.empty(P, **f32), 'plse': torch.empty(P, **f32),
             'Hs': torch.empty(P, H, **f32), 'dH': torch.empty(P, H, **f32), 'dM': torch.empty(P, H, **f32), 'dM_hl': pair(self.ldx),
             'dZ_hl': pair(self.lda), 'dO': torch.empty(P, H, **f32), 'dQKV_hl': pair(self.ld3), 'ws': torch.empty(B, A, **f32)}
        b['O_hl'][0][:, H] = 1.0      # [O | 1]: the kernel writes columns [0, H)
        self._buf, self._cap = b, (P, B)
        return b

    def _refresh(self):
        """The bf16 hi / lo operands of W~_in, W~_out and W~_a from theta."""
        for g, r in self._rows.items():
            hi, lo = self.W_hl[g]
            call('dae_split_bf16', self._theta(g).data_ptr(), r, self.dim + 1, self.dim + 1, hi.data_ptr(), lo.data_ptr(), self.ldx, -1,
                 1.0, _stream())

    def _layout(self, pk):
        """off (int64 [T + 1]) and the users' window lengths (int32 [B]) on the device, and T."""
        return (_upload(pk.off.astype(np.int64), self.device), _upload(pk.L.astype(np.int32), self.device), len(pk.n))

    # ---- training ---------------------------------------------------------------------------------------------------------
    def _forward(self, b, pk, emb, items, st):
        H, A, P = self.dim, self.attention_dim, pk.P
        self._dev_layout = off, lens, T = self._layout(pk)
        X_hi, X_lo = b['X_hl']
        call('dae_gather_split_bf16', emb.data_ptr(), emb.stride(0), items.data_ptr(), P, H, X_hi.data_ptr(), X_lo.data_ptr(), self.ldx,
             H, st)
        self._gemm(P, 3 * H, H + 1, b['X_hl'], 0, self.W_hl['in'], 0, b['QKV'], 3 * H)
        self._mark('input_projection')
        O_hi, O_lo = b['O_hl']
        call('dae_seq_attention_fwd', pk.B, T, off.data_ptr(), lens.data_ptr(), H, self.heads, b['QKV'].data_ptr(), 3 * H,
             b['O'].data_ptr(), H, O_hi.data_ptr(), O_lo.data_ptr(), self.ldx, b['lse'].data_ptr(), self.heads, st)
        self._mark('attention')
        self._gemm(P, H, H + 1, b['O_hl'], 0, self.W_hl['out'], 0, b['M'], H)
        M_hi, M_lo = b['M_hl']
        call('dae_split_bf16', b['M'].data_ptr(), P, H, H, M_hi.data_ptr(), M_lo.data_ptr(), self.ldx, H, 1.0, st)
        self._gemm(P, A, H + 1, b['M_hl'], 0, self.W_hl['pool'], 0, b['Z'], A)
        self._mark('output_projection')
        call('dae_seq_pool_fwd', pk.B, T, off.data_ptr(), lens.data_ptr(), H, A, b['Z'].data_ptr(), A, self._theta('query').data_ptr(),
             b['M'].data_ptr(), H, b['Hs'].data_ptr(), H, b['score'].data_ptr(), b['plse'].data_ptr(), st)
        self._mark('pooling')

    def _backward(self, b, pk, st):
        H, A, P = self.dim, self.attention_dim, pk.P
        off, lens, T = self._dev_layout
        dZ_hi, dZ_lo = b['dZ_hl']
        call('dae_seq_pool_bwd', pk.B, T, off.data_ptr(), lens.data_ptr(), H, A, b['dH'].data_ptr(), H, b['Hs'].data_ptr(), H,
             b['M'].data_ptr(), H, b['Z'].data_ptr(), A, self._theta('query').data_ptr(), b['score'].data_ptr(), b['plse'].data_ptr(),
             b['dM'].data_ptr(), H, dZ_hi.data_ptr(), dZ_lo.data_ptr(), self.lda, self._theta('query', self.grad).data_ptr(),
             b['ws'].data_ptr(), st)
        self._gemm(P, H, A, b['dZ_hl'], 0, self.W_hl['pool'], 1, b['dM'], H, accumulate=1)
        dM_hi, dM_lo = b['dM_hl']
        call('dae_split_bf16', b['dM'].data_ptr(), P, H, H, dM_hi.data_ptr(), dM_lo.data_ptr(), self.ldx, -1, 1.0, st)
        self._mark('pooling_backward')
        self._gemm(P, H, H, b['dM_hl'], 0, self.W_hl['out'], 1, b['dO'], H)
        dQ_hi, dQ_lo = b['dQKV_hl']
        call('dae_seq_attention_bwd', pk.B, T, off.data_ptr(), lens.data_ptr(), H, self.heads, b['QKV'].data_ptr(), 3 * H,
             b['O'].data_ptr(), H, b['lse'].data_ptr(), self.heads, b['dO'].data_ptr(), H, dQ_hi.data_ptr(), dQ_lo.data_ptr(), self.ld3,
             st)
        self._mark('attention_backward')
        for g, dA, Bop in (('in', 'dQKV_hl', 'X_hl'), ('out', 'dM_hl', 'O_hl'), ('pool', 'dZ_hl', 'M_hl')):
            self._gemm(self._rows[g], H + 1, P, b[dA], 1, b[Bop], 1, self._theta(g, self.grad), H + 1, k_splits=-1)
        self._mark('weight_gradients')

    def _input_grad(self, b):
        return b['dQKV_hl'], self.W_hl['in'], 3 * self.dim

    def _step_split(self):
        return None, None, 0, 0, 0

    # ---- inference --------------------------------------------------------------------------------------------------------
    def _infer_buffers(self, B):
        self._refresh()
        return None

    def _states(self, pk, emb):
        """Hs of every position of pk (one forward pass)."""
        b = self._buffers(pk.P, pk.B)
        self._forward(b, pk, emb, _upload(pk.items, self.device), _stream())
        return b['Hs']

    def _last_states(self, pk, emb, s):
        last = pk.off[pk.L - 1] + np.arange(pk.B)
        return self._states(pk, emb).index_select(0, _upload(last.astype(np.int64), self.device))

    def _run_capture(self, pk, emb, s, cap_step, cap_row, cap_imp, out):
        cap = _upload(np.stack([pk.off[cap_step] + cap_row, cap_imp]).astype(np.int64), self.device)
        out.index_copy_(0, cap[1], self._states(pk, emb).index_select(0, cap[0]))


def history_matrix(indptr, items, n_items):
    """The users' read articles as a scipy CSR [U, n_items] with 1 per article read (helpers.recommend's histories).  Built on
    copies: scipy sorts the arrays it is given in place."""
    import scipy.sparse as sp
    m = sp.csr_matrix((np.ones(len(items), np.float32), np.array(items), np.array(indptr)), shape=(len(indptr) - 1, n_items))
    m.sum_duplicates()
    m.data[:] = 1.0
    return m


def prefix_histories(sequences, impressions, n_items):
    """The reads before each impression as a scipy CSR [I, n_items] with 1 per article read (history_matrix of the prefixes
    items[indptr[user] : indptr[user] + time], whole, not truncated to max_len): the histories of the mean-profile baseline,
    helpers.user_profiles(prefix_histories(...), embeddings)."""
    indptr, items = check_sequences(sequences, n_items, 'prefix_histories')
    imp = check_impressions(impressions, n_items, 'prefix_histories', indptr)
    t = imp['time']
    p_indptr = np.concatenate([[0], np.cumsum(t)]).astype(np.int64)
    src = np.repeat(indptr[imp['user']] - p_indptr[:-1], t) + np.arange(int(p_indptr[-1]))
    return history_matrix(p_indptr, items[src], n_items)


def negatives_from_draws(pos, c, n_items):
    """dae_seq_negatives' map from the 32-bit Philox draw c to the negative of positive `pos`: (pos + 1 + floor(c (N - 1) / 2^32)) mod N."""
    pos, c = np.asarray(pos, np.int64), np.asarray(c, np.uint64)
    return ((pos + 1 + ((c * np.uint64(n_items - 1)) >> np.uint64(32)).astype(np.int64)) % n_items).astype(np.int32)
