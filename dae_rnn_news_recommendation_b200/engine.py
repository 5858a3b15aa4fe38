"""Device-side training/encoding engine: owns the torch buffers and sequences the C-ABI kernels of
libdae_sm100.so for one training step (the replacement of `tf_session.run([train_step, losses...])`,
reference autoencoder/autoencoder.py:233,241) and for `transform` (:494-497).

PyTorch is plumbing here (device memory, streams, torch.distributed); every arithmetic op of the hot path is a
kernel from the library.  There is no CPU path.
"""
import ctypes
import os

import numpy as np
import scipy.sparse as sp
import torch

from . import _cabi
from ._cabi import call, ptr, STAT, STAT_SLOTS

_BATCH_ALL, _BATCH_HARD, _EXPLICIT = (_cabi.STRATEGY[k] for k in ('batch_all', 'batch_hard', 'explicit'))
_COSINE = _cabi.LOSS['cosine_proximity']


def _stream():
    return torch.cuda.current_stream().cuda_stream


def canonical_csr(x):
    """scipy sparse / ndarray -> canonical CSR (sorted, no duplicates), fp32 values, like the feed built by
    utils.get_sparse_ind_val_shape (autoencoder/utils.py:171-178)."""
    if isinstance(x, np.ndarray):
        m = sp.csr_matrix(x)
    else:
        m = sp.csr_matrix(x)
    if not m.has_canonical_format:
        m = m.copy()
        m.sum_duplicates()
    m.sort_indices()
    return m


def canonical_values(x, values, m):
    """values: one value per stored entry of x, in x's own entry order (the storage order of a CSR / CSC / COO matrix, the row-major
    nonzeros of an ndarray) -> those values in the entry order of m = canonical_csr(x), summed where x holds duplicate entries as m's
    values are: the corrupted copy of a batch lands on the columns of the clean entries it was drawn from."""
    v = np.asarray(values, dtype=np.float32).reshape(-1)
    if sp.issparse(x) and x.format == 'csr' and x.has_canonical_format:
        if v.size != m.nnz:
            raise ValueError('x_corr_values: %d values for %d stored entries' % (v.size, m.nnz))
        return v
    c = sp.coo_matrix(x)
    if v.size != c.nnz:
        raise ValueError('x_corr_values: %d values for %d stored entries' % (v.size, c.nnz))
    mc = canonical_csr(sp.coo_matrix((v, (c.row, c.col)), shape=c.shape))
    assert np.array_equal(mc.indptr, m.indptr) and np.array_equal(mc.indices, m.indices)
    return mc.data


class DeviceCSR:
    """CSR matrix resident in HBM: indptr int64[N+1], indices int32[nnz], values fp32[nnz]."""

    def __init__(self, m, device, pin=False):
        m = canonical_csr(m)
        self.shape = m.shape
        self.nnz = int(m.nnz)
        self.max_row_nnz = int(np.diff(m.indptr).max()) if m.shape[0] else 0
        ip = torch.from_numpy(m.indptr.astype(np.int64))
        ix = torch.from_numpy(m.indices.astype(np.int32))
        va = torch.from_numpy(m.data.astype(np.float32))
        if pin:
            ip, ix, va = ip.pin_memory(), ix.pin_memory(), va.pin_memory()
        self.h2d_bytes = ip.numel() * 8 + ix.numel() * 4 + va.numel() * 4
        self.indptr = ip.to(device, non_blocking=True)
        self.indices = ix.to(device, non_blocking=True)
        self.values = va.to(device, non_blocking=True)

    @staticmethod
    def from_tensors(indptr, indices, values, shape):
        """A DeviceCSR over device tensors that already hold a canonical CSR (int64 indptr, int32 indices, fp32 values)."""
        m = DeviceCSR.__new__(DeviceCSR)
        m.shape, m.nnz, m.h2d_bytes = tuple(shape), int(indices.numel()), 0
        m.max_row_nnz = int((indptr[1:] - indptr[:-1]).max()) if shape[0] else 0
        m.indptr, m.indices, m.values = indptr, indices, values
        return m

    @staticmethod
    def vstack(mats, device):
        return DeviceCSR(sp.vstack([canonical_csr(m) for m in mats]).tocsr(), device)


class HostFeed:
    """One step's inputs packed into ONE pinned host buffer (what `feed_dict` is to the reference's session.run,
    autoencoder/autoencoder.py:228): [indptr int64 | indices int32 | values f32 | corrupted values f32 | labels f32]."""

    def __init__(self, x_batch, x_corr_values, labels, cap_nnz=None):
        """x_corr_values: the corrupted values, one per stored entry of x_batch in its own entry order (canonical_values), or None (the
        clean values).  cap_nnz: lay the buffer out for up to cap_nnz stored entries, so that every feed of a run has the SAME device
        layout and the step can be replayed from one captured CUDA graph."""
        m = canonical_csr(x_batch)
        B, real_nnz = m.shape[0], int(m.nnz)
        assert cap_nnz is None or cap_nnz >= real_nnz
        self.cap_nnz = cap_nnz
        nnz = real_nnz if cap_nnz is None else int(cap_nnz)   # layout size
        self.B, self.nnz, self.F = B, nnz, m.shape[1]

        def al(n):
            return (n + 15) // 16 * 16
        self.off_indptr = 0
        self.off_indices = al(8 * (B + 1))
        self.off_values = self.off_indices + al(4 * nnz)
        self.off_values_c = self.off_values + al(4 * nnz)
        self.off_labels = self.off_values_c + al(4 * nnz)
        self.nbytes = self.off_labels + al(4 * B)
        self.host = torch.empty(self.nbytes, dtype=torch.uint8).pin_memory()
        hb = self.host.numpy()
        hb[self.off_indptr:self.off_indptr + 8 * (B + 1)] = m.indptr.astype(np.int64).view(np.uint8)
        hb[self.off_indices:self.off_indices + 4 * real_nnz] = m.indices.astype(np.int32).view(np.uint8)
        hb[self.off_values:self.off_values + 4 * real_nnz] = m.data.astype(np.float32).view(np.uint8)
        xc = m.data if x_corr_values is None else canonical_values(x_batch, x_corr_values, m)
        hb[self.off_values_c:self.off_values_c + 4 * real_nnz] = np.asarray(xc, dtype=np.float32).view(np.uint8)
        lab = np.zeros(B, np.float32) if labels is None else np.asarray(labels, dtype=np.float32).reshape(-1)
        hb[self.off_labels:self.off_labels + 4 * B] = lab.view(np.uint8)
        self.has_labels = labels is not None


class _CSRView:
    def __init__(self, indptr, indices, values, shape):
        self.indptr, self.indices, self.values, self.shape, self.nnz = indptr, indices, values, shape, values.numel()
        self.max_row_nnz = None


def resolve_deterministic(deterministic):
    """deterministic: True / False, or None = the environment variable DAE_DETERMINISTIC ('1' turns the mode on)."""
    if deterministic is None:
        return os.environ.get('DAE_DETERMINISTIC', '0') == '1'
    return bool(deterministic)


def check_deterministic_supported(gemm=None, process_group=None):
    """The deterministic mode covers the tensor-core path of one process; anything else is refused before any buffer exists."""
    mode = gemm or os.environ.get('DAE_GEMM', 'tc')
    if mode != 'tc':
        raise ValueError("deterministic=True needs the tensor-core path (gemm='tc', got %r): the fp32 CUDA-core validation kernels "
                         "add split-K partials and column sums with atomics" % (mode,))
    world = 1
    if process_group is not None or (torch.distributed.is_available() and torch.distributed.is_initialized()):
        world = torch.distributed.get_world_size(process_group)
    if world > 1:
        raise ValueError('deterministic=True runs in one process only (world size %d): the gradient exchange across ranks has no '
                         'fixed summation order' % world)


def check_mining_block_rows(R):
    """mining_block_rows: None (the B x B mining buffers, batches up to MAX_TRIPLET_BATCH rows) or the anchor rows R of S held at once
    (batches up to MAX_BLOCKED_BATCH rows): a multiple of 128 (the Gram block's TMA base and tiles stay aligned) in [128, 32768]."""
    if R is None:
        return None
    if isinstance(R, bool) or int(R) != R or not (128 <= int(R) <= 32768 and int(R) % 128 == 0):
        raise ValueError('mining_block_rows must be None or a multiple of 128 in [128, 32768] (got %r)' % (R,))
    return int(R)


class TrainEngine:
    """Flat parameters + per-batch workspaces + the kernel sequence of one step."""

    def __init__(self, n_features, n_components, enc_act_func='sigmoid', dec_act_func='sigmoid',
                 loss_func='cross_entropy', opt='gradient_descent', learning_rate=0.1, momentum=0.5, alpha=1.0,
                 triplet_strategy='batch_all', device='cuda:0', process_group=None, gemm=None, allreduce=None,
                 mining_block_rows=None, deterministic=None):
        """mining_block_rows: None = batch_all / batch_hard mine the whole B x B similarity matrix at once (12 B^2 bytes, batches up to
        MAX_TRIPLET_BATCH rows); R = they mine it R anchor rows at a time (12 R B bytes, batches up to MAX_BLOCKED_BATCH rows;
        tensor-core path only).
        deterministic: True = every floating-point sum of the step runs in a fixed order, so the same seed, inputs, build and GPU model
        give bit-identical parameters, optimizer slots, per-step scalars and transform output on every run (DESIGN 4.7); False = the
        atomic kernels (faster); None (default) = the environment variable DAE_DETERMINISTIC ('1' = on).  Tensor-core path and one
        process only."""
        self.block_rows = check_mining_block_rows(mining_block_rows)
        self.deterministic = resolve_deterministic(deterministic)
        if self.deterministic:
            check_deterministic_supported(gemm, process_group)
        _cabi.lib()  # fail loudly if the CUDA library is missing
        if not torch.cuda.is_available():
            raise _cabi.DaeError('no CUDA device: the DAE hot path has no CPU fallback')
        self.device = torch.device(device)
        self.F, self.H = int(n_features), int(n_components)
        self.enc_act = _cabi.act_code(enc_act_func)
        self.dec_act = _cabi.act_code(dec_act_func)
        self.loss = _cabi.LOSS[loss_func]
        self.opt = _cabi.OPT[opt]
        self.strategy = _cabi.STRATEGY[triplet_strategy]
        self.lr, self.momentum, self.alpha = float(learning_rate), float(momentum), float(alpha)
        self.pg = process_group
        self.world = 1
        if process_group is not None or (torch.distributed.is_available() and torch.distributed.is_initialized()):
            self.world = torch.distributed.get_world_size(process_group)
        n = self.F * self.H + self.H + self.F
        self.n_params = n
        f32 = dict(dtype=torch.float32, device=self.device)
        self.theta = torch.zeros(n, **f32)
        self.grad = torch.zeros(n, **f32)
        self.slot1 = torch.full((n,), 0.1 if opt == 'ada_grad' else 0.0, **f32) if opt != 'gradient_descent' else None
        self.slot2 = torch.zeros(n, **f32) if opt == 'adam' else None
        self.step_count = 0
        self.stats = torch.zeros(STAT_SLOTS, dtype=torch.float64, device=self.device)
        self._ws_B = 0
        self._w_split_valid = False
        # dense contractions: 'tc' = wgmma bf16x3 kernels (production), 'ffma' = fp32 CUDA-core validation kernels.  The two small
        # contractions of the mining branch (S = E.E^T, dE2 = alpha (G + G^T) E; 0.64 GFLOP each) follow it: on the tensor cores the
        # fp32 CUDA-core kernel would co-reside with the persistent tensor-core CTAs (17 KB of shared memory) but is several times
        # slower on these shapes
        self.gemm_mode = gemm or os.environ.get('DAE_GEMM', 'tc')
        assert self.gemm_mode in ('tc', 'ffma')
        if self.block_rows is not None:
            assert self.gemm_mode == 'tc', 'mining_block_rows needs the tensor-core path (gemm="tc")'
        # the batch preparation exports of this engine: the block-mined one accepts batches above MAX_TRIPLET_BATCH
        self._prepare = 'dae_batch_prepare' if self.block_rows is None else 'dae_batch_prepare_blocked'
        self._prepare_next = 'dae_batch_prepare_next' if self.block_rows is None else 'dae_batch_prepare_next_blocked'
        # encode backward: 'gather' = column-bucketed, atomic-free dW accumulation; 'atomic' = red.global.add per entry
        self.enc_bwd_mode = 'gather'
        if self.H > (1024 if self.H % 4 == 0 else (512 if self.H % 2 == 0 else 256)):
            self.enc_bwd_mode = 'atomic'
        if self.deterministic:   # stable column buckets, fixed-order sums (any H)
            self.enc_bwd_mode = 'det'
        self._ent_cap = 0
        self.fork_branches = True   # parallel branches of the step (False: one stream, what the per-kernel timing pass uses)
        self._sides = [None, None]
        self.Hp = (self.H + 1 + 63) // 64 * 64   # K padding of E / W (+1: the all-ones column that turns dW into [dW | dbv])
        self.Fp = (self.F + 31) // 32 * 32
        self.in_scale = 1.0  # decay noise folds into the encode kernels (utils.decay_noise, autoencoder/utils.py:147-159)
        self.launches = 0  # kernels launched by this engine (bench.py reports it)
        self.timed = None  # {kernel name: [(start_event, end_event), ...]} when per-kernel timing is on
        # the data binding (set_data, corrupt_*, _feed_bind)
        self.csr = self.csr_c = self.values_c = self.labels = None
        # per-batch workspaces, sized by _ensure_ws for _ws_B rows (S, G and the GG pair: mining strategies; the bf16 operands and
        # tile_ptr: tensor-core path; gemm_ws, loss_parts, loss_slots: deterministic mode)
        self.E = self.dE = self.dE2 = self.row_loss = self.weight = self.rows = self.labels_b = self.seg_lo = self.seg_hi = None
        if self.loss == _COSINE or self.gemm_mode != 'tc':   # the other engines never hold Z = E.W^T (F floats per batch row)
            self.Z = None
        self._stage = self.S = self.G = self.GG_hi = self.GG_lo = None
        self.E_hi = self.E_lo = self.dZ_hi = self.dZ_lo = self.tile_ptr = self.W_hi = self.W_lo = None
        self.Bp = self.n_loss_parts = 0
        self.gemm_ws = self.loss_parts = self.loss_slots = None
        # scratch of the encode backward (_ensure_bucket_scratch), the salt-and-pepper buffers, the SM count
        self.col_count = self.col_start = self.col_cursor = self.ent_col = self.ent_row = self.ent_val = self.enc_det_ws = None
        self._sp = self._sms = None
        # graph replay: the fit's step graph (+ the optimizer graph of the 'nccl' exchange) and what it was captured on, the device
        # cursors ctl and the step's view of them (_ctl: ctl when the running step is captured, else None), the host feeds' graphs
        self._graph = self._graph2 = self._graph_meta = None
        self.graph_launches = None
        self.ctl = self._ctl = None
        self._ctl_owner = None
        self._ctl_host, self._ctl_host_i = None, 0
        self._feed_dev = None
        self._feed_graph = None
        self._feed_stream = None
        self._labels_next = None
        self._mm = None   # the multimem exchange's symmetric-memory handles
        self._stats_host = torch.empty(STAT_SLOTS, dtype=torch.float64).pin_memory()
        # gradient exchange of the data-parallel step: 'multimem' = in-switch reduction by dae_allreduce_multimem (a plain kernel,
        # captured inside the step's graph; needs NVSwitch multicast); 'nccl_graph' = the NCCL all-reduce captured inside the step's
        # graph; 'auto' (default) = multimem where the multicast rendezvous succeeds on every rank, else nccl_graph; 'nccl' = the
        # round-1 scheme, an eager ncclAllReduce between two captured graphs.
        self.allreduce_mode = (allreduce or os.environ.get('DAE_ALLREDUCE', 'auto')) if self.world > 1 else 'none'
        assert self.allreduce_mode in ('none', 'auto', 'nccl', 'nccl_graph', 'multimem')
        if self.allreduce_mode == 'auto':      # in-switch exchange where the fabric offers multicast, NCCL inside the graph otherwise
            try:
                self._setup_multimem()
                ok = 1
            except Exception:   # noqa: BLE001 -- no multicast / symmetric memory on this fabric
                ok = 0
            flag = torch.tensor([ok], dtype=torch.int32, device=self.device)
            torch.distributed.all_reduce(flag, op=torch.distributed.ReduceOp.MIN, group=self.pg)   # all ranks take the same path
            self.allreduce_mode = 'multimem' if int(flag.item()) == 1 else 'nccl_graph'
            if self.allreduce_mode != 'multimem' and self._mm is not None:
                self._mm = None
                self.grad = torch.zeros(n, **f32)
        elif self.allreduce_mode == 'multimem':
            self._setup_multimem()

    @property
    def _mines(self):
        """batch_all / batch_hard: the step mines its triplets from the batch's labels."""
        return self.strategy in (_BATCH_ALL, _BATCH_HARD)

    # ---- kernel launch plumbing --------------------------------------------------------------------------------------
    def time_kernels(self, names):
        """Bracket every launch of the named C-ABI entry points with CUDA events on the launching stream."""
        self.timed = None if names is None else {n: [] for n in names}

    def kernel_times_ms(self):
        torch.cuda.synchronize(self.device)
        return {n: [a.elapsed_time(b) for a, b in ev] for n, ev in (self.timed or {}).items()}

    def _k(self, name, *args, n_launch=1, tag=None):
        key = tag or name
        if self.timed is not None and key in self.timed:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call(name, *args)
            b.record()
            self.timed[key].append((a, b))
        else:
            call(name, *args)
        self.launches += n_launch

    # ---- per-step host feed (the session.run(feed_dict) analog) ---------------------------------------------------------
    def run_feed(self, feed, stats_log_row=None):
        """H2D copy of one packed pinned HostFeed, one training step on it, D2H read of the step's scalars.
        Feeds built with a common `cap_nnz` share one device layout: the step is then captured once and replayed."""
        self._check_feed(feed)
        if self._feed_dev is None or self._feed_dev.numel() < feed.nbytes:
            self._feed_dev = torch.empty(max(feed.nbytes, 1 << 20), dtype=torch.uint8, device=self.device)
            self._feed_graph = None
        d = self._feed_dev
        d[:feed.nbytes].copy_(feed.host, non_blocking=True)
        key = (feed.B, feed.nnz, feed.has_labels, feed.F)
        B, explicit_n = self._feed_batch(feed.B)
        fixed = feed.cap_nnz is not None and os.environ.get('DAE_CUDA_GRAPH', '1') == '1'
        if not (fixed and self._feed_graph is not None and self._feed_graph[0] == key):
            self._feed_bind(feed)
            if fixed:   # capture the step on this layout (restores the parameters after its warm-up steps)
                self._feed_graph = (key, *self._capture(None, B, None, 0, None, explicit_n))
                self._ctl_owner = None
        if fixed:
            if self._ctl_owner != 'feed':   # cursors: offset 0 / log row 0 never move (stride 0); the optimizer step advances on the device
                self.ctl.copy_(torch.tensor([0, 0, self.step_count + 1, 0], dtype=torch.int64))
                self._ctl_owner = 'feed'
            self._replay(self._feed_graph[1], self._feed_graph[2])
        else:
            self._step(None, 0, B, stats_log_row, explicit_n=explicit_n)
        self._stats_host.copy_(self.stats, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        s = self._stats_host.numpy()
        return {k: float(s[i]) for k, i in STAT.items()}

    def _check_feed(self, feed):
        """Refuse a feed this engine's step cannot train on, before any device work."""
        if self._mines and not feed.has_labels:
            raise ValueError('triplet strategy %s mines the batch by its labels: this feed has none'
                             % next(k for k, v in _cabi.STRATEGY.items() if v == self.strategy))
        if self.strategy == _EXPLICIT and feed.B % 3 != 0:
            raise ValueError('explicit triplets: the feed holds stacked [org; pos; neg] rows, a multiple of 3 (got %d rows)' % feed.B)

    def _feed_batch(self, rows):
        """(B, explicit_n) of the step on a feed of `rows` rows: explicit triplets stack [org; pos; neg], rows / 3 of each."""
        return (rows // 3, rows // 3) if self.strategy == _EXPLICIT else (rows, None)

    def _feed_bind(self, feed, buf=None):
        """Point the engine's batch views (CSR, corrupted values, labels) at the feed layout inside `buf` (default: run_feed's buffer)."""
        d, B, nnz = (self._feed_dev if buf is None else buf), feed.B, feed.nnz
        v = lambda off, nb, dt: d[off:off + nb].view(dt)
        self.csr = self.csr_c = _CSRView(v(feed.off_indptr, 8 * (B + 1), torch.int64), v(feed.off_indices, 4 * nnz, torch.int32),
                                         v(feed.off_values, 4 * nnz, torch.float32), (B, feed.F))
        self.values_c = v(feed.off_values_c, 4 * nnz, torch.float32)
        self.labels = v(feed.off_labels, 4 * B, torch.float32) if feed.has_labels else None

    def run_feeds(self, feeds):
        """A stream of host feeds (same layout: built with one `cap_nnz`), the input pipeline of a training loop: the H2D copies of the
        next two feeds run on a copy stream while step i computes (three device feed buffers, one captured graph each), the triplet
        strategies prepare feed i+1's batch (label sort, segments, weights) on a side branch of step i, every step's scalars leave
        through an asynchronous D2H copy into a pinned ring, and the host synchronises once, after the last step.  Returns the list
        of per-step stats dicts (identical to calling run_feed on each feed in turn)."""
        feeds = list(feeds)
        if not feeds:
            return []
        f0 = feeds[0]
        assert all(f.cap_nnz is not None and (f.B, f.nnz, f.has_labels, f.F, f.nbytes) == (f0.B, f0.nnz, f0.has_labels, f0.F, f0.nbytes)
                   for f in feeds), 'run_feeds needs feeds of one common layout (HostFeed(..., cap_nnz=...))'
        self._check_feed(f0)
        key = (f0.B, f0.nnz, f0.has_labels, f0.F)
        out = []
        if not (self._feed_graph is not None and self._feed_graph[0] == key and self._feed_dev.numel() >= f0.nbytes):
            out.append(self.run_feed(f0))    # first use of this layout: captures the step on it
            feeds = feeds[1:]
        if self._feed_graph is None:         # graph replay disabled (DAE_CUDA_GRAPH=0): plain per-feed calls
            return out + [self.run_feed(f) for f in feeds]
        n = len(feeds)
        if n == 0:
            return out
        LOG_ROWS = 1024
        if n > LOG_ROWS:                     # the per-step scalars go through a device log of LOG_ROWS rows
            for i in range(0, n, LOG_ROWS):
                out.extend(self.run_feeds(feeds[i:i + LOG_ROWS]))
            return out
        # The streamed loop owns NS = 3 device feed buffers and ONE CAPTURED GRAPH PER BUFFER (the step reads its batch where the H2D
        # copy put it: no device-to-device hop), each writing its scalars into row ctl[1] of a device log.  Step j replays graph
        # j % 3; the H2D copy of feed j+2 runs on the copy stream meanwhile, and so does the D2H copy of step j-1's log row.  Triplet
        # strategies: graph k prepares the NEXT batch (label sort / class segments / data weights, dae_batch_prepare_next, one CTA,
        # ~20 us) on a side branch from the labels inside buffer (k+1) % 3, and starts with the copy-out dae_batch_commit.
        NS = 3
        B, nb = f0.B, f0.nbytes
        staged = self._mines          # (mined feeds carry labels: _check_feed)
        st = self._feed_stream
        if st is None or st['owner'] is not self._feed_graph:
            bufs = [torch.empty(self._feed_dev.numel(), dtype=torch.uint8, device=self.device) for _ in range(NS)]
            for bk in bufs:
                bk[:nb].copy_(self._feed_dev[:nb])       # a valid batch of this layout for the captures' warm-up steps
            log = torch.zeros(LOG_ROWS, STAT_SLOTS, dtype=torch.float64, device=self.device)
            graphs = []
            step_B, explicit_n = self._feed_batch(B)
            try:
                for k in range(NS):
                    self._feed_bind(f0, bufs[k])
                    if staged:
                        self._labels_next = bufs[(k + 1) % NS][f0.off_labels:f0.off_labels + 4 * B].view(torch.float32)
                    # staged: the next batch comes from rows 0..B-1 (stride 0) of the next feed, its labels from self._labels_next
                    graphs.append(self._capture(None, step_B, log, 0, (B, 0) if staged else None, explicit_n))
            finally:
                self._labels_next = None
                self._feed_bind(f0)
            st = self._feed_stream = {'owner': self._feed_graph, 'bufs': bufs, 'log': log, 'graphs': graphs,
                                      'copy_stream': torch.cuda.Stream(device=self.device),
                                      'ring': torch.empty(LOG_ROWS, STAT_SLOTS, dtype=torch.float64).pin_memory()}
        bufs, log, graphs, cs, ring = st['bufs'], st['log'], st['graphs'], st['copy_stream'], st['ring']
        self._set_ctl(0, 0)                  # batch cursor 0 (stride 0), log row 0, optimizer step: continues
        self._ctl_owner = 'feed'
        main = torch.cuda.current_stream()
        ev_copy = [torch.cuda.Event() for _ in range(NS)]
        ev_done = [None] * n

        def issue_copy(j):                   # feed j -> buffer j % NS, once step j-3 (its previous reader) and step j-4's label read are done
            with torch.cuda.stream(cs):
                if j >= NS:
                    cs.wait_event(ev_done[j - NS])
                bufs[j % NS][:nb].copy_(feeds[j].host, non_blocking=True)
                ev_copy[j % NS].record(cs)
        cs.wait_stream(main)                 # (earlier work on the main stream may still read the buffers)
        for j in range(min(n, NS - 1)):
            issue_copy(j)
        for j in range(n):
            k = j % NS
            main.wait_event(ev_copy[k])
            if staged:
                if j == 0:                       # the first step's batch; every later one is staged by the step before it
                    self._feed_bind(f0, bufs[0])
                    self.stage_batch(None, 0, B)
                    self._feed_bind(f0)
                if j + 1 < n:
                    main.wait_event(ev_copy[(j + 1) % NS])      # labels of feed j+1 (copy issued a whole step ago)
            if j + NS - 1 < n:
                issue_copy(j + NS - 1)           # into the buffer of feed j-1: runs while step j computes
            self._replay(*graphs[k])
            ev_done[j] = torch.cuda.Event()
            ev_done[j].record(main)
            with torch.cuda.stream(cs):          # D2H of step j's scalars, off the main stream
                cs.wait_event(ev_done[j])
                ring[j].copy_(log[j], non_blocking=True)
        cs.synchronize()
        main.synchronize()
        r = ring.numpy()
        out.extend({k: float(r[i, j]) for k, j in STAT.items()} for i in range(n))
        return out

    # ---- parameter views -----------------------------------------------------------------------------------------
    @property
    def W(self):
        return self.theta[:self.F * self.H].view(self.F, self.H)

    @property
    def bh(self):
        return self.theta[self.F * self.H:self.F * self.H + self.H]

    @property
    def bv(self):
        return self.theta[self.F * self.H + self.H:]

    def _gW(self):
        return self.grad[:self.F * self.H]

    def _gbh(self):
        return self.grad[self.F * self.H:self.F * self.H + self.H]

    def _gbv(self):
        return self.grad[self.F * self.H + self.H:]

    def set_parameters(self, W, bh=None, bv=None):
        self._w_split_valid = False
        self.W.copy_(torch.as_tensor(np.asarray(W, dtype=np.float32)))
        if bh is not None:
            self.bh.copy_(torch.as_tensor(np.asarray(bh, dtype=np.float32)))
        if bv is not None:
            self.bv.copy_(torch.as_tensor(np.asarray(bv, dtype=np.float32)))

    def get_parameters(self):
        return {'enc_w': self.W.cpu().numpy().copy(), 'enc_b': self.bh.cpu().numpy().copy(),
                'dec_b': self.bv.cpu().numpy().copy()}

    # ---- workspaces ----------------------------------------------------------------------------------------------
    def _drop_graphs(self):
        """Buffers move: the captured step graphs (if any) are stale and must be re-captured."""
        self._graph = self._graph2 = None
        self._feed_graph = None

    def _ensure_ws(self, B):
        if B <= self._ws_B:
            return
        self._drop_graphs()
        f32 = dict(dtype=torch.float32, device=self.device)
        i32 = dict(dtype=torch.int32, device=self.device)
        self.E = torch.empty(B, self.H, **f32)
        self.dE = torch.empty(B, self.H, **f32)
        self.dE2 = torch.empty(B, self.H, **f32)   # triplet part of dL/dE, alpha (G + G^T) E (written on the mining branch)
        if self.loss == _COSINE or self.gemm_mode != 'tc':   # Z = E.W^T is only materialised by the cosine loss and the CUDA-core path
            self.Z = torch.empty(B, self.F, **f32)
        self.row_loss = torch.empty(B, **f32)
        self.weight = torch.empty(B, **f32)
        self.rows = torch.empty(B, **i32)
        self.labels_b = torch.empty(B, **f32)
        self.seg_lo = torch.empty(B, **i32)
        self.seg_hi = torch.empty(B, **i32)
        # staged copy of the per-batch buffers (rows, labels, seg_lo, seg_hi, weight, stats): the NEXT batch of a replayed step
        self._stage = (torch.zeros(B, **i32), torch.zeros(B, **f32), torch.zeros(B, **i32), torch.zeros(B, **i32), torch.zeros(B, **f32),
                       torch.zeros(STAT_SLOTS, dtype=torch.float64, device=self.device))
        # the mining's S / G (and their bf16 hi / lo pair below): B x B, or R anchor rows x B when mined in blocks
        mine_rows = B if self.block_rows is None else min(self.block_rows, B)
        if self._mines:
            self.S = torch.empty(mine_rows, B, **f32)
            self.G = torch.empty(mine_rows, B, **f32)
        if self.gemm_mode == 'tc':
            bf = dict(dtype=torch.bfloat16, device=self.device)
            self.Bp = (B + 7) // 8 * 8
            self.E_hi = torch.zeros(B, self.Hp, **bf)   # columns [H+1, Hp) stay zero, column H is the all-ones column
            self.E_lo = torch.zeros(B, self.Hp, **bf)
            self.E_hi[:, self.H] = 1.0
            self.dZ_hi = torch.empty(B, self.Fp, **bf)
            self.dZ_lo = torch.empty(B, self.Fp, **bf)
            self.tile_ptr = torch.empty(B, 4 * ((self.F + 255) // 256) + 1, **i32)
            if self.W_hi is None:
                self.W_hi = torch.empty(self.F, self.Hp, **bf)
                self.W_lo = torch.empty(self.F, self.Hp, **bf)
            if self._mines:
                self.GG_hi = torch.empty(mine_rows, self.Bp, **bf)
                self.GG_lo = torch.empty(mine_rows, self.Bp, **bf)
        if self.deterministic:
            # stream-K slots of the three GEMMs that can run at once (dE on the main branch, dW on branch B, batch_all's dE2 on branch
            # A), the fused decode's per-(half tile, row) loss partials and one fp64 triplet-loss slot per anchor
            nb = _cabi.query('dae_gemm_det_workspace')
            self.gemm_ws = [torch.empty(nb, dtype=torch.uint8, device=self.device) for _ in range(3)]
            self.n_loss_parts = _cabi.query('dae_decode_loss_parts', self.F, ctype=ctypes.c_int32)
            self.loss_parts = torch.empty(self.n_loss_parts, B, **f32)
            self.loss_slots = torch.empty(B, dtype=torch.float64, device=self.device)
        self._ws_B = B

    def _ensure_bucket_scratch(self, B):
        """Scratch of dae_encode_csr_bwd_gather: per-column counts / offsets and the bucketed (row, value) entries."""
        c = self.csr_c
        cap = int(c.nnz) if c.max_row_nnz is None else int(min(c.nnz, B * max(c.max_row_nnz, 1)))
        if self.col_count is None:
            i32 = dict(dtype=torch.int32, device=self.device)
            self.col_count = torch.zeros(self.F, **i32)
            self.col_start = torch.zeros(self.F + 1, **i32)
            self.col_cursor = torch.zeros(self.F, **i32)
        if cap > self._ent_cap:
            cap = int(cap * 1.5) if c.max_row_nnz is None else cap   # per-step host feeds vary in size: grow geometrically
            self._drop_graphs()
            self.ent_col = torch.empty(cap, dtype=torch.int32, device=self.device)
            self.ent_row = torch.empty(cap, dtype=torch.int32, device=self.device)
            self.ent_val = torch.empty(cap, dtype=torch.float32, device=self.device)
            self._ent_cap = cap
        if self.enc_bwd_mode == 'det':
            need = _cabi.query('dae_encode_csr_bwd_det_workspace', B, self.F, self.H, self._ent_cap)
            if self.enc_det_ws is None or self.enc_det_ws.numel() < need:   # (laid out per call from B and the cap)
                self._drop_graphs()
                self.enc_det_ws = torch.empty(need, dtype=torch.uint8, device=self.device)

    # ---- data ----------------------------------------------------------------------------------------------------
    def set_data(self, csr, values_corrupt=None, labels=None, csr_corrupt=None):
        """csr: DeviceCSR of the CLEAN training rows (loss target); values_corrupt: fp32[nnz] values of the corrupted
        copy sharing the same structure (None = uncorrupted); csr_corrupt: a corrupted copy with its OWN structure
        (salt-and-pepper adds entries); labels: fp32[N] or None."""
        self.csr = csr
        self.csr_c = csr if csr_corrupt is None else csr_corrupt
        self.values_c = self.csr_c.values if values_corrupt is None else values_corrupt
        self.labels = labels

    def corrupt_masking(self, corr_frac, keep_host=None, seed=0, epoch=0):
        """Masking noise on the device copy of the values (utils.masking_noise, autoencoder/utils.py:94-115).
        keep_host: uint8[nnz] host mask (np.random.rand(nnz) >= v) for RNG-stream parity; else Philox on device."""
        self.csr_c = self.csr
        if self.values_c is self.csr.values or self.values_c.numel() != self.csr.nnz:
            self.values_c = torch.empty_like(self.csr.values)
        keep = None
        if keep_host is not None:
            keep = torch.from_numpy(np.ascontiguousarray(keep_host, dtype=np.uint8)).to(self.device, non_blocking=True)
        self._k('dae_mask_values', ptr(self.csr.values), ptr(keep), self.csr.nnz, float(corr_frac), int(seed), int(epoch),
                ptr(self.values_c), _stream())

    def salt_pepper_buffers(self, v):
        """The corrupted-CSR buffers of salt-and-pepper noise with v draws per row over the current clean set, allocated once per data set
        (and v): a captured step graph reads every epoch's corruption at the same addresses.  Capacity sum_r min(F, nnz_r + v) entries
        (8 B each); max_row_nnz is the bound min(F, max_r nnz_r + v), so the step's scratch sized from it never grows between epochs."""
        c, F, v = self.csr, self.F, int(v)
        if self._sp is not None and self._sp['csr'] is c and self._sp['v'] == v:
            return self._sp
        self._sp = None
        N = c.shape[0]
        cap = int(torch.clamp(c.indptr[1:] - c.indptr[:-1] + v, max=F).sum().item()) if N else 0
        ws_bytes = _cabi.query('dae_salt_pepper_workspace', N, ctype=ctypes.c_size_t)
        dev = self.device
        out = _CSRView(torch.zeros(N + 1, dtype=torch.int64, device=dev), torch.empty(max(cap, 1), dtype=torch.int32, device=dev),
                       torch.empty(max(cap, 1), dtype=torch.float32, device=dev), c.shape)
        out.max_row_nnz = min(F, int(c.max_row_nnz or 0) + v)
        self._sp = {'csr': c, 'v': v, 'cap': cap, 'out': out, 'ws': torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev),
                    'overflow': torch.zeros(1, dtype=torch.int32, device=dev), 'draws': None}
        return self._sp

    def corrupt_salt_pepper(self, v, lo, hi, seed=0, epoch=0, draws_host=None, segments=None):
        """Salt-and-pepper noise of the WHOLE clean set on the device (utils.salt_and_pepper_noise, autoencoder/utils.py:118-144): the
        corrupted copy, with its own structure, lands in the buffers of `salt_pepper_buffers(v)` and becomes the encode input csr_c.
        segments: [(row0, n, lo, hi), ...] consecutive row ranges with their own lo / hi, appended into one CSR (the stacked [org; pos;
        neg] set); None = one range over all rows with (lo, hi).  draws_host: uint32[rows * v] host draws in segment order
        (utils.salt_and_pepper_draws: the reference's NumPy stream), else Philox keyed by (seed, epoch, global row)."""
        b = self.salt_pepper_buffers(v)
        v = b['v']
        N = self.csr.shape[0]
        segs = [(0, N, lo, hi)] if segments is None else [(int(r0), int(n), l, h) for r0, n, l, h in segments]
        assert segs[0][0] == 0 and all(s[0] + s[1] == t[0] for s, t in zip(segs, segs[1:])) and segs[-1][0] + segs[-1][1] == N, \
            'segments must tile the rows in order'
        draws = None
        if draws_host is not None:
            dh = np.ascontiguousarray(draws_host, dtype=np.uint32).reshape(-1)
            assert dh.size == N * v, 'draws_host: %d draws for %d rows x v = %d' % (dh.size, N, v)
            if b['draws'] is None:   # one device buffer for the data set (N * v * 4 B)
                b['draws'] = torch.empty(max(dh.size, 1), dtype=torch.int32, device=self.device)
            b['draws'][:dh.size].copy_(torch.from_numpy(dh.view(np.int32)))
            draws = b['draws']
        out, ws = b['out'], b['ws']
        for r0, n, l, h in segs:
            self._k('dae_salt_pepper_csr', ptr(self.csr.indptr), ptr(self.csr.indices), ptr(self.csr.values), r0, n, self.F, v, float(l),
                    float(h), None if draws is None else ptr(draws) + 4 * r0 * v, int(seed), int(epoch), ptr(out.indptr), ptr(out.indices),
                    ptr(out.values), b['cap'], ptr(b['overflow']), ptr(ws), ws.numel(), _stream(), n_launch=3)
        self.csr_c = out
        self.values_c = out.values

    def check_corruption(self):
        """Raise if a salt-and-pepper call found its output beyond the buffers' capacity (it then leaves its rows empty; with the
        capacity of salt_pepper_buffers this cannot happen).  One 4-byte read: call it once per epoch."""
        b = self._sp
        if b is not None and int(b['overflow'].item()) != 0:
            raise _cabi.DaeError('dae_salt_pepper_csr: corrupted CSR beyond its capacity of %d entries' % b['cap'])

    # ---- the GEMM used for the dense contractions (v1: fp32 CUDA-core kernel) ---------------------------------------
    def _gemm(self, M, N, K, alpha, A, sam, sak, Bm, sbn, sbk, beta, Cm, ldc, tag='gemm'):
        self._k('dae_sgemm', M, N, K, float(alpha), ptr(A), sam, sak, ptr(Bm), sbn, sbk, float(beta), ptr(Cm), ldc, _stream(),
                tag=tag)

    # ---- tensor-core path helpers -------------------------------------------------------------------------------------------
    def _tc_gemm(self, M, N, K, alpha, A, a_mn, Bm, b_mn, C, ldc, n_store=0, special_col=-1, special_out=None, k_splits=1,
                 accumulate=0, tag='gemm', ws=None):
        """ws: a deterministic-mode GEMM workspace (stream-K partial tiles are summed in k order by a fixup kernel), or None."""
        (a_hi, a_lo), (b_hi, b_lo) = A, Bm
        if ws is not None:
            # kernels launched (the engine's launch count): the GEMM, plus the fixup where the export runs stream-K -- k_splits = -1 and
            # 128 x 128 tiles that do not fill the SMs in whole waves (its test, reproduced here)
            tiles = ((M + 127) // 128) * ((N + 127) // 128)
            n_launch = 2 if (k_splits < 0 and tiles % self._sm_count() != 0) else 1
            self._k('dae_gemm_bf16x3_det', M, N, K, float(alpha), ptr(a_hi), ptr(a_lo), a_hi.stride(0), a_mn, ptr(b_hi), ptr(b_lo),
                    b_hi.stride(0), b_mn, ptr(C), ldc, n_store, special_col, ptr(special_out), k_splits, accumulate, ptr(ws), ws.numel(),
                    _stream(), n_launch=n_launch, tag=tag)
            return
        self._k('dae_gemm_bf16x3', M, N, K, float(alpha), ptr(a_hi), ptr(a_lo), a_hi.stride(0), a_mn, ptr(b_hi), ptr(b_lo),
                b_hi.stride(0), b_mn, ptr(C), ldc, n_store, special_col, ptr(special_out), k_splits, accumulate, _stream(),
                tag=tag)

    def _sm_count(self):
        if self._sms is None:
            self._sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        return self._sms

    def _ensure_w_split(self):
        """W as a bf16 hi/lo pair; refreshed by the optimizer kernel after every update, so only (re)built here after
        parameters were set from outside."""
        if not self._w_split_valid:
            self._tc_split(self.W, self.F, self.H, self.H, self.W_hi, self.W_lo)
            self._w_split_valid = True

    def _tc_split(self, src, rows, cols, ld_src, hi, lo, ones_col=-1, scale=1.0):
        self._k('dae_split_bf16', ptr(src), rows, cols, ld_src, ptr(hi), ptr(lo), hi.stride(0), ones_col, float(scale), _stream())

    # ---- one training step -----------------------------------------------------------------------------------------
    def _side_stream(self, i):
        if self._sides[i] is None:
            self._sides[i] = torch.cuda.Stream(device=self.device)
        return self._sides[i]

    @staticmethod
    def _record(stream):
        ev = torch.cuda.Event()
        ev.record(stream)
        return ev

    @staticmethod
    def _fork(src, dst):
        """dst waits for everything issued on src so far (an edge of the step's graph once captured)."""
        dst.wait_event(TrainEngine._record(src))

    def step(self, perm, offset, B, stats_log_row=None, train=True, ctl=None, staged=None):
        """perm: int32 device tensor (epoch permutation) or None (identity); rows perm[offset:offset+B] form the batch.
        stats_log_row: optional float64[STAT_SLOTS] device view receiving this step's scalars.
        staged = (n_perm, stride): graph-replayed steps of the triplet strategies take their batch from the staging buffers
        (dae_batch_commit) and stage the batch at cursor + stride for the next replay on a side branch."""
        self._step(perm, offset, B, stats_log_row, train, ctl, staged)

    def step_explicit(self, perm, offset, B, n_rows_each, stats_log_row=None, ctl=None):
        """self.csr holds [org; pos; neg] stacked (3*n_rows_each rows). autoencoder_triplet.py:256-258,286-288,303-314."""
        self._step(perm, offset, B, stats_log_row, ctl=ctl, explicit_n=n_rows_each)

    def _step(self, perm, offset, B, stats_log_row, train=True, ctl=None, staged=None, explicit_n=None, defer_update=False):
        """One step (train=False: its forward and scalars only) on the batch at `offset`.  explicit_n: the rows per block of the
        stacked [org; pos; neg] set -- the step then runs on 3 B rows, B of each block.  defer_update: stop before the optimizer
        (the 'nccl' exchange captures it into a graph of its own)."""
        rows = B if explicit_n is None else 3 * B
        self._ensure_ws(rows)
        self._ctl = ctl  # device int64[4] cursors (offset, log row, optimizer step) when the step is graph-captured
        st = _stream()
        stage_next = None
        if explicit_n is not None:
            self._k('dae_batch_prepare_explicit', ptr(perm), int(offset), ptr(ctl), B, int(explicit_n), ptr(self.rows), ptr(self.stats), st)
        elif staged is not None and self._mines and train:
            self._k('dae_batch_commit', B, *[ptr(t) for t in self._stage], ptr(self.rows), ptr(self.labels_b), ptr(self.seg_lo),
                    ptr(self.seg_hi), ptr(self.weight), ptr(self.stats), st)
            stage_next = (perm, staged)
        else:
            self._k(self._prepare, ptr(perm), int(offset), ptr(ctl), B, ptr(self.labels), self.strategy, ptr(self.rows),
                    ptr(self.labels_b), ptr(self.seg_lo), ptr(self.seg_hi), ptr(self.weight), ptr(self.stats), st)
        prologue_b = self._branch_b_prologue(rows, train)
        self._encode_forward(rows, train)
        self._train_tail(rows, prologue_b, stats_log_row, train, stage_next, B if explicit_n is not None else 0, defer_update)

    def _stage_next_batch(self, perm, staged, B, stream):
        n_perm, stride = staged
        labels = self.labels if self._labels_next is None else self._labels_next    # (run_feeds: the NEXT feed's labels)
        self._k(self._prepare_next, ptr(perm), int(n_perm), int(stride), ptr(self._ctl), B, ptr(labels), self.strategy,
                *[ptr(t) for t in self._stage], stream.cuda_stream)

    def stage_batch(self, perm, offset, B):
        """Host-side staging of the batch at `offset` (the first replay after a cursor jump, e.g. an epoch start)."""
        self._ensure_ws(B)
        s = self._stage
        self._k(self._prepare, ptr(perm), int(offset), None, B, ptr(self.labels), self.strategy, ptr(s[0]), ptr(s[1]), ptr(s[2]),
                ptr(s[3]), ptr(s[4]), ptr(s[5]), _stream())

    def _branch_b_prologue(self, B, train):
        """Start of branch B, forked BEFORE K1: everything the later kernels need that depends on nothing but the batch's row ids --
        zero the gradient buffer (dense dW, sparse dW and dbh accumulate into it) and dE (its stream-K GEMM accumulates), and the
        row-id part of the fused decode (row-loss zeroing, per-tile CSR offsets).  Returns (decode prepared, the branch's event), or
        None when the step has no branch B (CUDA-core path, forward only, or fork_branches off)."""
        if not (self.gemm_mode == 'tc' and train and self.fork_branches):
            return None
        main, sideB = torch.cuda.current_stream(), self._side_stream(1)
        self._fork(main, sideB)
        prepared = 0
        with torch.cuda.stream(sideB):
            if self.loss != _COSINE:   # first on the branch: it becomes runnable together with K1 (whose 800 CTAs then fill the machine)
                c = self.csr
                self._k('dae_decode_prepare', B, self.F, ptr(c.indptr), ptr(c.indices), ptr(self.rows), ptr(self.row_loss),
                        ptr(self.tile_ptr), sideB.cuda_stream)
                prepared = 1
            self.grad.zero_()
            self.dE.zero_()
            return prepared, self._record(sideB)

    def _encode_forward(self, B, train):
        """K1 on the batch rows; also emits E as the bf16 hi/lo pair (plus the all-ones column kept in E_hi) the tensor-core GEMMs
        consume and, for training, the per-column entry counts of the backward gather."""
        cc = self.csr_c
        gather = train and self.enc_bwd_mode in ('gather', 'det')
        if gather:
            self._ensure_bucket_scratch(B)
        tc = self.gemm_mode == 'tc'
        self._k('dae_encode_csr_fwd', ptr(cc.indptr), ptr(cc.indices), ptr(self.values_c), ptr(self.rows), B, self.F, self.H,
                self.in_scale, ptr(self.W), ptr(self.bh), self.enc_act, ptr(self.E), self.H, ptr(self.col_count) if gather else None,
                ptr(self.E_hi) if tc else None, ptr(self.E_lo) if tc else None, self.Hp, _stream())
        if tc:
            self._ensure_w_split()

    def _train_tail(self, B, prologue_b, stats_log_row, train, stage_next=None, explicit_B=0, defer_update=False):
        """Everything after the encode forward.  Dependencies of the step (tensor-core path):

            batch -+-> K1 -+-> decode(+loss, dZ) -> dE = dZ.W ----------+-> encode backward (dA, dbh, sparse dW) -+-> exchange, optimizer
                   |       |                                            |      dA = f'(A) (dE + dE2)             |
                   |       +-> [A: S = E.E^T, triplets, dE2 = a(G+G^T)E]+                                         |
                   |              ... [finalize, stage next batch] (tail of branch A)                            |
                   +-> [B: zero grad / dE, decode row-id tables] ........ dW = dZ^T.[E|1] (dense dW, dbv) --------+
                                                                          (issued once dE owns the SMs)

        batch_all's mining needs only E (its data weights are closed-form) and runs as branch A next to the decode chain; the
        dense dW GEMM only meets the sparse dW of the encode backward in the (zeroed) gradient buffer, where both accumulate, so it
        runs as branch B next to the latency-bound encode-backward kernels.  batch_hard's weights come out of the mining kernel,
        so there the mining stays in line.  Eagerly these are streams + events; captured, parallel branches of ONE graph.
        prologue_b: what _branch_b_prologue returned.  stage_next: (perm, staged) of the batch the step stages for the next replay."""
        F, H = self.F, self.H
        main = torch.cuda.current_stream()
        tc = self.gemm_mode == 'tc'
        mines = self._mines
        weight = self.weight if mines else None
        gather = train and self.enc_bwd_mode == 'gather'
        branch_b = prologue_b is not None                  # branch B exists (tensor-core training with fork_branches)
        branch_a = branch_b and self.strategy == _BATCH_ALL  # branch A exists: the mining runs on it
        # dE2 = alpha (G + G^T) E has a GEMM of its own unless the block loop of _mining_blocked accumulated it; without branch A it
        # goes on the side stream when branch B exists (batch_hard), in line otherwise
        dE2_gemm = mines and tc and train and self.block_rows is None
        dE2_side = dE2_gemm and branch_b and not branch_a
        # the next batch is staged at the tail of branch A, else on a side branch of its own, forked before the decode
        stage_fork = stage_next is not None and not branch_a
        used_a = branch_a or dE2_side or stage_fork
        # side stream A is created by the first step that forks, used or not: torch hands out its pooled CUDA streams in creation order
        sideA = self._side_stream(0) if (branch_b or stage_next is not None) else None
        sideB = self._side_stream(1) if branch_b else None
        ev_mined = None
        if branch_a:
            self._fork(main, sideA)
            with torch.cuda.stream(sideA):
                self._mining(B, train)
                if dE2_gemm:
                    self._dE_triplet(B, sideA)
                ev_mined = self._record(sideA)
        elif mines:
            self._mining(B, train)                # in line: batch_hard's data weights come out of the mining kernel
            if dE2_side:                          # ... but its dE contribution can still run next to the decode chain
                self._fork(main, sideA)
                self._dE_triplet(B, sideA)
                ev_mined = self._record(sideA)
            elif dE2_gemm:
                self._dE_triplet(B, main)
        dec_prepared = 0
        if branch_b:
            dec_prepared, ev_zero = prologue_b
            main.wait_event(ev_zero)              # zeroed gradient / dE buffers (issued before K1)
            if gather:   # the column-bucket offsets of the backward gather only need K1's counts: branch B, far from any critical path
                self._fork(main, sideB)
                with torch.cuda.stream(sideB):
                    self._k('dae_col_scan', ptr(self.col_count), F, ptr(self.col_start), ptr(self.col_cursor), sideB.cuda_stream)
                    ev_scan = self._record(sideB)
        if stage_fork:                            # the staging buffers were consumed by dae_batch_commit: refill them now
            self._fork(main, sideA)
            with torch.cuda.stream(sideA):
                self._stage_next_batch(*stage_next, B, sideA)
        if tc:
            self._decode_tc(B, weight, train, prepared=dec_prepared)
        else:
            self._decode_and_backward(B, weight, train)
        if not train:
            if explicit_B:   # forward only: the kernel's loss statistics are what is wanted, its dE contribution lands in scratch
                self._triplet_explicit(explicit_B, main)
            self._finalize(B, weight, stats_log_row, main)
            return
        if branch_a:
            # the step's scalars only need the decode row losses (main branch) and the mining statistics (branch A): reduce them on
            # branch A while the main one continues with the backward GEMMs / encode backward / optimizer
            self._fork(main, sideA)
            with torch.cuda.stream(sideA):
                self._finalize(B, weight, stats_log_row, sideA)
        if tc:
            Whl, dZhl = (self.W_hi, self.W_lo), (self.dZ_hi, self.dZ_lo)
            if not branch_b:   # in line: the dense dW is stored first, the encode backward then adds its sparse part
                self._dW_gemm(B, accumulate=0)
            # k_splits = -1: stream-K (the 28 tiles of dE / 316 tiles of dW do not fill the 132 SMs in whole waves); with branch B
            # the output was zeroed there, so the GEMM accumulates and needs no memset node of its own
            det = self.deterministic   # (deterministic: stored, the zeroing on branch B notwithstanding)
            self._tc_gemm(B, H, F, 1.0, dZhl, 0, Whl, 1, self.dE, H, k_splits=-1, accumulate=1 if (branch_b and not det) else 0,
                          tag='gemm_decode_dE', ws=self.gemm_ws[0] if det else None)
        if explicit_B:   # explicit (org, pos, neg) triplets: row-wise softplus(e.e- - e.e+), adds its dE (autoencoder_triplet.py:303-314)
            self._triplet_explicit(explicit_B, main)
        if branch_b:
            self._fork(main, sideB)           # branch B: after the zeroing (already on sideB) and once dE owns the SMs; it needs
            with torch.cuda.stream(sideB):    # nothing from the mining branch, so it does not wait for it
                self._dW_gemm(B, accumulate=1)
        if ev_mined is not None:              # dE += alpha (G + G^T) E: on the tensor-core path the product already sits in dE2
            main.wait_event(ev_mined)
        if mines and not tc:
            self._gemm(B, H, B, self.alpha, self.G, B, 1, self.E, 1, H, 1.0, self.dE, H, tag='gemm_dE_tri')
            self._gemm(B, H, B, self.alpha, self.G, 1, B, self.E, 1, H, 1.0, self.dE, H, tag='gemm_dE_tri')
        if branch_b and gather:
            main.wait_event(ev_scan)
        self._encode_backward(B, dE_add=self.dE2 if (tc and mines) else None, dbh_zeroed=1 if branch_b else 0,
                              scan_done=branch_b and gather)
        if not branch_a:
            self._finalize(B, weight, stats_log_row, main)
        elif stage_next is not None:          # tail of branch A, after the step's scalars
            with torch.cuda.stream(sideA):
                self._stage_next_batch(*stage_next, B, sideA)
        if branch_b:
            self._fork(sideB, main)           # the dense dW / dbv are in the gradient buffer
        if self.enc_bwd_mode == 'det':        # deterministic: the sparse dW joins the stored dense dW in one fixed-order add
            self._k('dae_encode_sparse_dw_add', B, F, H, self._ent_cap, ptr(self.enc_det_ws), self.enc_det_ws.numel(), ptr(self._gW()),
                    main.cuda_stream)
        # branch A's tail (the step's scalars, the NEXT batch's staging: a 1-CTA sort that only gets an SM once a GEMM CTA retires)
        # does not feed the update: it joins after the optimizer, before the cursors advance / the next step reuses `stats`
        if not defer_update:
            self._apply_update()
        if used_a:
            self._fork(sideA, main)

    def _triplet(self, name, *args, stream, anchors=0, n_launch=1):
        """The triplet-loss export `name`.  Deterministic: its `_det` twin, which leaves one fp64 loss per anchor in loss_slots, then
        (anchors > 0) dae_triplet_loss_sum adds the first `anchors` slots to the statistics in anchor order."""
        if not self.deterministic:
            self._k(name, *args, stream, n_launch=n_launch)
            return
        self._k(name + '_det', *args, ptr(self.loss_slots), stream, n_launch=n_launch)
        self._sum_loss_slots(anchors, stream)

    def _sum_loss_slots(self, anchors, stream):
        if self.deterministic and anchors:
            self._k('dae_triplet_loss_sum', ptr(self.loss_slots), anchors, ptr(self.stats), stream)

    def _triplet_explicit(self, Bx, stream):
        E, d, H = self.E, self.dE, self.H
        self._triplet('dae_triplet_explicit', ptr(E[0:Bx]), ptr(E[Bx:2 * Bx]), ptr(E[2 * Bx:3 * Bx]), Bx, H, H, self.alpha, ptr(d[0:Bx]),
                      ptr(d[Bx:2 * Bx]), ptr(d[2 * Bx:3 * Bx]), ptr(self.stats), stream=stream.cuda_stream, anchors=Bx)

    def _dE_triplet(self, B, stream):
        """dE2 = alpha (G + G^T) E, the triplet part of dL/dE; the encode backward adds it to the decode part (dE_add)."""
        st = stream.cuda_stream
        with torch.cuda.stream(stream):
            if self.strategy == _BATCH_ALL:
                # batch_all: the sweep wrote G as bf16 hi / lo; ONE GEMM walks G's columns and then its rows: alpha (G + G^T) E
                args = (B, self.H, float(self.alpha), ptr(self.GG_hi), ptr(self.GG_lo), self.GG_hi.stride(0), ptr(self.E_hi),
                        ptr(self.E_lo), self.E_hi.stride(0), ptr(self.dE2), self.H, 0)
                if self.deterministic:
                    ws = self.gemm_ws[2]
                    self._k('dae_gemm_sym_bf16x3_det', *args, ptr(ws), ws.numel(), st, n_launch=2, tag='gemm_dE_tri')
                else:
                    self._k('dae_gemm_sym_bf16x3', *args, st, tag='gemm_dE_tri')
            else:
                self._k('dae_sym_split_bf16', ptr(self.G), B, B, self.alpha, ptr(self.GG_hi), ptr(self.GG_lo), self.GG_hi.stride(0), st)
                self._tc_gemm(B, self.H, B, 1.0, (self.GG_hi, self.GG_lo), 0, (self.E_hi, self.E_lo), 1, self.dE2, self.H, tag='gemm_dE_tri')

    def _finalize(self, B, weight, stats_log_row, stream):
        if self.deterministic and self.loss != _COSINE:
            # the fused decode's per-(half tile, row) partials, summed in part order by one thread per row (the finalize's parts path does
            # the same sums on ONE CTA: 4-5x slower at B = 800)
            self._k('dae_reduce_parts', ptr(self.loss_parts), self.n_loss_parts, B, ptr(self.row_loss), stream.cuda_stream)
        self._k('dae_step_finalize', ptr(self.row_loss), None, 0, ptr(weight), B, self.strategy, self.alpha, ptr(self.stats),
                ptr(stats_log_row), ptr(self._ctl), stream.cuda_stream)

    def _dW_gemm(self, B, accumulate):
        """[dW_dec | dbv] = dZ^T . [E | 1]  (F x (H+1): the all-ones column of E_hl delivers dbv)."""
        det = self.deterministic   # (deterministic: the dense part is stored; the sparse part is added after the join)
        self._tc_gemm(self.F, self.H + 1, B, 1.0, (self.dZ_hi, self.dZ_lo), 1, (self.E_hi, self.E_lo), 1, self._gW(), self.H,
                      n_store=self.H, special_col=self.H, special_out=self._gbv(), k_splits=-1, accumulate=0 if det else accumulate,
                      tag='gemm_decode_dW', ws=self.gemm_ws[1] if det else None)

    def _mining(self, B, train=True):
        """S = E.E^T and the triplet kernel (loss, statistics, G = dL/dS; batch_hard: also the data weights)."""
        if self.block_rows is not None:
            self._mining_blocked(B, train)
            return
        H, st = self.H, _stream()
        tc = self.gemm_mode == 'tc'
        if tc:
            Ehl = (self.E_hi, self.E_lo)
            self._tc_gemm(B, B, H, 1.0, Ehl, 0, Ehl, 0, self.S, B, tag='gemm_gram')
        else:
            self._gemm(B, B, H, 1.0, self.E, H, 1, self.E, H, 1, 0.0, self.S, B, tag='gemm_gram')  # S = E.E^T
        if self.strategy == _BATCH_ALL:
            # G also leaves as the bf16 hi / lo pair the (G + G^T).E GEMM reads
            self._triplet('dae_triplet_batch_all', ptr(self.S), B, B, ptr(self.seg_lo), ptr(self.seg_hi), ptr(self.G), B, ptr(self.stats),
                          0, ptr(self.GG_hi) if tc else None, ptr(self.GG_lo) if tc else None, self.GG_hi.stride(0) if tc else 0,
                          stream=st, anchors=B)
        else:
            self._triplet('dae_triplet_batch_hard', ptr(self.S), B, B, ptr(self.labels_b), ptr(self.G), B, ptr(self.weight),
                          ptr(self.stats), stream=st, anchors=B, n_launch=2)

    def _mining_blocked(self, B, train):
        """The mining one block of R anchor rows at a time, for r0 = 0, R, 2R, ... (the last block is short):
            S_blk = E[r0:r0+n].E^T;  the strategy's rows kernel -> G_blk (batch_all: scaled, with its bf16 hi / lo pair; batch_hard:
            unscaled, split to hi / lo times alpha here);  training: dE2[r0:r0+n] += a G_blk.E  and  dE2 += a G_blk^T.E[r0:r0+n].
        Both strategies are row-local in S, and dE2 = alpha (G + G^T) E splits over row blocks, so this equals _mining + _dE_triplet
        on the whole matrix.  batch_hard's 1/(number of active anchors) is known after the last block: dae_triplet_batch_hard_finish
        applies it to dE2 (and fills SUM_W)."""
        R, H, st = self.block_rows, self.H, _stream()
        Ehl = (self.E_hi, self.E_lo)
        Ghl = (self.GG_hi, self.GG_lo)
        lds, ldg, ldgg = self.S.stride(0), self.G.stride(0), self.GG_hi.stride(0)
        batch_all = self.strategy == _BATCH_ALL
        if not batch_all:
            self.weight.zero_()          # the rows kernels accumulate the data weights
        if train:
            self.dE2.zero_()
        a = self.alpha if batch_all else 1.0   # batch_hard's hi / lo already carry alpha
        for r0 in range(0, B, R):
            n = min(R, B - r0)
            Eblk = (self.E_hi[r0:], self.E_lo[r0:])
            self._tc_gemm(n, B, H, 1.0, Eblk, 0, Ehl, 0, self.S, lds, tag='gemm_gram')
            if batch_all:
                self._triplet('dae_triplet_batch_all_rows', ptr(self.S), lds, r0, n, B, ptr(self.seg_lo), ptr(self.seg_hi), ptr(self.G),
                              ldg, ptr(self.stats), 0, ptr(self.GG_hi) if train else None, ptr(self.GG_lo) if train else None,
                              ldgg if train else 0, stream=st)
            else:
                self._triplet('dae_triplet_batch_hard_rows', ptr(self.S), lds, r0, n, B, ptr(self.labels_b), ptr(self.G), ldg,
                              ptr(self.weight), ptr(self.stats), stream=st)
                if train:
                    self._tc_split(self.G, n, B, ldg, self.GG_hi, self.GG_lo, scale=self.alpha)
            if train:
                self._tc_gemm(n, H, B, a, Ghl, 0, Ehl, 1, self.dE2[r0:], H, accumulate=1, tag='gemm_dE_tri')
                self._tc_gemm(B, H, n, a, Ghl, 1, Eblk, 1, self.dE2, H, accumulate=1, tag='gemm_dE_tri')
        self._sum_loss_slots(B, st)
        if not batch_all:
            self._k('dae_triplet_batch_hard_finish', ptr(self.weight), B, ptr(self.stats), ptr(self.dE2) if train else None, H, H, st)

    def evaluate(self, csr, labels, B=None):
        """Forward-only cost of the whole set fed as ONE batch with x_corr = x, like the reference's validation pass
        (autoencoder/autoencoder.py:300-309).  Returns the stats dict."""
        return self._evaluate(csr, labels, csr.shape[0] if B is None else B)

    def evaluate_explicit(self, csr_stacked, n_each):
        """Forward-only cost of a stacked [org; pos; neg] set fed as ONE batch with x_corr = x: the validation pass of
        DenoisingAutoencoderTriplet (reference autoencoder/autoencoder_triplet.py:166-199).  Returns the stats dict."""
        return self._evaluate(csr_stacked, None, int(n_each), explicit_n=int(n_each))

    def _evaluate(self, csr, labels, B, explicit_n=None):
        saved = (self.csr, self.csr_c, self.values_c, self.labels, self.in_scale)
        try:
            self.set_data(csr, None, labels)
            self.in_scale = 1.0
            self._step(None, 0, B, None, train=False, explicit_n=explicit_n)
            return self.read_stats()
        finally:
            self.csr, self.csr_c, self.values_c, self.labels, self.in_scale = saved

    def _decode_and_backward(self, B, weight, train=True):
        """fp32 CUDA-core validation path of the decode chain (gemm_mode 'ffma')."""
        F, H, st = self.F, self.H, _stream()
        c, rows = self.csr, self.rows
        self._gemm(B, F, H, 1.0, self.E, H, 1, self.W, H, 1, 0.0, self.Z, F, tag='gemm_decode_fwd')  # Z = E.W^T
        self._k('dae_decode_loss_bwd', ptr(c.indptr), ptr(c.indices), ptr(c.values), ptr(rows), B, F, ptr(self.bv),
                self.dec_act, self.loss, ptr(weight), ptr(self.stats), ptr(self.Z), F, ptr(self.row_loss), st)
        if not train:
            return
        self._k('dae_colsum', ptr(self.Z), B, F, F, ptr(self._gbv()), st)  # dbv
        self._gemm(F, H, B, 1.0, self.Z, 1, F, self.E, 1, H, 0.0, self._gW(), H, tag='gemm_decode_dW')  # dW_dec = dZ^T.E
        self._gemm(B, H, F, 1.0, self.Z, F, 1, self.W, 1, H, 0.0, self.dE, H, tag='gemm_decode_dE')    # dE = dZ.W

    def _decode_tc(self, B, weight, train=True, prepared=0):
        """Decode forward + loss on the tensor cores (bf16x3):  Z = E.W^T with the loss epilogue fused (no Z / D / dense X in
        HBM); dZ leaves as the bf16 hi/lo pair the two backward GEMMs consume."""
        F, H, st = self.F, self.H, _stream()
        c, rows = self.csr, self.rows
        Ehl, Whl = (self.E_hi, self.E_lo), (self.W_hi, self.W_lo)
        if self.loss != _COSINE:
            det = self.deterministic   # deterministic: the row-loss partials are stored to [n_parts x B], not added
            self._k('dae_decode_fused_bf16x3_det' if det else 'dae_decode_fused_bf16x3', B, F, H, ptr(self.E_hi), ptr(self.E_lo), self.Hp, ptr(self.W_hi), ptr(self.W_lo),
                    self.Hp, ptr(c.indptr), ptr(c.indices), ptr(c.values), ptr(rows), ptr(self.bv), self.dec_act, self.loss,
                    ptr(weight), ptr(self.stats), ptr(self.dZ_hi), ptr(self.dZ_lo), self.Fp, ptr(self.loss_parts if det else self.row_loss),
                    ptr(self.tile_ptr), int(prepared), st, n_launch=1 if prepared else 2, tag='gemm_decode_fwd')
        else:  # cosine proximity needs whole-row norms before dZ: GEMM -> Z, elementwise loss, split
            self._tc_gemm(B, F, H, 1.0, Ehl, 0, Whl, 0, self.Z, F, tag='gemm_decode_fwd')
            self._k('dae_decode_loss_bwd', ptr(c.indptr), ptr(c.indices), ptr(c.values), ptr(rows), B, F, ptr(self.bv),
                    self.dec_act, self.loss, ptr(weight), ptr(self.stats), ptr(self.Z), F, ptr(self.row_loss), st)
            if train:
                self._tc_split(self.Z, B, F, F, self.dZ_hi, self.dZ_lo)

    def _encode_backward(self, B, dE_add=None, dbh_zeroed=0, scan_done=False):
        """K5: dA = dE * f'(A), dbh, and the sparse part of dW (X_c^T . dA) accumulated into the gradient buffer.  scan_done: the
        gather's column scan already ran (dae_col_scan on branch B)."""
        F, H, st = self.F, self.H, _stream()
        c = self.csr_c
        head = (ptr(c.indptr), ptr(c.indices), ptr(self.values_c), ptr(self.rows), B, F, H, self.in_scale, ptr(self.E), ptr(self.bh),
                self.enc_act, ptr(self.dE), ptr(dE_add), H)
        if self.enc_bwd_mode == 'det':   # dA, dbh stored; the sparse dW waits in the workspace for dae_encode_sparse_dw_add
            self._k('dae_encode_csr_bwd_det', *head, ptr(self._gbh()), ptr(self.col_count), self._ent_cap, ptr(self.enc_det_ws),
                    self.enc_det_ws.numel(), st, tag='dae_encode_csr_bwd',
                    n_launch=8)   # column scan, tile count, tile scan, placement, rows (dA), two dbh levels, gather
        elif self.enc_bwd_mode == 'gather':
            self._k('dae_encode_csr_bwd_gather', *head, ptr(self._gW()), ptr(self._gbh()), int(dbh_zeroed), None if scan_done else ptr(self.col_count),
                    ptr(self.col_start), ptr(self.col_cursor), ptr(self.ent_col), ptr(self.ent_row), ptr(self.ent_val), st, n_launch=3,
                    tag='dae_encode_csr_bwd')
        else:
            self._k('dae_encode_csr_bwd', *head, ptr(self._gW()), ptr(self._gbh()), int(dbh_zeroed), st)

    def _setup_multimem(self, n_blocks=132):
        """Move the gradient buffer into symmetric memory bound to a multicast address and create the peer-mapped flag words
        of dae_allreduce_multimem.  Collective over the process group."""
        import torch.distributed._symmetric_memory as symm
        group = self.pg if self.pg is not None else torch.distributed.group.WORLD
        grad = symm.empty(self.n_params, dtype=torch.float32, device=self.device)
        grad.zero_()
        h_grad = symm.rendezvous(grad, group)
        if not getattr(h_grad, 'has_multicast_support', False) or not h_grad.multicast_ptr:
            raise _cabi.DaeError('DAE_ALLREDUCE=multimem: this process group has no NVSwitch multicast support')
        flags = symm.empty(2 * n_blocks * self.world, dtype=torch.int32, device=self.device)
        flags.zero_()
        h_flags = symm.rendezvous(flags, group)
        self.grad = grad
        self._mm = {'grad': h_grad, 'flags': h_flags, 'flag_buf': flags, 'mc_ptr': int(h_grad.multicast_ptr),
                    'epochs': torch.zeros(n_blocks, dtype=torch.int32, device=self.device),
                    'flag_ptrs': int(h_flags.buffer_ptrs_dev), 'rank': int(h_grad.rank), 'blocks': int(n_blocks)}
        torch.cuda.synchronize(self.device)
        torch.distributed.barrier(group)   # every rank's flag words are zero before the first exchange

    def _allreduce_grad(self):
        if self.allreduce_mode == 'multimem':
            m = self._mm
            self._k('dae_allreduce_multimem', m['mc_ptr'], m['flag_ptrs'], ptr(m['epochs']), m['rank'], self.world, self.n_params, m['blocks'], _stream())
        else:
            torch.distributed.all_reduce(self.grad, group=self.pg)

    def _apply_update(self, reduce=True):
        """Data parallel: ONE all-reduce of the flat [dW | dbh | dbv] buffer, then the fused optimizer (1/P folded in)."""
        F, H, st = self.F, self.H, _stream()
        gscale = 1.0
        if self.world > 1:
            if reduce:
                self._allreduce_grad()
            gscale = 1.0 / self.world
        self.step_count += 1
        if self._ctl is None:       # an eager step: the device step counter ctl[2] stays behind step_count, so the next
            self._ctl_owner = None  # run_feed replay re-synchronises it (Adam's bias correction reads it)
        tc = self.gemm_mode == 'tc'
        self._k('dae_optimizer_step', ptr(self.theta), ptr(self.grad), ptr(self.slot1), ptr(self.slot2), self.n_params,
                self.opt, self.lr, self.momentum, gscale, self.step_count, ptr(self._ctl),
                ptr(self.W_hi) if tc else None, ptr(self.W_lo) if tc else None, F, H, self.Hp, st)

    # ---- transform ------------------------------------------------------------------------------------------------------
    # dae_encode_csr_fwd_hot (hot rows of W staged in shared memory by bulk TMA) is OFF by default: it cuts the L2 -> L1 gather traffic
    # but the staged set costs the occupancy that hides the cold gathers' latency (tools/bench_transform.py compares the two kernels).
    # HOT_MIN_ROWS = N turns it on for launches of at least N rows.
    HOT_MIN_ROWS = 1 << 62
    HOT_BYTES = 200 * 1024  # staged set per CTA (the CTAs per SM follow from it)
    HOT_GROUPS = 8          # row groups of 128 threads per CTA

    def _hot_columns(self, csr):
        """The K most frequent feature columns of `csr` (K rows of W fit 200 KB of shared memory) and the column -> slot table
        of dae_encode_csr_fwd_hot.  One histogram pass over the column ids; cached on the matrix."""
        hot = getattr(csr, '_hot', None)
        K = max(1, min(self.F, self.HOT_BYTES // (self.H * 4)))
        if hot is None or hot[2] != K:
            counts = torch.bincount(csr.indices, minlength=self.F)
            cols = torch.topk(counts, K).indices.to(torch.int32)
            slot = torch.full((self.F,), -1, dtype=torch.int32, device=self.device)
            slot[cols.long()] = torch.arange(K, dtype=torch.int32, device=self.device)
            hot = (cols.contiguous(), slot, K)
            csr._hot = hot
        return hot

    def encode(self, csr, in_scale=1.0, out=None, values=None, rows=None):
        """E = f(in_scale * X.W + bh) - f(bh) for every row of csr (autoencoder.py:479-505).  rows = (lo, hi): only that row range
        (a rank's shard of a data-parallel transform: no collective, each rank writes its slice of E)."""
        lo, hi = (0, csr.shape[0]) if rows is None else (int(rows[0]), int(rows[1]))
        N = hi - lo
        if out is None:
            out = torch.empty(N, self.H, dtype=torch.float32, device=self.device)
        if N == 0:
            return out
        indptr = csr.indptr[lo:hi + 1]      # absolute offsets into indices / values: a row range is just a window of indptr
        vals = csr.values if values is None else values
        if N >= self.HOT_MIN_ROWS and self.H % 4 == 0 and self.H <= 1024:
            cols, slot, K = self._hot_columns(csr)
            self._k('dae_encode_csr_fwd_hot', ptr(indptr), ptr(csr.indices), ptr(vals), N, self.F, self.H, float(in_scale), ptr(self.W),
                    ptr(self.bh), self.enc_act, ptr(out), self.H, ptr(cols), ptr(slot), K, self.HOT_GROUPS, _stream(), tag='encode_transform')
        else:
            self._k('dae_encode_csr_fwd', ptr(indptr), ptr(csr.indices), ptr(vals), None, N, self.F, self.H, float(in_scale),
                    ptr(self.W), ptr(self.bh), self.enc_act, ptr(out), self.H, None, None, None, 0, _stream(), tag='encode_transform')
        return out

    # ---- CUDA-graph replay of the step --------------------------------------------------------------------------------
    def capture_step_graph(self, perm_buf, B, log_buf, row_stride=None, staged=True, explicit_n=None):
        """Capture ONE training step (all kernels, the gradient exchange included) into a CUDA graph.  Everything that
        changes between steps lives in device memory: the batch cursor / log row / optimizer step in `self.ctl`
        (moved by dae_step_advance, the last node of the graph), the permutation in `perm_buf`, the corrupted values in
        `self.values_c`.  staged: the triplet strategies take their (label-sorted) batch from staging buffers filled by the
        previous replay (set_step_cursor stages the first one).  explicit_n: rows per block of the stacked [org; pos; neg] set
        (DenoisingAutoencoderTriplet).  Returns the graph; replay with `replay_step()` after `set_step_cursor()`."""
        stride = int(B if row_stride is None else row_stride)
        use_stage = bool(staged) and explicit_n is None and self._mines and perm_buf is not None
        self._graph, self._graph2 = self._capture(perm_buf, B, log_buf, stride, (int(perm_buf.numel()), stride) if use_stage else None,
                                                  explicit_n)
        self._graph_meta = {'perm': perm_buf, 'B': B, 'staged': use_stage}
        return self._graph

    def _capture(self, perm_buf, B, log_buf, stride, staged, explicit_n):
        """Capture the step of `_step(perm_buf, 0, B, log_buf, ctl=self.ctl, staged=staged, explicit_n=explicit_n)` followed by
        dae_step_advance(stride), after two warm-up steps whose parameter updates are undone.  Returns (g, g2): g2 is the optimizer
        graph of the 'nccl' exchange, else None."""
        if self.ctl is None:
            self.ctl = torch.zeros(4, dtype=torch.int64, device=self.device)
        saved = (self.step_count, self.timed)
        self.timed = None

        def one_step(defer_update=False):
            self._step(perm_buf, 0, B, log_buf, ctl=self.ctl, staged=staged, explicit_n=explicit_n, defer_update=defer_update)
        # warm-up outside capture (workspace allocation, function attributes, NCCL channels)
        snap = (self.theta.clone(), None if self.slot1 is None else self.slot1.clone(), None if self.slot2 is None else self.slot2.clone(),
                self.ctl.clone())
        self.ctl.copy_(torch.tensor([0, 0, 1, 0], dtype=torch.int64))  # warm-up / capture run on the first rows of perm_buf
        if staged is not None:
            self.stage_batch(perm_buf, 0, B)
        for _ in range(2):
            one_step()
            call('dae_step_advance', ptr(self.ctl), stride, _stream())
        torch.cuda.synchronize(self.device)
        self.theta.copy_(snap[0]); self.ctl.copy_(snap[3])
        if snap[1] is not None: self.slot1.copy_(snap[1])
        if snap[2] is not None: self.slot2.copy_(snap[2])
        self._w_split_valid = False
        self._ensure_ws(3 * B if explicit_n is not None else B)
        if self.gemm_mode == 'tc':
            self._ensure_w_split()
        torch.cuda.synchronize(self.device)
        launches0 = self.launches
        # world == 1 or an in-graph exchange ('nccl_graph', 'multimem'): one graph for the whole step.  'nccl': the all-reduce stays
        # OUTSIDE (graph 1 = everything up to the gradients and the step's scalars, eager all-reduce, graph 2 = optimizer + advance).
        g = torch.cuda.CUDAGraph()
        g2 = None
        if self.world == 1 or self.allreduce_mode in ('multimem', 'nccl_graph'):
            # thread_local: NCCL's watchdog thread may query events while this thread captures
            with torch.cuda.graph(g, capture_error_mode='thread_local' if self.world > 1 else 'global'):
                one_step()
                call('dae_step_advance', ptr(self.ctl), stride, _stream())
        else:
            with torch.cuda.graph(g, capture_error_mode='thread_local'):
                one_step(defer_update=True)
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2, capture_error_mode='thread_local'):
                self._apply_update(reduce=False)
                call('dae_step_advance', ptr(self.ctl), stride, _stream())
        self.graph_launches = self.launches - launches0 + 1   # kernels per replay
        self.launches = launches0
        self.step_count = saved[0]
        self.timed = saved[1]
        return g, g2

    def set_step_cursor(self, offset, log_row=0):
        """Host-side (re)positioning of the device cursors, e.g. at an epoch start."""
        self._ctl_owner = 'fit'
        self._set_ctl(offset, log_row)
        m = self._graph_meta
        if m is not None and m['staged']:      # the replayed step takes its batch from the staging buffers
            self.stage_batch(m['perm'], int(offset), m['B'])

    def _set_ctl(self, offset, log_row):
        if self._ctl_host is None:
            self._ctl_host = [torch.zeros(4, dtype=torch.int64).pin_memory() for _ in range(8)]   # ring: the copies are asynchronous
        h = self._ctl_host[self._ctl_host_i % len(self._ctl_host)]
        self._ctl_host_i += 1
        h[0], h[1], h[2], h[3] = int(offset), int(log_row), self.step_count + 1, 0
        self.ctl.copy_(h, non_blocking=True)

    def replay_step(self):
        self._replay(self._graph, self._graph2)

    def _replay(self, g, g2):
        g.replay()
        if g2 is not None:
            torch.distributed.all_reduce(self.grad, group=self.pg)
            g2.replay()
        self.step_count += 1
        self.launches += self.graph_launches

    def read_stats(self):
        s = self.stats.cpu().numpy()
        return {k: float(s[i]) for k, i in STAT.items()}
