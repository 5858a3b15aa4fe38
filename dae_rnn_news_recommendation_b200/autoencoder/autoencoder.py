"""DenoisingAutoencoder: the reference's sklearn-like estimator (reference autoencoder/autoencoder.py) with the
TensorFlow session replaced by the sm_90a engine (`..engine.TrainEngine` -> libdae_sm100.so).

Same constructor signature, `fit` / `transform` / `load_model` / `get_model_parameters`, same public attributes, same
`results/<algo>/<main_dir>/{models,data,logs,data/tsv,data/plot}` layout and `parameter.txt` dump.  Additive keyword
extensions (never required): `device`, `rng_mode`, `W_init`.

What differs, on purpose:
  * parameters stay resident in HBM between `fit` and `transform` (the reference restores the checkpoint from disk in
    every `transform` call, autoencoder.py:491); the checkpoint is still written at the end of `fit`.
  * the checkpoint is an .npz holding the reference's three variable names ('enc-w','hidden-bias','visible-bias',
    autoencoder.py:365-367) plus optimizer slots -- a TF checkpoint cannot be written without TensorFlow.
  * no TensorBoard summaries (autoencoder.py:391-393,413-415 histogram the B x F decode every step).
  * labels are optional when triplet_strategy == 'none' (the reference hits a NameError, autoencoder.py:224-230).
"""
import os
import time

import numpy as np
import torch

from . import utils
from .. import _cabi
from ..engine import TrainEngine, DeviceCSR, canonical_csr, check_mining_block_rows, resolve_deterministic
from .._cabi import STAT, STAT_SLOTS, MAX_TRIPLET_BATCH, MAX_BLOCKED_BATCH


class DenoisingAutoencoder(object):

    def __init__(self, algo_name='dae', model_name='dae', compress_factor=10, main_dir='dae/', enc_act_func='tanh',
                 dec_act_func='none', loss_func='mean_squared', num_epochs=10, batch_size=10,
                 xavier_init=1, opt='gradient_descent', learning_rate=0.01, momentum=0.5, corr_type='none',
                 corr_frac=0., verbose=True, verbose_step=5, seed=-1, alpha=1, triplet_strategy='batch_all',
                 device=None, rng_mode='device', W_init=None, mining_block_rows=None, deterministic=False):
        """Arguments as in the reference (autoencoder.py:20-45).  Extensions: device ('cuda:N'; default: LOCAL_RANK or 0),
        rng_mode ('device' = Philox mask + device permutation, the default: an epoch of the UCI config is 3 ms of GPU time, the host
        RNG alone would take 6 ms; 'numpy' = the reference's host NumPy RNG stream for corruption and shuffling, drawn one epoch
        ahead on a worker thread -- bit-identical masks and batch order to a seeded reference run), W_init (ndarray F x H
        overriding the Xavier draw), mining_block_rows (None: batch_all / batch_hard hold the B x B similarity matrix, batches up to
        MAX_TRIPLET_BATCH rows; R, a multiple of 128 up to 32768: they mine it R anchor rows at a time in 12 R B bytes, batches up to
        MAX_BLOCKED_BATCH rows), deterministic (True: every sum of the training step runs in a fixed order, so a run with the same seed
        >= 0, rng_mode, data, build and GPU model reproduces its parameters, losses and transform output bit for bit; slower, one
        process, tensor-core path only; None: the environment variable DAE_DETERMINISTIC)."""
        self.algo_name = algo_name
        self.model_name = model_name
        self.compress_factor = compress_factor
        self.main_dir = main_dir
        self.enc_act_func = enc_act_func
        self.dec_act_func = dec_act_func
        self.loss_func = loss_func
        self.num_epochs = num_epochs
        self.batch_size = batch_size
        self.xavier_init = xavier_init
        self.opt = opt
        self.learning_rate = learning_rate
        self.momentum = momentum
        self.corr_type = corr_type
        self.corr_frac = corr_frac
        self.verbose = verbose
        self.verbose_step = verbose_step
        self.seed = seed
        self.alpha = alpha
        self.triplet_strategy = triplet_strategy

        assert type(self.verbose_step) == int
        assert self.verbose >= 0
        assert self.triplet_strategy in ['batch_all', 'batch_hard', 'none']
        assert rng_mode in ('numpy', 'device')

        if self.seed >= 0:
            np.random.seed(self.seed)  # autoencoder.py:72-74 (TF's graph seed has no counterpart here)

        self.models_dir, self.data_dir, self.tf_summary_dir, self.tsv_dir, self.plot_dir = self._create_data_directories()
        self.model_path = self.models_dir + self.model_name
        self.parameter_file = self.tf_summary_dir + 'parameter.txt'

        self.sparse_input = None
        self.n_components = None
        self.train_cost_batch = [], [], []
        self.fraction_triplet_batch = []
        self.num_triplet_batch = []
        self.train_time = None

        if device is None:
            device = 'cuda:%d' % int(os.environ.get('LOCAL_RANK', 0))
        self.device = device
        self.rng_mode = rng_mode
        self.W_init = W_init
        self.mining_block_rows = check_mining_block_rows(mining_block_rows)   # not in parameter.txt: its layout is the reference's
        self.deterministic = resolve_deterministic(deterministic)              # (nor this)
        self.engine = None

    # ------------------------------------------------------------------------------------------------------------------
    def _write_parameter_to_file(self, restore):
        names = ['algo_name', 'model_name', 'compress_factor', 'main_dir', 'enc_act_func', 'dec_act_func', 'loss_func',
                 'num_epochs', 'batch_size', 'xavier_init', 'opt', 'learning_rate', 'momentum', 'corr_type', 'corr_frac',
                 'verbose', 'verbose_step', 'seed', 'alpha', 'triplet_strategy']
        with open(self.parameter_file, 'a+' if restore else 'w') as fh:
            print('---------------------------------------', file=fh)
            for n in names:
                print('{}={}'.format(n, getattr(self, n)), file=fh)

    def _strategy_name(self):
        return self.triplet_strategy

    def _make_engine(self, n_features):
        assert self.opt in _cabi.OPT, 'unknown optimizer %r' % (self.opt,)
        assert self.loss_func in _cabi.LOSS, 'unknown loss %r' % (self.loss_func,)
        eng = TrainEngine(n_features, int(self.n_components), enc_act_func=self.enc_act_func,
                          dec_act_func=self.dec_act_func, loss_func=self.loss_func, opt=self.opt,
                          learning_rate=self.learning_rate, momentum=self.momentum, alpha=self.alpha,
                          triplet_strategy=self._strategy_name(), device=self.device, mining_block_rows=self.mining_block_rows,
                          deterministic=self.deterministic)
        return eng

    def _init_parameters(self, n_features, restore_previous_model):
        eng = self.engine
        if restore_previous_model:
            self._load_checkpoint(self.model_path)
            return
        if self.W_init is not None:
            W0 = np.asarray(self.W_init, dtype=np.float32)
            assert W0.shape == (n_features, int(self.n_components))
        else:
            # own RandomState: the reference draws W0 from TF's graph-level RNG, NOT from the NumPy global stream, so the
            # global stream (masking noise, shuffles) stays aligned with a seeded reference run
            rng = np.random.RandomState(self.seed) if self.seed >= 0 else np.random.RandomState()
            W0 = utils.xavier_init(n_features, int(self.n_components), self.xavier_init, rng=rng)
        eng.set_parameters(W0, np.zeros(int(self.n_components), np.float32), np.zeros(n_features, np.float32))
        if eng.world > 1:
            torch.distributed.broadcast(eng.theta, src=0, group=eng.pg)

    # ------------------------------------------------------------------------------------------------------------------
    def fit(self, train_set, validation_set=None, train_set_label=None, validation_set_label=None,
            restore_previous_model=False):
        """Fit the model (reference autoencoder.py:126-156).  train_set: ndarray or any scipy sparse matrix."""
        if self.triplet_strategy != 'none':
            assert train_set_label is not None
        if train_set_label is not None:
            assert train_set.shape[0] == len(train_set_label)
        if validation_set is not None:
            assert validation_set_label is None or validation_set.shape[0] == len(validation_set_label)

        n_features = train_set.shape[1]
        self.sparse_input = False if isinstance(train_set, np.ndarray) else True
        self.n_components = np.floor(n_features / self.compress_factor).astype(int)

        self.engine = self._make_engine(n_features)
        self._init_parameters(n_features, restore_previous_model)
        self._write_parameter_to_file(restore_previous_model)
        self._train_model(train_set, validation_set, train_set_label, validation_set_label)
        self._save_checkpoint(self.model_path)

    # ------------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _labels_to_device(labels, device):
        if labels is None:
            return None
        arr = np.asarray(labels, dtype=np.float32).reshape(-1)  # fed as 'float' (autoencoder.py:352)
        return torch.from_numpy(arr).to(device)

    def _host_rng_prefetch(self, train_csr_host, n):
        """rng_mode='numpy': the reference's per-epoch draws from the global NumPy stream -- rand(nnz) for the masking noise
        (utils.py:111) or the salt-and-pepper draws (utils.py:137-139), then the shuffle of the row order (utils.py:50-51) -- produced IN
        THAT ORDER by a worker thread that runs one epoch ahead of the GPU.  Returns a function handing out (keep mask / packed draws or
        None, permutation) epoch by epoch.  The salt-and-pepper draws take N * v * 4 bytes per epoch (1.2 GB at 100 000 rows of 10 000
        features, corr_frac 0.3): at most one epoch waits in the queue, so the host holds at most three (queued, being drawn, in use)."""
        import queue
        import threading
        if self.rng_mode != 'numpy' or self.corr_type not in ('masking', 'none', 'decay', 'salt_and_pepper'):
            return None
        sp_v = self._salt_pepper_v(train_csr_host) if self.corr_type == 'salt_and_pepper' else None
        q = queue.Queue(maxsize=1 if sp_v is not None else 2)

        def work():
            try:
                for _ in range(self.num_epochs):
                    keep = None
                    if self.corr_type == 'masking':
                        keep = utils.masking_keep_mask(train_csr_host, self.corr_frac)
                    elif sp_v is not None:
                        keep = utils.salt_and_pepper_draws(train_csr_host, sp_v)
                    order = list(range(n))
                    np.random.shuffle(order)
                    q.put((keep, np.asarray(order, dtype=np.int32)))
            except BaseException as e:   # noqa: BLE001 -- hand the failure to the consumer instead of dying silently
                q.put(e)
        t = threading.Thread(target=work, daemon=True)
        t.start()

        def take():
            item = q.get()
            if isinstance(item, BaseException):
                raise item
            return item
        take.thread = t
        return take

    def _salt_pepper_v(self, train_csr_host):
        return int(np.round(self.corr_frac * train_csr_host.shape[1]))  # autoencoder.py:187

    def _salt_pepper_range(self, train_csr_host):
        """(lo, hi) of salt-and-pepper noise: X.min() / X.max() over the whole matrix, implicit zeros included (utils.py:129), computed
        once per host matrix."""
        c = getattr(self, '_sp_range', None)
        if c is None or c[0] is not train_csr_host:
            c = self._sp_range = (train_csr_host, float(train_csr_host.min()), float(train_csr_host.max()))
        return c[1], c[2]

    def _corrupt_on_device(self, train_csr_host, epoch, keep=None):
        """Per-epoch corruption of the WHOLE training set (autoencoder.py:218,248-270).  keep: rng_mode='numpy' draws of the epoch (the
        masking keep mask, or the packed salt-and-pepper draws), or None to draw them here."""
        eng = self.engine
        eng.in_scale = 1.0
        if self.corr_type == 'masking':
            if self.rng_mode == 'numpy':
                if keep is None:
                    keep = utils.masking_keep_mask(train_csr_host, self.corr_frac)
                eng.corrupt_masking(self.corr_frac, keep_host=keep)
            else:
                eng.corrupt_masking(self.corr_frac, seed=max(self.seed, 0), epoch=epoch)
        elif self.corr_type == 'decay':
            eng.set_data(eng.csr, None, eng.labels)
            eng.in_scale = 1.0 - self.corr_frac
        elif self.corr_type == 'salt_and_pepper':
            v = self._salt_pepper_v(train_csr_host)
            lo, hi = self._salt_pepper_range(train_csr_host)
            if self.rng_mode == 'numpy':
                if keep is None:
                    keep = utils.salt_and_pepper_draws(train_csr_host, v)
                eng.corrupt_salt_pepper(v, lo, hi, draws_host=keep)
            else:
                eng.corrupt_salt_pepper(v, lo, hi, seed=max(self.seed, 0), epoch=epoch)
        elif self.corr_type == 'none':
            eng.set_data(eng.csr, None, eng.labels)
        else:
            raise AssertionError('unknown corr_type %r' % (self.corr_type,))

    def _epoch_permutation(self, n):
        if self.rng_mode == 'numpy':
            order = list(range(n))
            np.random.shuffle(order)  # utils.py:50-51
            return torch.from_numpy(np.asarray(order, dtype=np.int32)).to(self.engine.device, non_blocking=True)
        return torch.randperm(n, device=self.engine.device, dtype=torch.int32)

    def _train_model(self, train_set, validation_set, train_set_label, validation_set_label):
        eng = self.engine
        host_csr = canonical_csr(train_set)
        csr = DeviceCSR(host_csr, eng.device)
        eng.set_data(csr, None, self._labels_to_device(train_set_label, eng.device))
        n = host_csr.shape[0]
        bs = utils._resolve_batch_size(n, self.batch_size)
        world = eng.world
        rank = torch.distributed.get_rank(eng.pg) if world > 1 else 0
        starts = utils.shard_batch_starts(n, bs, world, rank)  # data parallel: rank r takes batches r, r+P, ...
        log = torch.zeros(max(len(starts), 1), STAT_SLOTS, dtype=torch.float64, device=eng.device)
        if self.rng_mode == 'device' and self.seed >= 0:
            torch.manual_seed(self.seed)
        # Full-size batches are replayed from ONE captured CUDA graph (their offsets are start0 + g * stride, advanced on the
        # device); a short last batch runs eagerly.  Every corruption writes into buffers allocated once, so the graph reads each
        # epoch's corrupted copy at the same addresses.
        full = [s0 for s0 in starts if s0 + bs <= n]
        tail = [s0 for s0 in starts if s0 + bs > n]
        use_graph = (os.environ.get('DAE_CUDA_GRAPH', '1') == '1' and len(full) >= 2)
        perm_buf = torch.zeros(n, dtype=torch.int32, device=eng.device)
        R = self.mining_block_rows
        nv = 0 if validation_set is None else validation_set.shape[0]
        if self.triplet_strategy != 'none' and R is None:   # the mining branch keeps S, G and G's bf16 copy: B x B x 12 bytes
            cap = MAX_TRIPLET_BATCH
            hint = ' Set mining_block_rows (e.g. 4096) to mine the similarity matrix in blocks of rows, up to %d rows.' % MAX_BLOCKED_BATCH
            assert bs <= cap, ('triplet strategies need batch_size <= %d rows (got %d: the B x B similarity / gradient buffers would '
                               'take %.1f GB).' % (cap, bs, 12.0 * bs * bs / 1e9) + hint)
            assert nv <= cap, ('the validation set is fed as ONE batch (autoencoder.py:300-309): at most %d rows with a triplet '
                               'strategy (got %d: its B x B buffers would take %.1f GB).' % (cap, nv, 12.0 * nv * nv / 1e9) + hint)
        elif self.triplet_strategy != 'none':   # block mining: R x B rows of S, G and G's bf16 copy, plus dZ's bf16 hi / lo pair
            cap = MAX_BLOCKED_BATCH
            Fp = (host_csr.shape[1] + 31) // 32 * 32

            def gb(b):
                return (12.0 * min(R, b) * b + 4.0 * b * Fp) / 1e9
            assert bs <= cap, ('triplet strategies with mining_block_rows need batch_size <= %d rows (got %d: its mining blocks and '
                               'dZ would take %.1f GB)' % (cap, bs, gb(bs)))
            assert nv <= cap, ('the validation set is fed as ONE batch (autoencoder.py:300-309): at most %d rows with mining_block_rows '
                               '(got %d: its mining blocks and dZ would take %.1f GB)' % (cap, nv, gb(nv)))
        if validation_set is not None:        # size the workspaces once: a larger validation batch must not force a re-capture
            eng._ensure_ws(max(bs, validation_set.shape[0]))
        prefetch = self._host_rng_prefetch(host_csr, n)

        self.history = []  # additive: per-epoch float64 arrays [steps x STAT_SLOTS] of every step's scalars
        i = -1
        for i in range(self.num_epochs):
            self.train_cost_batch = [], [], []
            self.fraction_triplet_batch = []
            self.num_triplet_batch = []
            torch.cuda.synchronize(eng.device)
            t0 = time.time()
            if prefetch is not None:
                keep, order = prefetch()
                self._corrupt_on_device(host_csr, i, keep)
                perm_buf.copy_(torch.from_numpy(order).to(eng.device, non_blocking=True))
            else:
                self._corrupt_on_device(host_csr, i)
                perm_buf.copy_(self._epoch_permutation(n))
            if world > 1:   # every rank must slice the SAME permutation (also when the run is unseeded)
                torch.distributed.broadcast(perm_buf, src=0, group=eng.pg)
            if use_graph:
                if eng._graph is None:  # first epoch, or the workspaces were re-allocated (e.g. by a larger validation batch)
                    eng.capture_step_graph(perm_buf, bs, log, row_stride=bs * world)
                eng.set_step_cursor(full[0], 0)
                for _ in full:
                    eng.replay_step()
                for k, s0 in enumerate(tail):
                    eng.step(perm_buf, s0, n - s0, log[len(full) + k])
            else:
                for k, s0 in enumerate(starts):
                    eng.step(perm_buf, s0, min(bs, n - s0), log[k])
            torch.cuda.synchronize(eng.device)
            self.train_time = time.time() - t0
            if self.corr_type == 'salt_and_pepper':
                eng.check_corruption()
            vals = log[:len(starts)].cpu().numpy()
            self.history.append(vals.copy())
            self.train_cost_batch = (list(vals[:, STAT['cost']].astype(np.float32)),
                                     list(vals[:, STAT['ae_loss']].astype(np.float32)) if self.triplet_strategy != 'none' else [],
                                     list(vals[:, STAT['triplet_loss']].astype(np.float32)) if self.triplet_strategy != 'none' else [])
            if self.triplet_strategy != 'none':
                self.fraction_triplet_batch = list(vals[:, STAT['fraction']].astype(np.float32))
                self.num_triplet_batch = list(vals[:, STAT['num']].astype(np.float32))
            if (i + 1) % self.verbose_step == 0:
                self._run_validation_error_and_summaries(i + 1, validation_set, validation_set_label)
        else:
            if self.num_epochs != 0 and (i + 1) % self.verbose_step != 0:
                self._run_validation_error_and_summaries(i + 1, validation_set, validation_set_label)

    def _run_validation_error_and_summaries(self, epoch, validation_set, validation_set_label):
        """Same console lines as the reference (autoencoder.py:283-320)."""
        if self.verbose == 1:
            print('At step %d (%.2f seconds): ' % (epoch, self.train_time), end='')
            print('[Train Stat (average over past steps)] - ', end='')
            if self.triplet_strategy != 'none':
                print('Triplet: ', end='')
                print('Fraction=%.4f\t' % np.mean(self.fraction_triplet_batch), end='')
                print('Number=%.2f\t' % np.mean(self.num_triplet_batch), end='')
            print('Cost: ', end='')
            print('Overall=%.4f\t' % (np.mean(self.train_cost_batch[0])), end='')
            if self.triplet_strategy != 'none':
                print('Autoencoder=%.4f\t' % np.mean(self.train_cost_batch[1]), end='')
                print('Triplet=%.4f\t' % np.mean(self.train_cost_batch[2]), end='')
        if validation_set is None:
            if self.verbose == 1:
                print()
            return
        eng = self.engine
        vcsr = DeviceCSR(validation_set, eng.device)
        res = eng.evaluate(vcsr, self._labels_to_device(validation_set_label, eng.device))
        self.validation_cost = res
        if self.verbose:
            print("[Validation Stat (at this step)] - Cost: ")
            print('Overall=%.4f' % res['cost'], end='')
            if self.triplet_strategy != 'none':
                print('Autoencoder=%.4f\t' % res['ae_loss'], end='')
                print('Triplet=%.4f\t' % res['triplet_loss'], end='')
            print()

    # ------------------------------------------------------------------------------------------------------------------
    def transform(self, data, name='train', save=False, shard=False):
        """Encode `data` with the trained model (reference autoencoder.py:479-505) -> float32 ndarray [N, n_components].
        shard=True (additive; data-parallel runs): this rank encodes only its contiguous row range `shard_rows(N)` and returns /
        saves (as `<name>.rank<r>`) that slice -- rows are independent, so there is no collective."""
        if self.engine is None:
            raise _cabi.DaeError('transform() before fit()/load_model()')
        eng = self.engine
        rows, suffix = None, ''
        if shard and eng.world > 1:
            rank = torch.distributed.get_rank(eng.pg)
            rows = self.shard_rows(data.shape[0], eng.world, rank)
            suffix = '.rank%d' % rank
            data = data[rows[0]:rows[1]]          # only the shard travels to the device
            rows = None
        csr = DeviceCSR(data, eng.device)
        encoded = eng.encode(csr, rows=rows).cpu().numpy()
        if save:
            np.save(self.data_dir + name + suffix, encoded)
            if not suffix or suffix == '.rank0':
                np.save(self.data_dir + 'weights', eng.W.cpu().numpy())
        return encoded

    @staticmethod
    def shard_rows(n, world, rank):
        """Contiguous row range [lo, hi) of rank `rank` of `world` ranks over n rows (the ranges tile [0, n))."""
        return (n * rank) // world, (n * (rank + 1)) // world

    def load_model(self, shape, model_path):
        """Restore a trained model (reference autoencoder.py:507-527). shape = (n_features, n_components)."""
        self.n_components = shape[1]
        self.engine = self._make_engine(shape[0])
        self._load_checkpoint(model_path)

    def get_model_parameters(self):
        """{'enc_w','enc_b','dec_b'} as numpy arrays (reference autoencoder.py:529-542)."""
        if self.engine is None:
            raise _cabi.DaeError('get_model_parameters() before fit()/load_model()')
        return self.engine.get_parameters()

    # ------------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _ckpt_file(path):
        return path if str(path).endswith('.npz') else str(path) + '.npz'

    def _save_checkpoint(self, path):
        eng = self.engine
        if eng.world > 1 and torch.distributed.get_rank(eng.pg) != 0:
            return
        p = eng.get_parameters()
        blob = {'enc-w': p['enc_w'], 'hidden-bias': p['enc_b'], 'visible-bias': p['dec_b'],
                'step': np.int64(eng.step_count)}
        if eng.slot1 is not None:
            blob['slot1'] = eng.slot1.cpu().numpy()
        if eng.slot2 is not None:
            blob['slot2'] = eng.slot2.cpu().numpy()
        np.savez(self._ckpt_file(path), **blob)

    def _load_checkpoint(self, path):
        eng = self.engine
        with np.load(self._ckpt_file(path)) as z:
            eng.set_parameters(z['enc-w'], z['hidden-bias'], z['visible-bias'])
            if 'slot1' in z and eng.slot1 is not None:
                eng.slot1.copy_(torch.from_numpy(z['slot1']))
            if 'slot2' in z and eng.slot2 is not None:
                eng.slot2.copy_(torch.from_numpy(z['slot2']))
            eng.step_count = int(z['step']) if 'step' in z else 0

    def _create_data_directories(self):
        """results/<algo_name>/<main_dir>/{models,data,logs,data/tsv,data/plot}/ (reference autoencoder.py:544-564)."""
        algo = self.algo_name if self.algo_name.endswith('/') else self.algo_name + '/'
        main = self.main_dir if self.main_dir.endswith('/') else self.main_dir + '/'
        self.main_dir = algo + main
        base = 'results/' + self.main_dir
        models_dir, data_dir, summary_dir = base + 'models/', base + 'data/', base + 'logs/'
        tsv_dir, plot_dir = data_dir + 'tsv/', data_dir + 'plot/'
        for d in (models_dir, data_dir, summary_dir, tsv_dir, plot_dir):
            os.makedirs(d, exist_ok=True)
        return models_dir, data_dir, summary_dir, tsv_dir, plot_dir
