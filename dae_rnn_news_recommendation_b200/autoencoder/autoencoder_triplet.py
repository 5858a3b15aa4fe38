"""DenoisingAutoencoderTriplet: explicit (anchor, positive, negative) triplets (reference
autoencoder/autoencoder_triplet.py).  cost = sum over {org,pos,neg} of the mean reconstruction loss
+ alpha * mean softplus(e.e_neg - e.e_pos)   (autoencoder_triplet.py:303-314), one shared W.

The reference class crashes on its first batch (self.train_summary is never assigned, :146) and forgets the int cast of
a float batch size (utils.py:86-90); this follows the intended maths.  The three matrices are stacked into ONE CSR in
HBM ([org; pos; neg]) so a step is a single 3B-row pass through the same kernels as the base class.
"""
import os
import time

import numpy as np
import scipy.sparse as sp
import torch

from . import utils
from .autoencoder import DenoisingAutoencoder
from ..engine import DeviceCSR, canonical_csr
from .._cabi import STAT, STAT_SLOTS


class DenoisingAutoencoderTriplet(DenoisingAutoencoder):

    def __init__(self, algo_name='dae_triplet', model_name='dae_triplet', compress_factor=10, main_dir='dae_triplet/',
                 enc_act_func='tanh', dec_act_func='none', loss_func='mean_squared', num_epochs=10, batch_size=10,
                 xavier_init=1, opt='gradient_descent', learning_rate=0.01, momentum=0.5, corr_type='none',
                 corr_frac=0., verbose=True, verbose_step=5, seed=-1, alpha=1, **extensions):
        super().__init__(algo_name=algo_name, model_name=model_name, compress_factor=compress_factor, main_dir=main_dir,
                         enc_act_func=enc_act_func, dec_act_func=dec_act_func, loss_func=loss_func, num_epochs=num_epochs,
                         batch_size=batch_size, xavier_init=xavier_init, opt=opt, learning_rate=learning_rate,
                         momentum=momentum, corr_type=corr_type, corr_frac=corr_frac, verbose=verbose,
                         verbose_step=verbose_step, seed=seed, alpha=alpha, triplet_strategy='none', **extensions)

    def _strategy_name(self):
        return 'explicit'

    def fit(self, train_set, validation_set=None, restore_previous_model=False):
        """train_set: {'org','pos','neg'} of same-shaped matrices (reference autoencoder_triplet.py:40-77)."""
        for s in (train_set,) + ((validation_set,) if validation_set is not None else ()):
            assert type(s['org']) == type(s['pos'])
            assert type(s['org']) == type(s['neg'])
            assert s['org'].shape == s['pos'].shape
            assert s['org'].shape == s['neg'].shape
            assert (s['pos'] != s['neg']).sum()
        n_features = train_set['org'].shape[1]
        self.sparse_input = False if isinstance(train_set['org'], np.ndarray) else True
        self.n_components = np.floor(n_features / self.compress_factor).astype(int)
        self.engine = self._make_engine(n_features)
        self._init_parameters(n_features, restore_previous_model)
        self._write_parameter_to_file(restore_previous_model)
        self._train_model_triplet(train_set, validation_set)
        self._save_checkpoint(self.model_path)

    def _train_model_triplet(self, train_set, validation_set):
        eng = self.engine
        keys = ('org', 'pos', 'neg')
        host = [canonical_csr(train_set[k]) for k in keys]
        n = host[0].shape[0]
        stacked = sp.vstack(host).tocsr()
        csr = DeviceCSR(stacked, eng.device)
        eng.set_data(csr, None, None)
        bs = utils._resolve_batch_size(n, self.batch_size)
        world = eng.world
        rank = torch.distributed.get_rank(eng.pg) if world > 1 else 0
        starts = utils.shard_batch_starts(n, bs, world, rank)
        log = torch.zeros(max(len(starts), 1), STAT_SLOTS, dtype=torch.float64, device=eng.device)
        vcsr = None
        if validation_set is not None:
            vhost = [canonical_csr(validation_set[k]) for k in keys]
            vcsr = (DeviceCSR(sp.vstack(vhost).tocsr(), eng.device), vhost[0].shape[0])
            eng._ensure_ws(3 * max(bs, vcsr[1]))   # size the workspaces once: a larger validation batch must not force a re-capture
        # Full-size batches are replayed from ONE captured CUDA graph (device-side row ids and cursors); a short last batch runs eagerly.
        full = [s0 for s0 in starts if s0 + bs <= n]
        tail = [s0 for s0 in starts if s0 + bs > n]
        use_graph = (os.environ.get('DAE_CUDA_GRAPH', '1') == '1' and len(full) >= 2)
        if self.corr_type == 'salt_and_pepper':   # the reference calls salt_and_pepper_noise once per stream: lo / hi per stream
            sp_v = int(np.round(self.corr_frac * n_features_of(host[0])))
            sp_segments = [(k * n, n, float(h.min()), float(h.max())) for k, h in enumerate(host)]
        perm_buf = torch.zeros(n, dtype=torch.int32, device=eng.device)
        # DenoisingAutoencoder's condition (rng_mode 'numpy' draws from np.random, seeded in __init__), here only in the deterministic
        # mode: the default mode's explicit-triplet runs keep the device permutations they always drew
        if self.deterministic and self.rng_mode == 'device' and self.seed >= 0:
            torch.manual_seed(self.seed)
        i = -1
        for i in range(self.num_epochs):
            torch.cuda.synchronize(eng.device)
            t0 = time.time()
            eng.in_scale = 1.0
            if self.corr_type == 'masking':
                # the reference corrupts org, pos, neg in dict order with three rand(nnz) draws (:117-119)
                if self.rng_mode == 'numpy':
                    keep = np.concatenate([utils.masking_keep_mask(h, self.corr_frac) for h in host])
                    eng.corrupt_masking(self.corr_frac, keep_host=keep)
                else:
                    eng.corrupt_masking(self.corr_frac, seed=max(self.seed, 0), epoch=i)
            elif self.corr_type == 'decay':
                eng.in_scale = 1.0 - self.corr_frac
            elif self.corr_type == 'salt_and_pepper':
                # three appended calls over the stacked rows; rng_mode 'numpy' draws org, pos, neg in that order
                if self.rng_mode == 'numpy':
                    draws = np.concatenate([utils.salt_and_pepper_draws(h, sp_v).reshape(-1) for h in host])
                    eng.corrupt_salt_pepper(sp_v, None, None, draws_host=draws, segments=sp_segments)
                else:
                    eng.corrupt_salt_pepper(sp_v, None, None, seed=max(self.seed, 0), epoch=i, segments=sp_segments)
            perm_buf.copy_(self._epoch_permutation(n))
            if world > 1:
                torch.distributed.broadcast(perm_buf, src=0, group=eng.pg)
            if use_graph:
                if eng._graph is None:
                    eng.capture_step_graph(perm_buf, bs, log, row_stride=bs * world, explicit_n=n)
                eng.set_step_cursor(full[0], 0)
                for _ in full:
                    eng.replay_step()
                for k, s0 in enumerate(tail):
                    eng.step_explicit(perm_buf, s0, n - s0, n, log[len(full) + k])
            else:
                for k, s0 in enumerate(starts):
                    eng.step_explicit(perm_buf, s0, min(bs, n - s0), n, log[k])
            torch.cuda.synchronize(eng.device)
            self.train_time = time.time() - t0
            if self.corr_type == 'salt_and_pepper':
                eng.check_corruption()
            vals = log[:len(starts)].cpu().numpy()
            self.train_cost_batch = (list(vals[:, STAT['cost']].astype(np.float32)),
                                     list(vals[:, STAT['ae_loss']].astype(np.float32)),
                                     list(vals[:, STAT['triplet_loss']].astype(np.float32)))
            if (i + 1) % self.verbose_step == 0:
                self._run_validation_error_and_summaries_triplet(i + 1, vcsr)
        else:
            if self.num_epochs != 0 and (i + 1) % self.verbose_step != 0:
                self._run_validation_error_and_summaries_triplet(i + 1, vcsr)

    def _run_validation_error_and_summaries_triplet(self, epoch, vcsr):
        """Console lines of the reference (autoencoder_triplet.py:149-199): epoch means of the training scalars, then -- when a
        validation set was given -- the forward-only cost of the whole (org, pos, neg) validation set, x_corr = x."""
        if self.verbose == 1:
            print('At step %d (%.2f seconds): ' % (epoch, self.train_time), end='')
            print('[Train Stat (average over past steps)] - ', end='')
            print('Cost: ', end='')
            print('Overall=%.4f\t' % np.mean(self.train_cost_batch[0]), end='')
            print('Autoencoder=%.4f\t' % np.mean(self.train_cost_batch[1]), end='')
            print('Triplet=%.4f\t' % np.mean(self.train_cost_batch[2]), end='')
        if vcsr is None:
            if self.verbose == 1:
                print()
            return
        res = self.engine.evaluate_explicit(vcsr[0], vcsr[1])
        self.validation_cost = res
        if self.verbose:
            print('[Validation Stat (at this step)] - Cost: ', end='')
            print('Overall=%.4f\t' % res['cost'], end='')
            print('Autoencoder=%.4f\t' % res['ae_loss'], end='')
            print('Triplet=%.4f\t' % res['triplet_loss'], end='')
            print()


def n_features_of(m):
    return m.shape[1]
