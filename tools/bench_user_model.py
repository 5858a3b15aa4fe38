"""Training and inference speed of the GRU, LSTM or attention user encoder (user_model.UserGRU / UserLSTM / UserAttention), with a
torch.nn.GRU / torch.nn.LSTM (cuDNN) or torch.nn.MultiheadAttention arm.  One JSON line.

    python tools/bench_user_model.py [--cell gru|lstm|attention] [--n 100000] [--h 500] [--users 32768] [--batch_users 1024,4096]
                                     [--transform_users 100000,1000000]

Workload: --n clustered articles of width --h (device resident) and synth.make_sequences users (mean length 20, truncated to the
last 50 reads: about 18 reads each).  Reported:
  train[B]: positions/s and users/s over one epoch of --users users at batch_users B (after a warm-up epoch), and the time split
            over the phases of a batch (gather + input GEMM, forward recurrence, loss, backward recurrence, weight GEMMs, optimizer)
            from CUDA events in a separate epoch;
  cudnn[B]: the same batches (the same packed layout as a torch PackedSequence, the same negatives and loss) through
            torch.nn.GRU (--cell gru, the default) or torch.nn.LSTM (--cell lstm) in fp32 (cuDNN, TF32 off) with autograd and
            torch.optim.Adam;
  torch[B] (--cell attention, in place of cudnn): the same batches padded to [B, T, H] through torch.nn.MultiheadAttention with a
            causal mask plus the same pooling, negatives and loss, in fp32 with autograd and torch.optim.Adam;
  transform[U]: the encoder's transform of U users (batch_users 16384) and its peak device memory above the inputs and the output.
Times are CUDA-event or synchronised wall-clock spans around whole epochs / calls.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dae_rnn_news_recommendation_b200.synth import make_sequences  # noqa: E402
from dae_rnn_news_recommendation_b200.user_model import Packed, UserAttention, UserGRU, UserLSTM  # noqa: E402

CELLS = {'gru': (UserGRU, torch.nn.GRU), 'lstm': (UserLSTM, torch.nn.LSTM), 'attention': (UserAttention, None)}


def _gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi failed: %s' % e


def _epoch(m, indptr, items, emb, epoch, packs=None):
    """One training epoch; returns (seconds, positions, users, packs)."""
    if packs is None:
        packs = [Packed(indptr, items, u, m.max_len) for u in m.batches(indptr, epoch)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for bi, pk in enumerate(packs):
        m._forward_backward(pk, emb, epoch, bi)
        m._optimizer_step()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, sum(p.P for p in packs), sum(p.B for p in packs), packs


def train_arm(args, B, indptr, items, emb, deterministic=False):
    m = CELLS[args.cell][0](args.h, max_len=50, batch_users=B, seed=0, deterministic=deterministic)
    _epoch(m, indptr, items, emb, 0)                      # warm-up (buffers, module loads)
    packs = [Packed(indptr, items, u, m.max_len) for u in m.batches(indptr, 1)]   # host packing outside the timed span
    sec, pos, users, _ = _epoch(m, indptr, items, emb, 1, packs)
    m.phase_events = []
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    _epoch(m, indptr, items, emb, 2, packs)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    split = {}
    ev = m.phase_events
    for (_, a), (name, b) in zip(ev[:-1], ev[1:]):
        if name != 'start':
            split[name] = split.get(name, 0.0) + a.elapsed_time(b)
    m.phase_events = None
    res = {'batch_users': B, 'batches': len(packs), 'positions': pos, 'users': users, 'epoch_s': sec, 'positions_per_s': pos / sec,
           'users_per_s': users / sec, 'phase_ms_per_epoch': split, 'loss_last_epochs': m.train_loss, 'peak_bytes_above_inputs': int(peak)}
    return res, packs, m


def cudnn_arm(args, packs, emb, m_ref):
    torch.backends.cudnn.allow_tf32 = False
    H = args.h
    g = CELLS[args.cell][1](H, H).cuda()
    g.load_state_dict({k: v.cuda() for k, v in m_ref.state_dict().items()})
    opt = torch.optim.Adam(g.parameters(), lr=1e-3)
    negs = []
    for bi, pk in enumerate(packs):                       # the encoder's device negatives of the same batches
        m_ref._forward_backward(pk, emb, 1, bi)
        negs.append(m_ref._buf['neg'][:pk.P].clone())
    dev = [(torch.from_numpy(pk.items).cuda().long(), torch.from_numpy(pk.nxt).cuda().long(), torch.from_numpy(pk.n.copy()), pk.terms)
           for pk in packs]

    def epoch():
        for (it, nx, bs, terms), ng in zip(dev, negs):
            x = torch.nn.utils.rnn.PackedSequence(emb[it], bs)
            h = g(x)[0].data
            ok = nx >= 0
            hp = h[ok]
            s = (hp * emb[ng[ok].long()]).sum(1) - (hp * emb[nx[ok]]).sum(1)
            loss = torch.nn.functional.softplus(s).sum() / terms
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
    epoch()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    epoch()
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    pos, users = sum(p.P for p in packs), sum(p.B for p in packs)
    return {'epoch_s': sec, 'positions_per_s': pos / sec, 'users_per_s': users / sec}


def attention_torch_arm(args, packs, emb, m_ref):
    """torch.nn.MultiheadAttention (causal mask) plus the pooling over the batches padded to [B, T, H]: the padding lies after each
    user's reads, so the causal mask keeps it out of every real position."""
    torch.backends.cuda.matmul.allow_tf32 = False
    H = args.h
    sd = {k: v.cuda() for k, v in m_ref.state_dict().items()}
    mha = torch.nn.MultiheadAttention(H, m_ref.heads, batch_first=True).cuda()
    mha.load_state_dict({k[len('self_attn.'):]: v for k, v in sd.items() if k.startswith('self_attn.')})
    Wa, ba, q = (torch.nn.Parameter(sd[k].clone()) for k in ('pool.weight', 'pool.bias', 'pool.query'))
    opt = torch.optim.Adam(list(mha.parameters()) + [Wa, ba, q], lr=1e-3)
    negs = []
    for bi, pk in enumerate(packs):
        m_ref._forward_backward(pk, emb, 1, bi)
        negs.append(m_ref._buf['neg'][:pk.P].clone())
    dev = []
    for pk in packs:
        T = len(pk.n)
        i = np.concatenate([np.arange(int(n)) for n in pk.n])
        t = np.repeat(np.arange(T), pk.n)
        dev.append((torch.from_numpy(pk.items).cuda().long(), torch.from_numpy(pk.nxt).cuda().long(), torch.from_numpy(i * T + t).cuda(),
                    pk.B, T, torch.triu(torch.ones(T, T, dtype=torch.bool, device='cuda'), 1), pk.terms))

    def epoch():
        for (it, nx, dst, B, T, mask, terms), ng in zip(dev, negs):
            X = torch.zeros(B * T, H, device='cuda').index_copy_(0, dst, emb[it]).view(B, T, H)
            mm = mha(X, X, X, attn_mask=mask, need_weights=False)[0]
            a = torch.tanh(mm @ Wa.T + ba) @ q
            w = torch.softmax(a[:, None, :].expand(B, T, T).masked_fill(mask, float('-inf')), -1)
            h = (w @ mm).reshape(B * T, H)[dst]
            ok = nx >= 0
            hp = h[ok]
            s = (hp * emb[ng[ok].long()]).sum(1) - (hp * emb[nx[ok]]).sum(1)
            loss = torch.nn.functional.softplus(s).sum() / terms
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
    epoch()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    epoch()
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    pos, users = sum(p.P for p in packs), sum(p.B for p in packs)
    return {'epoch_s': sec, 'positions_per_s': pos / sec, 'users_per_s': users / sec}


def transform_arm(args, m, labels, emb, U):
    indptr, items, _ = make_sequences(U, labels, mean_len=20, seed=7, holdout=False)
    m.batch_users = 16384
    m.transform((indptr[:1001], items[:indptr[1000]]), emb, to_host=False)   # warm-up
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = m.transform((indptr, items), emb, to_host=False)
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - base - out.numel() * 4
    L = np.minimum(np.diff(indptr), 50)
    return {'users': U, 'positions': int(L.sum()), 's': sec, 'users_per_s': U / sec, 'peak_above_inputs_and_output_bytes': int(peak)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cell', default='gru', choices=sorted(CELLS))
    ap.add_argument('--n', type=int, default=100000)
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--users', type=int, default=32768)
    ap.add_argument('--batch_users', default='1024,4096')
    ap.add_argument('--transform_users', default='100000,1000000')
    ap.add_argument('--deterministic', action='store_true',
                    help='time the training arm in the deterministic mode against the default mode (DESIGN 4.21), alternating '
                         'the two; the cuDNN / torch and transform arms are skipped')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_user_model: no CUDA device')
    rng = np.random.RandomState(0)
    labels = rng.randint(0, 16, args.n)
    emb = torch.from_numpy(((rng.randn(16, args.h)[labels] + 0.6 * rng.randn(args.n, args.h)) / np.sqrt(args.h)).astype(np.float32)).cuda()
    indptr, items, _ = make_sequences(args.users, labels, mean_len=20, seed=1, holdout=False)
    res = {'N': args.n, 'H': args.h, 'train_users': args.users, 'mean_len_truncated': float(np.minimum(np.diff(indptr), 50).mean()),
           'gpu': _gpu_info(), 'device_name': torch.cuda.get_device_name(0), 'train': []}
    res['torch' if args.cell == 'attention' else 'cudnn'] = []
    if args.cell != 'gru':   # the default GRU line keeps its keys
        res['cell'] = args.cell
    if args.deterministic:
        res['deterministic'] = []
        for B in (int(b) for b in args.batch_users.split(',')):
            for _ in range(2):   # alternating arms: default, deterministic, default, deterministic
                for det in (False, True):
                    r = train_arm(args, B, indptr, items, emb, deterministic=det)[0]
                    r['deterministic'] = det
                    res['deterministic'].append(r)
        print(json.dumps(res))
        return
    m = None
    for B in (int(b) for b in args.batch_users.split(',')):
        r, packs, m = train_arm(args, B, indptr, items, emb)
        res['train'].append(r)
        c = (attention_torch_arm if args.cell == 'attention' else cudnn_arm)(args, packs, emb, m)
        c['batch_users'] = B
        res['torch' if args.cell == 'attention' else 'cudnn'].append(c)
        del packs
    res['transform'] = [transform_arm(args, m, labels, emb, int(u)) for u in args.transform_users.split(',')]
    print(json.dumps(res))


if __name__ == '__main__':
    main()
