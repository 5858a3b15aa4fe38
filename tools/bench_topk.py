"""k most similar articles for every article: the fused tensor-core top-k (helpers.top_k_similar) against the chunked similarity
matrix paths, on device-resident clustered embeddings (generated like tools/bench_evaluation.py's).  One JSON line.

    python tools/bench_topk.py [--n 100000] [--h 500] [--k 10] [--reps 5] [--warmup 2]
    python tools/bench_topk.py --sparse [--data synth|c1] [--n 100000] [--f 10000] [--kind tfidf|binary] [--queries Q] [--k 10]

Paths, each from fp32 embeddings on the device to (index, score) on the device, self match excluded:
  a  top_k_similar(k)                                  fused GEMM + k-best epilogue, O(N k) extra memory
  b  top_k_similar(k = 1)
  c  nearest_neighbors' path: chunked dae_gemm_bf16x3 into a chunk x N fp32 block + dae_row_argmax
  d  the same chunked GEMM + torch.topk(k) per chunk (what a user writes for k > 1 without the fused kernel)
They run in rotating order after warm-up; times are CUDA events around one call.  Peaks are the H100 SXM data-sheet figures
(dense BF16: 989 TFLOP/s); executed FLOPs count the three bf16 products of the bf16x3 scheme.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dae_rnn_news_recommendation_b200 import helpers  # noqa: E402
from dae_rnn_news_recommendation_b200._cabi import call  # noqa: E402

DATASHEET_BF16_DENSE_TFLOPS = 989.0   # H100 SXM, 700 W


def _gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi failed: %s' % e


def sparse_main(args):
    """--sparse: the k most similar rows of bag-of-words vectors.  Paths, each from the CSR operands on the device to (index, score)
    on the device:
      a  dae_csr_similarity_topk (top_k_similar on scipy sparse input)
      b  densify + the dense top_k_similar (bf16x3 tensor cores), when the dense operands fit in device memory
      c  pairwise_similarity(sparse) + torch.topk, self search up to 20 000 rows (it forms the N x N matrix)
    Pair updates = sum_f df_q(f) df_c(f), the multiply-adds of a, counted from the data."""
    import scipy.sparse as sp
    from dae_rnn_news_recommendation_b200.engine import DeviceCSR
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    if args.data == 'c1':
        z = np.load(os.path.join(ROOT, 'tests', 'golden', 'uci_c1.npz'))
        x = sp.csr_matrix((np.ones(z['train_indices'].shape[0], np.float32), z['train_indices'], z['train_indptr']),
                          shape=tuple(int(v) for v in z['train_shape']))
        kind = 'binary'
    else:
        x = make_sparse(args.n, args.f, args.nnz, args.kind, seed=args.seed)
        kind = args.kind
    metric = 'cosine' if kind == 'binary' else 'linear kernel'   # what main_autoencoder.evaluate uses for the input vectors
    self_mode = args.queries <= 0
    q_host = x if self_mode else x[x.shape[0] - args.queries:]
    c_host = x if self_mode else x[:x.shape[0] - args.queries]
    qop, cop = helpers._csr_operand(q_host, metric), helpers._csr_operand(c_host, metric)
    nq, nc, f = qop.shape[0], cop.shape[0], qop.shape[1]
    dfq = np.bincount(qop.indices, minlength=f).astype(np.float64)
    dfc = np.bincount(cop.indices, minlength=f).astype(np.float64)
    updates = float((dfq * dfc).sum())
    dev = torch.device('cuda:0')
    dq = DeviceCSR(qop, dev)
    dc = dq if self_mode else DeviceCSR(cop, dev)
    K = args.k

    def path_a():
        return helpers._csr_similarity_topk(dq, dc, K, exclude=self_mode)

    def dense(d):
        return torch.sparse_csr_tensor(d.indptr, d.indices, d.values, size=d.shape, device=dev).to_dense()

    def path_b():
        xq = dense(dq)
        return helpers.top_k_similar(xq, k=K, corpus=None if self_mode else dense(dc), metric='linear kernel', to_host=False)

    def path_c():
        s = helpers.pairwise_similarity(q_host, metric=metric, to_host=False)
        s.fill_diagonal_(float('-inf'))
        v, i = torch.topk(s, K, dim=1)
        return i.int(), v

    paths = {'a_csr_topk': path_a}
    head = dfc > nc / 8                      # head columns: in more than 1/8 of the corpus rows
    if args.split_time:
        # where a's time goes: the same call with empty query rows (postings + slab scan only) and with the head columns dropped
        # from the queries (postings + scan + the tail's updates); the difference to a is the head columns' share
        dq_empty = DeviceCSR(sp.csr_matrix(qop.shape, dtype=np.float32), dev)
        q_tail = qop.copy()
        q_tail.data[head[q_tail.indices]] = 0.0
        q_tail.eliminate_zeros()
        dq_tail = DeviceCSR(q_tail, dev)
        paths['a0_empty_queries'] = lambda: helpers._csr_similarity_topk(dq_empty, dc, K, exclude=self_mode)
        paths['a1_queries_without_head_columns'] = lambda: helpers._csr_similarity_topk(dq_tail, dc, K, exclude=self_mode)
    dense_bytes = (nq + (0 if self_mode else nc)) * f * 12     # fp32 dense + bf16 hi / lo operands
    free = torch.cuda.mem_get_info()[0]
    if dense_bytes < 0.8 * free:
        paths['b_densify_dense_topk'] = path_b
    if self_mode and nq <= 20000:
        paths['c_pairwise_sparse_torch_topk'] = path_c
    names = list(paths)
    outputs, mem = {}, {}
    for name in names:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        outputs[name] = paths[name]()
        torch.cuda.synchronize()
        mem[name] = {'peak_above_inputs_bytes': torch.cuda.max_memory_allocated() - base}
        for _ in range(args.warmup - 1):
            paths[name]()
    torch.cuda.synchronize()
    times = {n: [] for n in names}
    for rep in range(args.reps):
        order = names[rep % len(names):] + names[:rep % len(names)]
        for name in order:
            if not name.startswith('a') and rep >= args.reps_other:
                continue
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            paths[name]()
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b))
    res = {'mode': 'sparse', 'data': args.data if args.data == 'c1' else 'synth_%s' % kind, 'metric': metric, 'self': self_mode,
           'Nq': nq, 'Nc': nc, 'F': f, 'nnz_q': int(qop.nnz), 'nnz_c': int(cop.nnz), 'k': K, 'reps': args.reps,
           'pair_updates': updates, 'pair_updates_over_nq_nc': updates / (nq * nc), 'head_columns': int(head.sum()),
           'head_share_of_updates': float((dfq * dfc)[head].sum() / max(updates, 1.0)), 'dense_nq_nc_f_over_updates': nq * nc * f / updates,
           'inputs_bytes': int(dq.h2d_bytes + (0 if self_mode else dc.h2d_bytes)), 'paths': {}}
    for name in names:
        ms = float(np.median(times[name]))
        res['paths'][name] = {'ms_median': ms, 'ms_min': float(min(times[name])), 'ms_all': [round(t, 3) for t in times[name]], **mem[name]}
    res['paths']['a_csr_topk']['pair_updates_per_s'] = updates / (res['paths']['a_csr_topk']['ms_median'] * 1e-3)
    ia, va = (t.cpu().numpy() for t in outputs['a_csr_topk'])
    res['agreement'] = {}
    for name in names[1:]:
        if name.startswith('a'):
            continue
        io, vo = (t.cpu().numpy() for t in outputs[name])
        res['agreement']['a_vs_' + name[0]] = {'same_index_lists': float((ia == io).all(1).mean()),
                                               'same_index_sets': float((np.sort(ia, 1) == np.sort(io, 1)).all(1).mean()),
                                               'max_abs_score_diff': float(np.abs(va - vo).max())}
    res['gpu'] = _gpu_info()
    res['device_name'] = torch.cuda.get_device_name(0)
    print(json.dumps(res))
    return 0


ap = argparse.ArgumentParser()
ap.add_argument('--sparse', action='store_true', help='bag-of-words vectors through the sparse top-k instead (sparse_main)')
ap.add_argument('--data', default='synth', choices=['synth', 'c1'], help='--sparse: synth.make_sparse, or tests/golden/uci_c1.npz')
ap.add_argument('--f', type=int, default=10000, help='--sparse: columns of the synthetic data')
ap.add_argument('--nnz', type=int, default=100, help='--sparse: mean entries per synthetic row')
ap.add_argument('--kind', default='tfidf', choices=['tfidf', 'binary'], help='--sparse: synthetic values')
ap.add_argument('--seed', type=int, default=0, help='--sparse: synthetic data seed')
ap.add_argument('--queries', type=int, default=0, help='--sparse: > 0: the last Q rows query the others; 0: self search')
ap.add_argument('--reps_other', type=int, default=3, help='--sparse: timed repetitions of paths b and c')
ap.add_argument('--split_time', action='store_true', help='--sparse: also time path a without the head columns and without queries')
ap.add_argument('--n', type=int, default=100000)
ap.add_argument('--h', type=int, default=500)
ap.add_argument('--k', type=int, default=10)
ap.add_argument('--chunk', type=int, default=8192, help='row chunk of paths c and d (nearest_neighbors default)')
ap.add_argument('--reps', type=int, default=5)
ap.add_argument('--warmup', type=int, default=2)
args = ap.parse_args()
N, H, K = args.n, args.h, args.k

if not torch.cuda.is_available():
    sys.exit('bench_topk: no CUDA device')
if args.sparse:
    sys.exit(sparse_main(args))
rng = np.random.RandomState(0)
labels = rng.randint(0, 4, N)
emb = (rng.randn(4, H)[labels] * 0.15 + rng.randn(N, H)).astype(np.float32)
dev = torch.device('cuda:0')
x = torch.from_numpy(emb).to(dev)
del emb
st = torch.cuda.current_stream().cuda_stream


def path_a():
    return helpers.top_k_similar(x, k=K, to_host=False)


def path_b():
    return helpers.top_k_similar(x, k=1, to_host=False)


def path_c():
    hi, lo, _ = helpers._normalised_operands(x, 2)
    idx = torch.empty(N, dtype=torch.int32, device=dev)
    val = torch.empty(N, dtype=torch.float32, device=dev)
    buf = torch.empty(min(args.chunk, N), N, dtype=torch.float32, device=dev)
    for r0 in range(0, N, args.chunk):
        r1 = min(N, r0 + args.chunk)
        helpers._gemm_nt((hi[r0:r1], lo[r0:r1]), (hi, lo), r1 - r0, N, H, buf)
        call('dae_row_argmax', buf.data_ptr(), r1 - r0, N, buf.stride(0), r0, 0, idx[r0:r1].data_ptr(), val[r0:r1].data_ptr(), st)
    return idx, val


def path_d():
    hi, lo, _ = helpers._normalised_operands(x, 2)
    idx = torch.empty(N, K, dtype=torch.int64, device=dev)
    val = torch.empty(N, K, dtype=torch.float32, device=dev)
    buf = torch.empty(min(args.chunk, N), N, dtype=torch.float32, device=dev)
    for r0 in range(0, N, args.chunk):
        r1 = min(N, r0 + args.chunk)
        helpers._gemm_nt((hi[r0:r1], lo[r0:r1]), (hi, lo), r1 - r0, N, H, buf)
        b = buf[:r1 - r0]
        b.diagonal(r0).fill_(float('-inf'))
        torch.topk(b, K, dim=1, out=(val[r0:r1], idx[r0:r1]))
    return idx, val


paths = {'a_fused_topk_k%d' % K: path_a, 'b_fused_topk_k1': path_b, 'c_chunked_gemm_row_argmax_k1': path_c,
         'd_chunked_gemm_torch_topk_k%d' % K: path_d}
names = list(paths)

outputs, mem = {}, {}
for name in names:
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    outputs[name] = paths[name]()
    torch.cuda.synchronize()
    mem[name] = {'max_memory_allocated': torch.cuda.max_memory_allocated(), 'above_inputs': torch.cuda.max_memory_allocated() - base}
    for _ in range(args.warmup - 1):
        paths[name]()
torch.cuda.synchronize()

times = {n: [] for n in names}
for rep in range(args.reps):
    order = names[rep % len(names):] + names[:rep % len(names)]
    for name in order:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        paths[name]()
        b.record()
        torch.cuda.synchronize()
        times[name].append(a.elapsed_time(b))

alg = 2.0 * N * N * H
res = {'N': N, 'H': H, 'k': K, 'chunk': args.chunk, 'reps': args.reps, 'paths': {}}
for name in names:
    ms = float(np.median(times[name]))
    res['paths'][name] = {'ms_median': ms, 'ms_min': float(min(times[name])), 'ms_all': [round(t, 3) for t in times[name]],
                          'algorithmic_tflops': alg / ms / 1e9, 'executed_tflops': 3 * alg / ms / 1e9,
                          'executed_over_datasheet_bf16_dense': 3 * alg / ms / 1e9 / DATASHEET_BF16_DENSE_TFLOPS, **mem[name]}

ia, va = (t.cpu().numpy() for t in outputs[names[0]])
ib, vb = (t.cpu().numpy() for t in outputs[names[1]])
ic, vc = (t.cpu().numpy() for t in outputs[names[2]])
idd, vd = (t.cpu().numpy() for t in outputs[names[3]])
res['agreement'] = {
    'a_vs_d_same_index_lists': float((ia == idd).all(1).mean()),
    'a_vs_d_same_index_sets': float((np.sort(ia, 1) == np.sort(idd, 1)).all(1).mean()),
    'a_vs_d_max_abs_score_diff': float(np.abs(va - vd).max()),
    'b_vs_c_same_index': float((ib[:, 0] == ic).mean()),
    'b_vs_c_max_abs_score_diff': float(np.abs(vb[:, 0] - vc).max()),
}
res['gpu'] = _gpu_info()
res['device_name'] = torch.cuda.get_device_name(0)
res['datasheet_bf16_dense_tflops'] = DATASHEET_BF16_DENSE_TFLOPS
print(json.dumps(res))
