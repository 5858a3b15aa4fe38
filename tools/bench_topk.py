"""k most similar articles for every article: the fused tensor-core top-k (helpers.top_k_similar) against the chunked similarity
matrix paths, on device-resident clustered embeddings (generated like tools/bench_evaluation.py's).  One JSON line.

    python tools/bench_topk.py [--n 100000] [--h 500] [--k 10] [--reps 5] [--warmup 2]

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

ap = argparse.ArgumentParser()
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
try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                       text=True, timeout=30)
    res['gpu'] = q.stdout.strip().splitlines()
except (OSError, subprocess.SubprocessError) as e:
    res['gpu'] = 'nvidia-smi failed: %s' % e
res['device_name'] = torch.cuda.get_device_name(0)
res['datasheet_bf16_dense_tflops'] = DATASHEET_BF16_DENSE_TFLOPS
print(json.dumps(res))
