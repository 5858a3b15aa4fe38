"""Long top-k lists (DESIGN 4.14): time of each stage, candidates per row and peak device memory above the inputs, against the
register kernels at k = 32 and a chunked GEMM + torch.topk arm.  Prints one JSON line.

    python tools/bench_topk_long.py [--n 100000] [--h 500] [--users 100000] [--articles 1000000] [--reps 3]

Arms (CUDA-event medians over --reps rounds, the arms in a rotated order each round):
  self_k32_register   top_k_similar(k=32) of n clustered articles against themselves (the register kernels)
  self_k32_long       the same through the three long-list stages (forced)
  self_k100_long / self_k1000_long
  users_k100_long     `users` random profiles against `articles` articles, k = 100, 20 read articles per user excluded
  self_k100_torch     8192-row chunks of the fp32 similarity from dae_gemm_bf16x3, then torch.topk (no self exclusion)
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dae_rnn_news_recommendation_b200 import helpers  # noqa: E402

STAGES = {'dae_similarity_topk_bound_bf16x3': 'bound', 'dae_similarity_topk_collect_bf16x3': 'collect', 'dae_pairs_sort': 'sort',
          'dae_similarity_topk_select': 'select', 'dae_similarity_topk_bf16x3': 'register', 'dae_gemm_bf16x3': 'gemm'}


class Recorder:
    """Wraps helpers.call: CUDA events around each stage export, and the candidate count passed to the select stage."""

    def __init__(self):
        self.real = helpers.call
        self.events, self.candidates = [], 0

    def __call__(self, name, *args):
        if name not in STAGES:
            return self.real(name, *args)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        self.real(name, *args)
        b.record()
        self.events.append((STAGES[name], a, b))
        if name == 'dae_similarity_topk_select':
            self.candidates += int(args[1])

    def stages(self):
        torch.cuda.synchronize()
        out = {}
        for s, a, b in self.events:
            out[s] = out.get(s, 0.0) + a.elapsed_time(b)
        return out


def torch_topk(x, k, chunk=8192):
    q = helpers._normalised_operands(x, 2)[:2]
    n = x.shape[0]
    buf = torch.empty(chunk, n, dtype=torch.float32, device=x.device)
    idx = torch.empty(n, k, dtype=torch.int64, device=x.device)
    val = torch.empty(n, k, dtype=torch.float32, device=x.device)
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        helpers._gemm_nt((q[0][r0:r1], q[1][r0:r1]), q, r1 - r0, n, x.shape[1], buf)
        v, i = torch.topk(buf[:r1 - r0], k, dim=1)
        val[r0:r1], idx[r0:r1] = v, i
    return idx, val


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=100000)
    ap.add_argument('--h', type=int, default=500)
    ap.add_argument('--users', type=int, default=100000)
    ap.add_argument('--articles', type=int, default=1000000)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_topk_long: needs a CUDA device')
    dev = torch.device('cuda:0')
    rng = np.random.RandomState(0)
    labels = rng.randint(0, 4, a.n)
    art = torch.from_numpy((rng.randn(4, a.h)[labels] * 0.15 + rng.randn(a.n, a.h)).astype(np.float32)).to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    corpus = torch.randn(a.articles, a.h, device=dev, generator=g)
    prof = torch.randn(a.users, a.h, device=dev, generator=g)
    reads = torch.randint(0, a.articles, (a.users, 20), device=dev, generator=g).sort(1).values
    keep = torch.ones_like(reads, dtype=torch.bool)
    keep[:, 1:] = reads[:, 1:] != reads[:, :-1]
    counts = keep.sum(1)
    ptr = torch.zeros(a.users + 1, dtype=torch.int64, device=dev)
    ptr[1:] = torch.cumsum(counts, 0)
    lists = helpers._DeviceLists(ptr, reads[keep].to(torch.int32).contiguous(), int(ptr[-1]))

    def forced(fn):
        def run():
            old = helpers.TOPK_MAX_K
            helpers.TOPK_MAX_K = 0
            try:
                return fn()
            finally:
                helpers.TOPK_MAX_K = old
        return run

    arms = {
        'self_k32_register': (a.n, lambda: helpers.top_k_similar(art, k=32, to_host=False)),
        'self_k32_long': (a.n, forced(lambda: helpers.top_k_similar(art, k=32, long_lists=True, to_host=False))),
        'self_k100_long': (a.n, lambda: helpers.top_k_similar(art, k=100, long_lists=True, to_host=False)),
        'self_k1000_long': (a.n, lambda: helpers.top_k_similar(art, k=1000, long_lists=True, to_host=False)),
        'users_k100_long': (a.users, lambda: helpers._recommend_topk(prof, corpus, 100, 'cosine', lists)),
        'self_k100_torch': (a.n, lambda: torch_topk(art, 100)),
    }
    times = {name: [] for name in arms}
    stages, cand, peak = {}, {}, {}
    names = list(arms)
    for _, fn in arms.values():   # warm-up: module loads, cub's and torch's first calls
        fn()
    torch.cuda.synchronize()
    for rep in range(a.reps):
        order = names[rep % len(names):] + names[:rep % len(names)]
        for name in order:
            rows, fn = arms[name]
            rec = Recorder()
            helpers.call = rec
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            try:
                t0.record()
                out = fn()
                t1.record()
                torch.cuda.synchronize()
            finally:
                helpers.call = rec.real
            del out
            times[name].append(t0.elapsed_time(t1))
            peak[name] = max(peak.get(name, 0), torch.cuda.max_memory_allocated() - base)
            stages.setdefault(name, []).append(rec.stages())
            if rec.candidates:
                cand[name] = rec.candidates / rows
    power = os.popen('nvidia-smi --query-gpu=name,power.limit --format=csv,noheader').read().strip()
    res = {'gpu': power, 'n': a.n, 'h': a.h, 'users': a.users, 'articles': a.articles, 'reps': a.reps}
    for name in names:
        st = {s: float(np.median([d.get(s, 0.0) for d in stages[name]])) for s in stages[name][0]}
        res[name] = {'ms': float(np.median(times[name])), 'stage_ms': st, 'candidates_per_row': cand.get(name),
                     'peak_mb_above_inputs': peak[name] / 2 ** 20}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
