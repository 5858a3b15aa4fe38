"""References for the general GEMMs of csrc/gemm_tc.cu (dae_gemm_bf16x3, dae_gemm_bf16x3_det, dae_gemm_sym_bf16x3(_det)) and
csrc/sgemm.cu (dae_sgemm), for the kernel-level tests.  Tests only; nothing here needs a GPU.

Exact value.  The tensor-core kernels read every operand as two bf16 arrays and form, per 16-deep k step, three products:
    S = sum_k (a_hi b_hi + a_hi b_lo + a_lo b_hi)
(mma_kblock drops a_lo b_lo on purpose).  pair_exact() evaluates that sum in fp64 from the bit arrays the kernel actually reads.

Bound.  mining_kernel_oracle.gemm / gemm_c give |C - C_ref| <= c_K |alpha| sum_k |a_k b_k| (+ 2^-24 (|C_prev| + |C|) when C is
accumulated), with c_K = 2 x 2^-17 (the bf16 representation of each fp32 operand) + 2^-16 (the dropped lo.lo) + (3 K / 16) 2^-23
(the fp32 accumulator) + 2^-22 (the stream-K / split-K atomics).  Which terms apply:
  - fp32 operands split by dae_split_bf16, compared with the fp64 product of the fp32 values: all of c_K (gemm_c).
  - operands given as hi / lo pairs, compared with the fp64 product of the pair values hi + lo: no representation term
    (pair_c = gemm_c - 2 x 2^-17); the lo.lo term stays, because the reference keeps it and the kernel does not.
  - the exact operands of exact_operands(), compared with pair_exact(): no bound at all, bit for bit (below).

Exact operands.  exact_operands() writes hi and lo directly: hi holds integers in [-h, h], lo multiples of 2^-4 in [-1, 1], both
exactly representable in bf16.  Every product is then a multiple of 2^-4, and h is chosen from K so that K (h^2 + 2 h) <= 2^15: every
partial sum in any order and any split is a multiple of 2^-4 below 2^15 in magnitude, 19 significant bits, inside fp32's 24 with
room to spare for the tensor core's undocumented internal adder.  The sum is then exact in every engine, every split and every
atomic order.  alpha a power of two (negative too) keeps alpha S and C_0 + alpha S exact for C_0 on the same grid (exact_c0), so the
partial-tile paths must match bit for bit; on a path where one writer stores each element once, a general alpha gives exactly
fl32(alpha S) (and fl32(C_0 + fl32(alpha S)) when accumulating).

Dispatch.  dispatch() restates the host side of dae_gemm_bf16x3 / dae_gemm_bf16x3_det / dae_gemm_sym_bf16x3: stream-K or not, the
k_splits clamp and its no-empty-splits rounding, the cost64 / cost128 tile pick, the kernel instantiation and the CTA count; and
sk_cuts() the stream-K unit ranges u_c = c U / n_cta of Sched::init and sk_fixup_kernel.

dae_sgemm.  sgemm_ref(): fp64 with a per-element bound.  Each split runs one fp32 FMA chain over its k chunk (kchunk roundings),
then alpha acc (+ beta C) or, split-K, one atomic add per split onto beta C (pre-scaled, one rounding):
    |C - C_ref| <= 2^-24 (kchunk + splits + 2) (|alpha| sum_k |a_k b_k| + |beta C_0|).
"""
import re

import numpy as np

from mining_kernel_oracle import U, bf16_rn, gemm, gemm_c  # noqa: F401  (gemm re-exported for the tests)

BF16_NAN = 0x7FC0


def pair_c(K):
    """c_K for operands given as hi / lo pairs (no representation term)."""
    return gemm_c(K) - 2.0 * 2.0 ** -17


def bf16_value(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def pair_value(hi, lo):
    return bf16_value(hi) + bf16_value(lo)


def pair_exact(a_hi, a_lo, b_hi, b_lo):
    """sum_k (a_hi b_hi + a_hi b_lo + a_lo b_hi) in fp64 for A [M x K], B [N x K] given as bf16 bit arrays."""
    ah, al, bh, bl = (bf16_value(x) for x in (a_hi, a_lo, b_hi, b_lo))
    return ah @ bh.T + ah @ bl.T + al @ bh.T


def pair_bound(a_hi, a_lo, b_hi, b_lo, K, alpha=1.0, C0=None):
    """(reference, bound) of C = alpha A B^T (+ C0) with A, B given as hi / lo pairs (the pair_c terms)."""
    A, B = pair_value(a_hi, a_lo), pair_value(b_hi, b_lo)
    a = float(np.float32(alpha))
    C = a * (A @ B.T)
    bound = pair_c(K) * abs(a) * (np.abs(A) @ np.abs(B).T)
    if C0 is not None:
        C = C + C0
        bound = bound + U * (np.abs(C0) + np.abs(C))
    return C, bound


def exact_h(K):
    """Largest integer magnitude of hi with K (h^2 + 2 h) <= 2^15 (lo <= 1): every partial sum stays below 2^15."""
    h = 1
    while K * ((h + 1) ** 2 + 2 * (h + 1)) <= 2 ** 15 and h < 64:
        h += 1
    assert K * (h * h + 2 * h) <= 2 ** 15, 'K = %d too deep for exact operands' % K
    return h


def exact_operands(rng, rows, K, h=None):
    """hi (integers in [-h, h]) and lo (multiples of 2^-4 in [-1, 1]) bit arrays [rows x K]."""
    h = exact_h(K) if h is None else h
    hi = rng.integers(-h, h + 1, (rows, K)).astype(np.float32)
    lo = (rng.integers(-16, 17, (rows, K)) / 16.0).astype(np.float32)
    return bf16_rn(hi), bf16_rn(lo)


def exact_c0(rng, rows, cols):
    """C_0 on the 2^-4 grid, below 2^12."""
    return (rng.integers(-2 ** 16, 2 ** 16, (rows, cols)) / 16.0).astype(np.float32)


def check_exact(name, got, want):
    """Bit for bit: want (fp64) is exactly representable in fp32."""
    w32 = np.asarray(want, np.float64).astype(np.float32)
    assert np.array_equal(w32.astype(np.float64), np.asarray(want, np.float64)), '%s: the reference is not fp32-exact' % name
    got = np.asarray(got, np.float32)
    bad = got.view(np.uint32) != w32.view(np.uint32)
    if bad.any():
        idx = np.argwhere(bad)[:5].tolist()
        i = tuple(idx[0])
        raise AssertionError('%s: %d of %d elements differ; first %s: got %r want %r' % (name, int(bad.sum()), bad.size, idx, got[i], w32[i]))


# ---------------------------------------------------------------------------------------------------------------------------
# the host's dispatch (gemm_tc.cu: dae_gemm_bf16x3, dae_gemm_bf16x3_det, dae_gemm_sym_bf16x3(_det), launch_gemm_maj)
# ---------------------------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def dispatch(M, N, K, k_splits=1, sms=132, pair=False, lean=False, det=False, sym=False, a_mn=0, b_mn=0):
    """What the host launches.  Returns a dict:
        kernel    (BLOCK_N, STAGES, PAIR, MAJ, BK) of gemm_bf16x3_kernel
        stream_k  bool;   k_splits  after the clamp and the no-empty-splits rounding;   partial  split-K or stream-K
        tiles_m, tiles_n, tiles, kb (k-blocks of BK);   n_cta  CTAs (CTA pairs) of the launch;   fixup  sk_fixup_kernel<128> runs
    pair / lean: dae_gemm_config(1, 0) / (-1, 1) (dae_gemm_bf16x3 only; lean wins over pair).  sym: dae_gemm_sym_bf16x3(_det) with
    G [M x M] (K is ignored)."""
    maj = a_mn | (b_mn << 1)
    f32 = np.float32
    if sym:
        kb_half = _cdiv(M, 64)
        K = 2 * kb_half * 64
        cfg, stream_k, k_splits, maj = (128, 2, 0, 64), True, 1, 6
    else:
        tm, tn128, tn64 = _cdiv(M, 128), _cdiv(N, 128), _cdiv(N, 64)
        if det:
            stream_k = k_splits < 0 and (tm * tn128) % sms != 0
            k_splits = 1
            cost128 = f32(2.0) * f32(_cdiv(tm * tn128, sms))
            cost64 = f32(1.1) * f32(_cdiv(tm * tn64, sms))
            cfg = (128, 4, 0, 32) if stream_k else ((64, 3, 0, 64) if cost64 < cost128 else (128, 2, 0, 64))
        else:
            kblocks = _cdiv(K, 64)
            stream_k = False
            if k_splits < 0:
                stream_k = (tm * tn128) % sms != 0
                k_splits = 1
            k_splits = min(max(k_splits, 1), kblocks)
            per = _cdiv(kblocks, k_splits)
            k_splits = _cdiv(kblocks, per)
            cost128 = f32(2.0) * f32(_cdiv(tm * tn128 * k_splits, sms))
            cost64 = f32(1.1) * f32(_cdiv(tm * tn64 * k_splits, sms))
            if lean:
                cfg = (64, 2, 0, 64)
            elif pair:
                cfg = (128, 2, 1, 64)
            elif stream_k:
                cfg = (128, 4, 0, 32)
            elif cost64 < cost128:
                cfg = (64, 3, 0, 64)
            else:
                cfg = (128, 2, 0, 64)
    block_n, stages, pr, bk = cfg
    tiles_m = _cdiv(M, 128)
    if pr:
        tiles_m = _cdiv(tiles_m, 2)
    tiles_n = _cdiv(N, block_n)
    kb = _cdiv(K, bk)
    slots = sms // 2 if pr else sms
    if stream_k:
        n = min(max(tiles_m * tiles_n * kb // (6 * 64 // bk), 1), slots)
    else:
        n = min(tiles_m * tiles_n * k_splits, slots)
    return dict(kernel=(block_n, stages, pr, maj, bk), stream_k=bool(stream_k), k_splits=k_splits,
                partial=bool(stream_k or k_splits > 1), tiles_m=tiles_m, tiles_n=tiles_n, tiles=tiles_m * tiles_n, kb=kb, n_cta=n,
                fixup=bool(det and stream_k))


def sk_cuts(d):
    """Stream-K unit ranges [u_c, u_{c+1}) of the n_cta CTAs (u_c = c U / n_cta, U = tiles x kb), as Sched::init cuts them."""
    U = d['tiles'] * d['kb']
    return [c * U // d['n_cta'] for c in range(d['n_cta'] + 1)]


def sk_split_tiles(d):
    """Tiles whose k-blocks more than one CTA covers (a cut falls strictly inside the tile)."""
    kb = d['kb']
    return sorted({u // kb for u in sk_cuts(d)[1:-1] if u % kb})


def sk_aligned_partial(d):
    """CTAs whose range starts exactly at a tile's first k-block and ends inside that tile: their segment is the tile's first
    (workspace slot 0) although u_c == T0."""
    u, kb = sk_cuts(d), d['kb']
    return [c for c in range(d['n_cta']) if u[c] % kb == 0 and u[c + 1] - u[c] < kb and u[c + 1] > u[c]]


def sk_two_partials(d):
    """CTAs whose range covers the tail of one tile and the head of the next and nothing else (two partial segments)."""
    u, kb = sk_cuts(d), d['kb']
    return [c for c in range(d['n_cta']) if u[c] % kb and u[c + 1] % kb and u[c + 1] // kb == u[c] // kb + 1]


def split_k_stale(d, sms):
    """Uniform split-K: some CTA's second work item is one the requested (unrounded) k_splits would have made empty."""
    return d['tiles'] * d['k_splits'] > sms


KERNEL_RE = re.compile(r'gemm_bf16x3_kernel<(\d+), ?(\d+), ?(\d+), ?(\d+), ?(\d+)>')
FIXUP_RE = re.compile(r'sk_fixup_kernel<128>')


def kernel_of(name):
    """(BLOCK_N, STAGES, PAIR, MAJ, BK) of a gemm_bf16x3_kernel instantiation's demangled name, or None."""
    m = KERNEL_RE.search(name)
    return tuple(int(x) for x in m.groups()) if m else None


# ---------------------------------------------------------------------------------------------------------------------------
# dae_sgemm
# ---------------------------------------------------------------------------------------------------------------------------
def sgemm_splits(M, N, K, sms=132):
    """(splits, kchunk) of dae_sgemm: split-K when the 128 x 128 tiles do not fill the SMs and K >= 256."""
    tiles = _cdiv(N, 128) * _cdiv(M, 128)
    splits = 1
    if tiles < sms and K >= 256:
        splits = max(min(_cdiv(sms * 2, tiles), K // 64), 1)
    kchunk = _cdiv(_cdiv(K, splits), 16) * 16
    return _cdiv(K, kchunk), kchunk


def sgemm_c(M, N, K, sms=132):
    """c of dae_sgemm's bound c (|alpha| sum_k |a_k b_k| + |beta C_0|)."""
    splits, kchunk = sgemm_splits(M, N, K, sms)
    return U * (min(kchunk, K) + splits + 2)


def sgemm_ref(A, B, alpha, beta, C0, sms=132):
    """C = alpha A B^T + beta C0 (A [M x K], B [N x K], fp32 values), fp64, and the per-element bound (module docstring).  C0 may be
    None (beta = 0: the kernel never reads C)."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    M, K = A.shape
    N = B.shape[0]
    a, b = float(np.float32(alpha)), float(np.float32(beta))
    C = a * (A @ B.T)
    scale = abs(a) * (np.abs(A) @ np.abs(B).T)
    if b != 0.0:
        C0 = np.asarray(C0, np.float64)
        C = C + b * C0
        scale = scale + abs(b) * np.abs(C0)
    return C, sgemm_c(M, N, K, sms) * scale + 1e-37


def fl32_sum_orders(terms):
    """float32 sums of terms [n x K] along K in forward, reverse and blocked (16 blocks of partial sums, then the partials) order."""
    t = np.asarray(terms, np.float32)
    fwd = np.zeros(t.shape[0], np.float32)
    for k in range(t.shape[1]):
        fwd = fwd + t[:, k]
    rev = np.zeros(t.shape[0], np.float32)
    for k in reversed(range(t.shape[1])):
        rev = rev + t[:, k]
    parts = []
    for blk in np.array_split(np.arange(t.shape[1]), 16):
        s = np.zeros(t.shape[0], np.float32)
        for k in blk:
            s = s + t[:, k]
        parts.append(s)
    blocked = np.zeros(t.shape[0], np.float32)
    for s in reversed(parts):
        blocked = blocked + s
    return fwd, rev, blocked


def emulate_bf16x3(a_hi, a_lo, b_hi, b_lo):
    """float32 emulation of the kernel's main loop: per 16-deep k step the three products (lo.hi, hi.lo, hi.hi, small terms first)
    are each summed over the step in float32 and added to the float32 accumulator."""
    ah, al, bh, bl = (bf16_value(x).astype(np.float32) for x in (a_hi, a_lo, b_hi, b_lo))
    M, K = ah.shape
    acc = np.zeros((M, bh.shape[0]), np.float32)
    for k0 in range(0, K, 16):
        s = slice(k0, min(K, k0 + 16))
        for x, y in ((al, bh), (ah, bl), (ah, bh)):
            acc = (acc + (x[:, s] @ y[:, s].T).astype(np.float32)).astype(np.float32)
    return acc


def scaled_operand(rng, rows, cols, row_spread=20, col_spread=20):
    """fp32 [rows x cols] random normal with mixed signs, rows and columns scaled by 2^[-spread, spread]."""
    r = np.ldexp(1.0, rng.integers(-row_spread, row_spread + 1, rows))
    c = np.ldexp(1.0, rng.integers(-col_spread, col_spread + 1, cols))
    return (rng.standard_normal((rows, cols)) * r[:, None] * c[None, :]).astype(np.float32)


def worst_ratio(got, want, bound):
    return float(np.max(np.abs(np.asarray(got, np.float64) - want) / bound)) if np.size(want) else 0.0
