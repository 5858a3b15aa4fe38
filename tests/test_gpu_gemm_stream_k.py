"""The stream-K GEMM with the 4 x 32 operand ring (what dae_gemm_bf16x3 runs for every stream-K call in the default configuration)
against fp64, on shapes test_gpu_gemm_tc.py does not reach.  Every shape spreads its k loop over several CTAs, so partial tiles are
reduced across CTAs: K not a multiple of the 32-wide k-block (33: a tile's two k-blocks can land in two segments), the
[dW | dbv] special column in the last 128-wide n-tile, M not a multiple of 64, an odd C row stride, and alpha != 1 accumulated
into a non-zero C."""
import pytest
import torch

from helpers import rel_err
from test_gpu_gemm_tc import DEV, _gemm, _split

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('M,N,K', [(1000, 1001, 33), (100, 1001, 800), (333, 258, 3000), (200, 257, 4000)])
@pytest.mark.parametrize('a_mn,b_mn', [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_stream_k_ring(M, N, K, a_mn, b_mn):
    from dae_rnn_news_recommendation_b200 import _cabi
    _cabi.call('dae_gemm_config', -1, 0)
    # stream-K is chosen when the 128 x 128 tiles do not fill the SMs in whole waves; the 4 x 32 ring splits the
    # tiles x k-blocks units into segments of >= 12 k-blocks, so more than one CTA per tile means a cross-CTA reduction
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    tiles, kb = -(-M // 128) * -(-N // 128), -(-K // 32)
    n_cta = min(max(tiles * kb // 12, 1), sms)
    assert tiles % sms != 0 and any(c * tiles * kb // n_cta % kb for c in range(1, n_cta))   # a segment ends inside a tile
    g = torch.Generator(device=DEV).manual_seed(M * 3 + N + K)
    A = torch.randn(M, K, device=DEV, generator=g)
    B = torch.randn(N, K, device=DEV, generator=g)
    want = (A.double() @ B.double().t()).cpu().numpy()
    pad = lambda n: (n + 7) // 8 * 8
    Aop = _split(A.t().contiguous(), pad(M)) if a_mn else _split(A, pad(K))
    Bop = _split(B.t().contiguous(), pad(N)) if b_mn else _split(B, pad(K))
    # [C | special] = 0.5 A.B^T: the last column goes to its own vector (N = 258: C rows of 257 floats)
    C = torch.full((M, N - 1), float('nan'), device=DEV)
    sp = torch.full((M,), float('nan'), device=DEV)
    _gemm(M, N, K, Aop, a_mn, Bop, b_mn, C, n_store=N - 1, special_col=N - 1, special_out=sp, k_splits=-1, alpha=0.5)
    assert rel_err(C.cpu().numpy(), 0.5 * want[:, :N - 1]) < 2e-5
    assert rel_err(sp.cpu().numpy(), 0.5 * want[:, N - 1]) < 2e-5
    # C += -1.5 A.B^T on top of non-zero values
    C0 = torch.randn(M, N, device=DEV, generator=g)
    C2 = C0.clone()
    _gemm(M, N, K, Aop, a_mn, Bop, b_mn, C2, k_splits=-1, accumulate=1, alpha=-1.5)
    assert rel_err(C2.cpu().numpy(), C0.double().cpu().numpy() - 1.5 * want) < 2e-5
