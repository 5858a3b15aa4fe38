"""Host side of the attention user encoder (user_model.UserAttention): the fp64 oracle of tests/user_attention_oracle.py against a CPU
torch.nn.MultiheadAttention plus pooling and against autograd, the kernel references composed in the packed layout against the
whole-batch oracle, the C ABI's argument checks, the constructor, state dicts, save / load and the CLI flags.  No GPU needed."""
import os
import sys

import numpy as np
import pytest
import torch

import user_attention_oracle as ao

from dae_rnn_news_recommendation_b200 import _cabi as c
from dae_rnn_news_recommendation_b200.user_model import (ATTENTION_NAMES, UserAttention, UserGRU, UserLSTM, default_heads)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _params(H, A, rng):
    return {'self_attn.in_proj_weight': rng.uniform(-0.4, 0.4, (3 * H, H)), 'self_attn.in_proj_bias': rng.uniform(-0.1, 0.1, 3 * H),
            'self_attn.out_proj.weight': rng.uniform(-0.3, 0.3, (H, H)), 'self_attn.out_proj.bias': rng.uniform(-0.1, 0.1, H),
            'pool.weight': rng.uniform(-0.3, 0.3, (A, H)), 'pool.bias': rng.uniform(-0.1, 0.1, A), 'pool.query': rng.uniform(-1, 1, A)}


def test_oracle_matches_torch_mha_and_pooling():
    H, A, heads = 12, 7, 3
    rng = np.random.default_rng(0)
    p = {k: torch.from_numpy(v) for k, v in _params(H, A, rng).items()}
    mha = torch.nn.MultiheadAttention(H, heads, batch_first=True).double()
    mha.load_state_dict({k[len('self_attn.'):]: v for k, v in p.items() if k.startswith('self_attn.')})
    for L in (1, 2, 9):
        X = torch.from_numpy(rng.standard_normal((L, H)))
        u, m = ao.encode(p, X, heads)
        for t in range(L):                       # the state at t is the encoder on the first t + 1 reads
            mask = torch.triu(torch.ones(t + 1, t + 1, dtype=torch.bool), 1)     # causal: read s attends to reads <= s
            with torch.no_grad():
                mm = mha(X[None, :t + 1], X[None, :t + 1], X[None, :t + 1], attn_mask=mask, need_weights=False)[0][0]
            a = torch.tanh(mm @ p['pool.weight'].T + p['pool.bias']) @ p['pool.query']
            torch.testing.assert_close(u[t], torch.softmax(a, 0) @ mm, rtol=1e-12, atol=1e-12)
            torch.testing.assert_close(m[t], mm[t], rtol=1e-12, atol=1e-12)


def _layout(lens):
    lens = np.sort(np.asarray(lens, np.int64))[::-1]
    n = np.array([(lens > t).sum() for t in range(int(lens[0]))])
    return lens, np.concatenate([[0], np.cumsum(n)]).astype(np.int64)


def test_kernel_references_compose_to_the_oracle():
    """attention_fwd -> out_proj -> pool_fwd in the packed layout equals the whole-batch oracle; pool_bwd and attention_bwd chained
    through the projections equal autograd of sum(dU . u)."""
    H, A, heads = 8, 5, 2
    rng = np.random.default_rng(1)
    pn = _params(H, A, rng)
    lens, off = _layout([5, 3, 1, 3])
    P = int(off[-1])
    X = rng.standard_normal((P, H))
    p = {k: torch.tensor(v, requires_grad=True) for k, v in pn.items()}
    qkv = X @ pn['self_attn.in_proj_weight'].T + pn['self_attn.in_proj_bias']
    fw = ao.attention_fwd(qkv, off, lens, H, heads)
    O = fw['O'][0]
    M = O @ pn['self_attn.out_proj.weight'].T + pn['self_attn.out_proj.bias']
    Z = M @ pn['pool.weight'].T + pn['pool.bias']
    pf = ao.pool_fwd(Z, pn['pool.query'], M, off, lens, H, A)
    dU = rng.standard_normal((P, H))
    total = 0
    for i, L in enumerate(lens):
        r = ao.rows(off, i, int(L))
        u, _ = ao.encode(p, torch.from_numpy(X[r]), heads)
        np.testing.assert_allclose(pf['u'][0][r], u.detach().numpy(), rtol=1e-11, atol=1e-12)
        total = total + (u * torch.from_numpy(dU[r])).sum()
    total.backward()
    pb = ao.pool_bwd(dU, pf['u'][0], M, Z, pn['pool.query'], pf['score'][0], pf['plse'][0], off, lens, H, A)
    np.testing.assert_allclose(pb['dq'][0], p['pool.query'].grad.numpy(), rtol=1e-10, atol=1e-12)
    dZ = pb['dZ'][0]
    np.testing.assert_allclose(dZ.T @ M, p['pool.weight'].grad.numpy(), rtol=1e-10, atol=1e-12)
    dM = pb['dM'][0] + dZ @ pn['pool.weight']
    np.testing.assert_allclose(dM.T @ O, p['self_attn.out_proj.weight'].grad.numpy(), rtol=1e-10, atol=1e-12)
    dO = dM @ pn['self_attn.out_proj.weight']
    dQKV = ao.attention_bwd(qkv, O, fw['lse'][0], dO, off, lens, H, heads)['dQKV'][0]
    np.testing.assert_allclose(dQKV.T @ X, p['self_attn.in_proj_weight'].grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(dQKV.sum(0), p['self_attn.in_proj_bias'].grad.numpy(), rtol=1e-10, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------------------------
# the C ABI's argument checks (each refused before any CUDA call)
# ---------------------------------------------------------------------------------------------------------------------------
P_ = 4096
SHAPE = dict(B=2, T=3, off=P_, lens=P_, H=8, heads=2)
FWD_OK = dict(SHAPE, qkv=P_, ld_qkv=24, o=P_, ld_o=8, o_hi=P_, o_lo=P_, ld_split=16, lse=P_, ld_lse=2, stream=None)
BWD_OK = dict(SHAPE, qkv=P_, ld_qkv=24, o=P_, ld_o=8, lse=P_, ld_lse=2, dout=P_, ld_do=8, dqkv_hi=P_, dqkv_lo=P_, ld_dqkv=24, stream=None)
PSHAPE = dict(B=2, T=3, off=P_, lens=P_, H=8, A=5)
PFWD_OK = dict(PSHAPE, z=P_, ld_z=5, q=P_, m=P_, ld_m=8, u=P_, ld_u=8, score=P_, plse=P_, stream=None)
PBWD_OK = dict(PSHAPE, du=P_, ld_du=8, u=P_, ld_u=8, m=P_, ld_m=8, z=P_, ld_z=5, q=P_, score=P_, plse=P_, dm=P_, ld_dm=8, dz_hi=P_,
               dz_lo=P_, ld_dz=8, dq=P_, workspace=P_, stream=None)
SHAPE_BAD = [('B', 0), ('T', 0), ('T', 1025), ('off', None), ('lens', None), ('H', 0), ('heads', 0), ('heads', 3)]
CASES = ([('dae_seq_attention_fwd', FWD_OK, k, v) for k, v in SHAPE_BAD + [('H', 258), ('qkv', None), ('ld_qkv', 23), ('o', None),
                                                                            ('ld_o', 7), ('o_hi', None), ('o_lo', None),
                                                                            ('ld_split', 7), ('lse', None), ('ld_lse', 1)]] +
         [('dae_seq_attention_bwd', BWD_OK, k, v) for k, v in SHAPE_BAD + [('qkv', None), ('ld_qkv', 23), ('o', None), ('lse', None),
                                                                            ('ld_lse', 1), ('dout', None), ('ld_do', 7),
                                                                            ('dqkv_hi', None), ('dqkv_lo', None), ('ld_dqkv', 23)]] +
         [('dae_seq_pool_fwd', PFWD_OK, k, v) for k, v in [('B', 0), ('T', 1025), ('A', 0), ('z', None), ('ld_z', 4), ('q', None),
                                                            ('m', None), ('ld_m', 7), ('u', None), ('ld_u', 7), ('score', None),
                                                            ('plse', None)]] +
         [('dae_seq_pool_bwd', PBWD_OK, k, v) for k, v in [('B', 0), ('T', 1025), ('H', 0), ('du', None), ('ld_du', 7), ('u', None),
                                                            ('m', None), ('z', None), ('ld_z', 4), ('q', None), ('dm', None),
                                                            ('ld_dm', 7), ('dz_hi', None), ('ld_dz', 4), ('dq', None),
                                                            ('workspace', None)]])


@pytest.mark.parametrize('name,ok,key,value', CASES, ids=['%s-%s=%s' % (n, k, v) for n, _, k, v in CASES])
def test_export_argument_checks(name, ok, key, value):
    args = dict(ok)
    args[key] = value
    with pytest.raises(c.DaeError, match=name):
        c.call(name, *args.values())
    assert c.last_error().startswith(name + ': ')


# ---------------------------------------------------------------------------------------------------------------------------
# constructor, parameters, files, CLI
# ---------------------------------------------------------------------------------------------------------------------------
def test_constructor_checks_and_default_heads():
    assert (default_heads(500), default_heads(37), default_heads(64), default_heads(1)) == (20, 1, 16, 1)
    assert UserAttention(500, device='cpu').heads == 20 and UserAttention(37, device='cpu').heads == 1
    for kw, msg in ((dict(heads=3), 'heads = 3'), (dict(heads=0), 'heads'), (dict(heads=True), 'heads'),
                    (dict(heads=1), 'head dim'), (dict(attention_dim=0), 'attention_dim'), (dict(attention_dim=2.5), 'attention_dim'),
                    (dict(max_len=1025), 'max_len'), (dict(opt='rmsprop'), 'opt'), (dict(impression_loss='x'), 'impression_loss'),
                    (dict(impression_negatives=33), 'impression_negatives'), (dict(batch_users=0), 'dim')):
        with pytest.raises(ValueError, match='UserAttention: .*' + msg):
            UserAttention(256, device='cpu', **kw)
    assert UserAttention(256, heads=2, max_len=1024, device='cpu').heads == 2


def test_state_dict_torch_round_trip_and_init():
    H, A = 12, 9
    m = UserAttention(H, heads=3, attention_dim=A, seed=3, device='cpu')
    sd = m.state_dict()
    assert tuple(sd) == ATTENTION_NAMES
    mha = torch.nn.MultiheadAttention(H, 3, batch_first=True)
    mha.load_state_dict({k[len('self_attn.'):]: v for k, v in sd.items() if k.startswith('self_attn.')})
    assert not sd['self_attn.in_proj_bias'].any() and not sd['self_attn.out_proj.bias'].any() and not sd['pool.bias'].any()
    assert float(sd['self_attn.in_proj_weight'].abs().max()) <= np.sqrt(6 / (4 * H))
    assert float(sd['self_attn.out_proj.weight'].abs().max()) <= 1 / np.sqrt(H)
    assert float(sd['pool.weight'].abs().max()) <= np.sqrt(6 / (A + H)) and float(sd['pool.query'].abs().max()) <= np.sqrt(6 / (A + 1))
    assert m.theta.numel() == (4 * H + A) * (H + 1) + A
    m2 = UserAttention(H, heads=3, attention_dim=A, seed=5, device='cpu')
    m2.load_state_dict(dict(sd))
    for k in ATTENTION_NAMES:
        assert torch.equal(m2.state_dict()[k], sd[k])
    with pytest.raises(ValueError, match='UserAttention.load_state_dict: missing'):
        m.load_state_dict({k: v for k, v in sd.items() if k != 'pool.query'})
    with pytest.raises(ValueError, match='pool.weight has shape'):
        m.load_state_dict(dict(sd, **{'pool.weight': torch.zeros(A + 1, H)}))


def test_save_load_and_cross_model_files(tmp_path):
    m = UserAttention(8, heads=2, attention_dim=6, max_len=7, seed=3, device='cpu')
    m.save(tmp_path / 'a.npz')
    m2 = UserAttention.load(tmp_path / 'a.npz', device='cpu')
    assert (m2.dim, m2.heads, m2.attention_dim, m2.max_len) == (8, 2, 6, 7)
    for k in ATTENTION_NAMES:
        assert torch.equal(m2.state_dict()[k], m.state_dict()[k])
    UserGRU(8, device='cpu').save(tmp_path / 'g.npz')
    with pytest.raises(ValueError, match=r"UserAttention.load: .* lacks \['attention_dim', 'heads', 'pool.bias'"):
        UserAttention.load(tmp_path / 'g.npz', device='cpu')
    for cls in (UserGRU, UserLSTM):
        with pytest.raises(ValueError, match=r"%s.load: .* lacks \['bias_hh_l0'" % cls.__name__):
            cls.load(tmp_path / 'a.npz', device='cpu')


def test_cli_flags(tmp_path):
    sys.path.insert(0, ROOT)
    import main_autoencoder as cli
    p = cli.build_parser()
    s = tmp_path / 's.npz'
    np.savez(s, indptr=np.array([0, 1]), items=np.array([0]))
    base = ['--top_k', '5', '--user_sequences', str(s)]
    F = cli.check_flags(p.parse_args(base + ['--user_cell', 'attention', '--user_heads', '4', '--user_attention_dim', '32']))
    assert (F.user_cell, F.user_heads, F.user_attention_dim) == ('attention', 4, 32)
    F = cli.check_flags(p.parse_args(base + ['--user_cell', 'attention']))
    assert (F.user_heads, F.user_attention_dim) == (None, 200)
    for extra in (['--user_heads', '4'], ['--user_attention_dim', '32'], ['--user_cell', 'lstm', '--user_heads', '2']):
        with pytest.raises(AssertionError, match='needs --user_cell attention'):
            cli.check_flags(p.parse_args(base + extra))
    with pytest.raises(AssertionError, match='--user_attention_dim must be >= 1'):
        cli.check_flags(p.parse_args(base + ['--user_cell', 'attention', '--user_attention_dim', '0']))
