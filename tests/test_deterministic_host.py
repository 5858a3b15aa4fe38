"""Deterministic mode without a GPU: the flag and DAE_DETERMINISTIC plumbing, the refusals, the workspace sizes, the CLI flag and
parameter.txt."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_flag_and_environment_variable(monkeypatch):
    from dae_rnn_news_recommendation_b200.engine import resolve_deterministic
    monkeypatch.delenv('DAE_DETERMINISTIC', raising=False)
    assert resolve_deterministic(None) is False
    monkeypatch.setenv('DAE_DETERMINISTIC', '1')
    assert resolve_deterministic(None) is True
    assert resolve_deterministic(False) is False     # an explicit value wins over the environment
    monkeypatch.setenv('DAE_DETERMINISTIC', '0')
    assert resolve_deterministic(None) is False and resolve_deterministic(True) is True


def test_unsupported_configurations_are_refused_before_any_buffer(monkeypatch):
    from dae_rnn_news_recommendation_b200.engine import TrainEngine, check_deterministic_supported
    with pytest.raises(ValueError, match="gemm='tc'"):
        TrainEngine(100, 10, gemm='ffma', deterministic=True)
    monkeypatch.setenv('DAE_GEMM', 'ffma')
    with pytest.raises(ValueError, match='CUDA-core'):
        TrainEngine(100, 10, deterministic=True)
    monkeypatch.delenv('DAE_GEMM')
    check_deterministic_supported('tc', None)         # one process, tensor cores: accepted

    class _Dist:                                      # a process group of four ranks
        @staticmethod
        def is_available():
            return True

        @staticmethod
        def is_initialized():
            return True

        @staticmethod
        def get_world_size(pg=None):
            return 4
    import dae_rnn_news_recommendation_b200.engine as engine
    monkeypatch.setattr(engine.torch, 'distributed', _Dist)
    with pytest.raises(ValueError, match='world size 4'):
        check_deterministic_supported('tc', None)


def test_workspace_sizes_match_hand_counts():
    from dae_rnn_news_recommendation_b200 import _cabi
    import ctypes
    # decode loss partials: two per 128-column tile
    assert _cabi.query('dae_decode_loss_parts', 10000, ctype=ctypes.c_int32) == 2 * 79
    assert _cabi.query('dae_decode_loss_parts', 128, ctype=ctypes.c_int32) == 2
    assert _cabi.query('dae_decode_loss_parts', 129, ctype=ctypes.c_int32) == 4

    def al(b):
        return (b + 255) // 256 * 256
    # encode backward at C2: B = 800, F = 10 000, H = 500, 80 000 entries.  Row tiles of 8 rows (100 tiles), chunks of 64 entries.
    B, F, H, cap = 800, 10000, 500, 80000
    want = (al(4 * (F + 1)) + al(4 * F) + 3 * al(4 * cap) + al(4 * 100 * F) + al(4 * (B // 4) * H) + al(4 * F * H)
            + al(4 * (cap // 64) * 2 * H) + al(4 * 7 * H))          # dbh: 200 CTA rows in 7 groups of 32
    assert _cabi.query('dae_encode_csr_bwd_det_workspace', B, F, H, cap) == want
    # 100 000 rows: the tile table is capped at 2^24 entries (1677 tiles of 60 rows), the chunk partials at 256 MB (chunks of 256)
    B, cap = 100000, 10 ** 7
    T = 100000 // 60 + 1
    want = (al(4 * (F + 1)) + al(4 * F) + 3 * al(4 * cap) + al(4 * T * F) + al(4 * (B // 4) * H) + al(4 * F * H)
            + al(4 * ((cap + 255) // 256) * 2 * H) + al(4 * 782 * H))   # 25 000 CTA rows in 782 groups
    assert _cabi.query('dae_encode_csr_bwd_det_workspace', B, F, H, cap) == want
    with pytest.raises(_cabi.DaeError):
        _cabi.query('dae_encode_csr_bwd_det_workspace', 0, F, H, cap)


def test_cli_flag():
    import main_autoencoder as cli
    import main_autoencoder_triplet as cli3
    assert cli.build_parser().parse_args([]).deterministic is False
    assert cli.build_parser().parse_args(['--deterministic']).deterministic is True
    assert cli3.build_parser().parse_args(['--deterministic']).deterministic is True


def test_parameter_file_is_unchanged(tmp_path, monkeypatch):
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder, DenoisingAutoencoderTriplet
    monkeypatch.chdir(tmp_path)
    texts = []
    for det in (False, True):
        m = DenoisingAutoencoder(model_name='p%d' % det, main_dir='p%d/' % det, deterministic=det)
        assert m.deterministic is det
        m._write_parameter_to_file(False)
        texts.append(open(m.parameter_file).read().replace('p%d' % det, 'p'))
    assert texts[0] == texts[1] and 'deterministic' not in texts[1]
    assert DenoisingAutoencoderTriplet(model_name='t', main_dir='t/', deterministic=True).deterministic is True
