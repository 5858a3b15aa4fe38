"""The C-ABI library loads without a GPU and exports every symbol include/dae_sm100.h declares."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def _declared():
    text = (ROOT / 'include' / 'dae_sm100.h').read_text()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\bint\s+(dae_[a-z0-9_]+)\s*\(', text)))


def test_header_symbols_are_exported_and_bound():
    from dae_rnn_news_recommendation_b200 import _cabi
    lib = _cabi.lib()
    declared = _declared()
    assert len(declared) >= 10
    for name in declared:
        assert hasattr(lib, name), 'missing export %s' % name
    assert sorted(_cabi.exported_symbols()) == declared
    assert lib.dae_version() >= 100


def test_every_export_is_called_by_name_from_a_test():
    """Each declared export appears as a quoted name ('dae_x' or "dae_x") in some tests/test_*.py other than this one, so no kernel
    is reached only through the Python layer or not at all."""
    here = Path(__file__).resolve()
    texts = [p.read_text() for p in sorted((ROOT / 'tests').glob('test_*.py')) if p.resolve() != here]
    missing = [n for n in _declared() if not any(("'%s'" % n) in t or ('"%s"' % n) in t for t in texts)]
    assert not missing, 'exports no test calls by name: %s' % missing


def test_bad_arguments_fail_loudly_without_gpu():
    import pytest
    from dae_rnn_news_recommendation_b200 import _cabi
    with pytest.raises(_cabi.DaeError) as e:
        _cabi.call('dae_sgemm', 0, 0, 0, 1.0, None, 0, 0, None, 0, 0, 0.0, None, 0, None)
    assert 'dae_sgemm' in str(e.value)


def test_engine_refuses_to_run_without_cuda():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    from dae_rnn_news_recommendation_b200 import _cabi
    from dae_rnn_news_recommendation_b200.engine import TrainEngine
    with pytest.raises(_cabi.DaeError):
        TrainEngine(100, 10)
