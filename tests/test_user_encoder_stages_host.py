"""The stage recorder of tests/encoder_stages.py against the C ABI it decodes (no GPU needed): every export it knows is decoded
with the parameter names and count of its prototype in include/dae_sm100.h and its ctypes signature, and every export the user
encoders call is one it knows."""
import os
import re

import pytest

from encoder_stages import ARGS

from dae_rnn_news_recommendation_b200 import _cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _prototypes():
    """{export: (parameter names)} of the C prototypes in include/dae_sm100.h."""
    with open(os.path.join(ROOT, 'include', 'dae_sm100.h')) as f:
        text = re.sub(r'/\*.*?\*/', '', f.read(), flags=re.S)
    return {m.group(1): tuple(re.findall(r'(\w+)\s*$', p.strip())[0] for p in m.group(2).split(','))
            for m in re.finditer(r'\bint\s+(dae_\w+)\s*\(([^;{]*?)\)\s*;', text)}


@pytest.mark.parametrize('name', sorted(ARGS))
def test_decoded_arguments_match_the_c_abi(name):
    assert len(ARGS[name]) == len(_cabi._SIGNATURES[name][1]), name
    assert ARGS[name] == _prototypes()[name], name


def test_every_user_encoder_call_is_recorded():
    with open(os.path.join(ROOT, 'dae_rnn_news_recommendation_b200', 'user_model.py')) as f:
        called = set(re.findall(r"\bcall\(\s*'(dae_\w+)'", f.read()))
    assert len(called) >= 15, sorted(called)
    assert called <= set(ARGS), sorted(called - set(ARGS))


def test_unknown_export_fails():
    from encoder_stages import Recorder
    rec = Recorder(lambda *a: pytest.fail('an unknown export must not run'))
    with pytest.raises(AssertionError, match='does not know dae_colsum'):
        rec('dae_colsum', None, 1, 1, 1, None, None)
    assert rec.log == []
