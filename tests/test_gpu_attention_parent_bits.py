"""The fused attention computes exactly what it computed before its score loops were made branch-free: out, lse, dqkv
and the per-CTA table-gradient partials match, byte for byte, digests recorded from the earlier library
(tests/golden/attn_parent_bits.json, written by scripts/make_golden_attn_parent_bits.py)."""
import importlib.util
import json
import os

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script():
    spec = importlib.util.spec_from_file_location(
        "make_golden_attn_parent_bits", os.path.join(ROOT, "scripts", "make_golden_attn_parent_bits.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_MOD = _script()
with open(_MOD.FIXTURE) as _f:
    _GOLDEN = json.load(_f)["cases"]


@pytest.mark.parametrize("case", _MOD.CASES, ids=[c[0] for c in _MOD.CASES])
def test_attention_matches_parent_bits(case):
    got = _MOD.case_digests(*case)
    assert got == _GOLDEN[case[0]]
