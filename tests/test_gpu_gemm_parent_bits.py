"""The wgmma GEMM computes exactly what it computed while ptxas still serialised its wgmmas: every output written
without atomics matches, byte for byte, digests recorded from the earlier library (tests/golden/gemm_parent_bits.json,
written by scripts/make_golden_gemm_parent_bits.py) - at the tile width the planner picks, and at every width a call
can be forced to, since each output element sums its K-blocks in the same order whatever the tile."""
import importlib.util
import json
import os

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script():
    spec = importlib.util.spec_from_file_location(
        "make_golden_gemm_parent_bits", os.path.join(ROOT, "scripts", "make_golden_gemm_parent_bits.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_MOD = _script()
with open(_MOD.FIXTURE) as _f:
    _GOLDEN = json.load(_f)["cases"]


@pytest.mark.parametrize("case", _MOD.CASES)
def test_gemm_matches_parent_bits(case):
    assert _MOD.case_digests(case) == _GOLDEN[case]


@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("case", ["qkv_fwd", "fc2_fwd_resid", "fc2_dgrad_dgelu", "ragged_resid"])
def test_gemm_tile_width_does_not_change_bits(case, bn):
    from painter_b200._lib import lib
    lib().pk_gemm_force_bn(bn)
    try:
        got = _MOD.case_digests(case)
    finally:
        lib().pk_gemm_force_bn(0)
    assert got == _GOLDEN[case]
