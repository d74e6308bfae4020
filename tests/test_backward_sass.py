"""Machine code of the backward kernels that skip frozen-parameter work (no GPU): cuobjdump -sass of the built library.

The attention dQ kernel has two instantiations: with the G^T Q table-gradient partials (trainable rel-pos tables) and
without them (frozen tables).  Neither may contain a call, which would make ptxas serialise every wgmma (C7510; see
test_gemm_sass.py), or local-memory spills.  The one without the partials must have exactly one wgmma group (one
WARPGROUP.ARRIVE, four HGMMA) less: ptxas inserted no warpgroup.arrive of its own.  The LayerNorm and decoder-head
backward kernels, whose reductions are now optional, and the patch-embed input-gradient kernel must not spill: the
first two and the third use no local memory at all; the head backward's trainable forms keep a 128-byte local array
(as before this change), so its spills are read from ptxas's own report."""
import os
import re
import shutil
import subprocess

import pytest

from painter_b200 import _lib, build


def _cuobjdump():
    for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
              shutil.which("cuobjdump")):
        if c and os.path.exists(c):
            return c
    return None


@pytest.fixture(scope="module")
def kernels():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    assert os.path.exists(_lib.LIB_PATH), f"{_lib.LIB_PATH} not built"
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    out = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        out[name] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)
                     if not m.group(1).startswith("NOP")]
    return out


def _count(ins, pat):
    return sum(1 for i in ins if re.search(pat, i))


def _find(kernels, prefix):
    found = {n: ins for n, ins in kernels.items() if n.startswith(prefix)}
    assert found, prefix
    return found


def test_attention_dq_instantiations_have_no_call_or_spill(kernels):
    dq = _find(kernels, "_ZN2pk18attn_bwd_dq_kernelI")
    assert len(dq) == 2, sorted(dq)
    for name, ins in dq.items():
        assert _count(ins, r"\bCALL\b") == 0, name
        assert _count(ins, r"^(STL|LDL)\b") == 0, name


def test_dq_without_table_gradients_drops_exactly_one_wgmma_group(kernels):
    full = kernels["_ZN2pk18attn_bwd_dq_kernelILb1EEEvNS_8AttnArgsE"]
    lean = kernels["_ZN2pk18attn_bwd_dq_kernelILb0EEEvNS_8AttnArgsE"]
    assert _count(lean, r"^WARPGROUP\.ARRIVE") == _count(full, r"^WARPGROUP\.ARRIVE") - 1
    assert _count(lean, r"^HGMMA") == _count(full, r"^HGMMA") - 4


def test_backward_kernels_do_not_spill(kernels):
    for prefix in ("_ZN2pk13ln_bwd_kernelI", "_ZN2pk20ln_bwd_reduce_kernel", "_ZN2pk19col2im_patch_kernel"):
        for name, ins in _find(kernels, prefix).items():
            assert _count(ins, r"^(STL|LDL)\b") == 0, name


def test_head_backward_instantiations_do_not_spill():
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc (CUDA toolkit) not found")
    r = subprocess.run([nvcc, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, "decoder.cu"), "-o",
                        os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    report = {}
    name = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(_ZN2pk16head_bwd2_kernelI[^']*)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            report[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    assert len(report) == 3, report        # trainable head with / without dtgts, frozen head
    assert all(v == (0, 0) for v in report.values()), report
