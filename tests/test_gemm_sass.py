"""Machine code of the wgmma GEMM (no GPU): cuobjdump -sass of the built library.

ptxas serialises every wgmma of a kernel that contains a call (C7510: a wgmma pipeline crossing a function
boundary): each HGMMA is then followed by a wait for zero groups in flight, so the four k16 steps of a K-block wait
for each other and no K-block overlaps the release of the previous ring slot.  It does so silently, apart from an
info line, so the compiled kernels are checked here.  In every instantiation of gemm_bf16_kernel there is no CALL;
the K loop keeps one wgmma group in flight (`WARPGROUP.DEPBAR.LE gsb0, 0x1`), and the only wait for an empty wgmma
pipeline (`gsb0, 0x0`) is the one after the K loop, before the epilogue reads the accumulators."""
import os
import re
import shutil
import subprocess

import pytest

from painter_b200 import _lib

# 6 public epilogue kinds x BN 64 / 128 / 256, plus the decoder head (100) and the inverse pixel shuffle (101)
INSTANTIATIONS = [(k, bn) for k in range(6) for bn in (64, 128, 256)] + [(100, 64), (101, 64)]


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
        m = re.match(r"_ZN2pk16gemm_bf16_kernelILi(\d+)ELi(\d+)E", body)
        if not m:
            continue
        ins = []
        for line in body.split("\n"):
            im = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+([^;]*);", line)
            if im and not im.group(1).startswith("NOP"):
                ins.append(im.group(1).strip())
        out[(int(m.group(1)), int(m.group(2)))] = ins
    return out


def test_all_gemm_instantiations_present(kernels):
    assert sorted(kernels) == sorted(INSTANTIATIONS)


@pytest.mark.parametrize("kind,bn", INSTANTIATIONS)
def test_gemm_kernel_has_no_call(kernels, kind, bn):
    calls = [i for i in kernels[(kind, bn)] if re.search(r"\bCALL\b", i)]
    assert not calls, calls


@pytest.mark.parametrize("kind,bn", INSTANTIATIONS)
def test_gemm_wgmmas_are_not_serialised(kernels, kind, bn):
    ins = kernels[(kind, bn)]
    hgmma = [k for k, i in enumerate(ins) if i.startswith("HGMMA")]
    assert hgmma
    serial = [k for k in hgmma if k + 1 < len(ins) and re.match(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", ins[k + 1])]
    assert not serial, f"{len(serial)} of {len(hgmma)} HGMMA wait for an empty wgmma pipeline right after issue"
    drain = [i for i in ins if re.match(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", i)]
    assert len(drain) == 1, f"{len(drain)} waits for an empty wgmma pipeline (expected only the one after the K loop)"
    assert any(re.match(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", i) for i in ins), "no wgmma group is kept in flight"
