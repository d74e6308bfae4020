"""Register spills of the wgmma GEMM (no GPU): gemm.cu compiled for sm_90a with `-Xptxas -v`.

A spill inside gemm_bf16_kernel puts local-memory traffic into the epilogue of every tile.  Every instantiation the
planner can choose by default must compile without one; the fp32, residual and GELU' kinds at BN = 256 still spill
a few bytes (their staged epilogue holds the fragments and the aux loads at once), so the planner must never pick
that tile width for them."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from painter_b200 import _lib
from painter_b200.build import CSRC, FLAGS, NVCC

EPI_BF16, EPI_F32, EPI_GELU, EPI_RESID, EPI_DGELU, EPI_PIXSHUF = range(6)
INSTANTIATIONS = [(k, bn) for k in range(6) for bn in (64, 128, 256)] + [(100, 64), (101, 64)]
NOT_PLANNED = {(EPI_F32, 256), (EPI_RESID, 256), (EPI_DGELU, 256)}


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc (CUDA toolkit) not found")
    obj = tmp_path_factory.mktemp("ptxas") / "gemm.o"
    r = subprocess.run([nvcc, *FLAGS, "-Xptxas=-v", "-c", os.path.join(CSRC, "gemm.cu"), "-o", str(obj)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '_ZN2pk16gemm_bf16_kernelILi(\d+)ELi(\d+)E", line)
        if m:
            cur = (int(m.group(1)), int(m.group(2)))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            out[cur] = int(m.group(1)) + int(m.group(2))
            cur = None
    return out


def test_every_instantiation_is_reported(ptxas_report):
    assert sorted(ptxas_report) == sorted(INSTANTIATIONS)


@pytest.mark.parametrize("kind,bn", [i for i in INSTANTIATIONS if i not in NOT_PLANNED])
def test_planned_instantiations_do_not_spill(ptxas_report, kind, bn):
    assert ptxas_report[(kind, bn)] == 0, f"gemm_bf16_kernel<{kind}, {bn}> spills {ptxas_report[(kind, bn)]} bytes"


WIDE = [(12544, 1024, 4096), (12544, 4096, 1024), (25088, 3072, 1024)]
WGRAD = [(4096, 1024, 12544), (1024, 4096, 12544), (16384, 4096, 12544)]


@pytest.mark.parametrize("M,N,K,kind,acc", [(*s, k, 0) for s in WIDE for k in (EPI_F32, EPI_RESID, EPI_DGELU)] +
                         [(*s, EPI_F32, 2) for s in WGRAD])
def test_planner_keeps_spilling_widths_out(M, N, K, kind, acc):
    out = (ctypes.c_int * 9)()
    L = _lib.lib()
    assert L.pk_gemm_plan(M, N, K, kind, acc, out) == 0, L.pk_last_error()
    assert (kind, out[1]) not in NOT_PLANNED
