"""Host logic of the GEMM scheduler (no GPU): for every shape the engine issues, the work items of all workers
(persistent CTAs) must tile the (row block, column block, k-block) space exactly once - classic
split-K, stream-K and the grouped rasterisation all go through the same code the kernels execute
(gemm_common.cuh: GemmSched, gemm_tile_coords; exported on the host as pk_gemm_plan / pk_gemm_plan_walk)."""
import ctypes

import numpy as np
import pytest

from painter_b200 import _lib

EPI_BF16, EPI_F32, EPI_GELU, EPI_RESID, EPI_DGELU, EPI_PIXSHUF = 0, 1, 2, 3, 4, 5

SHAPES = [
    # (M, N, K, kind, accumulate)      block-level GEMMs at B=8 (M = 12544 tokens) and B'=16 (25088)
    (12544, 3072, 1024, EPI_BF16, 0), (12544, 1024, 1024, EPI_RESID, 0), (12544, 4096, 1024, EPI_GELU, 0),
    (12544, 1024, 4096, EPI_RESID, 0), (12544, 4096, 1024, EPI_DGELU, 0), (12544, 1024, 4096, EPI_F32, 0),
    (12544, 1024, 3072, EPI_F32, 0), (25088, 3072, 1024, EPI_BF16, 0),
    # weight gradients: zero-initialised fp32 output -> stream-K
    (4096, 1024, 12544, EPI_F32, 2), (1024, 4096, 12544, EPI_F32, 2), (3072, 1024, 12544, EPI_F32, 2),
    (1024, 1024, 12544, EPI_F32, 2), (1024, 768, 25088, EPI_F32, 2), (16384, 4096, 12544, EPI_F32, 2),
    # decoder_embed (weights do not fit L2 -> grouped rasterisation) and small / ragged cases
    (12544, 16384, 4096, EPI_PIXSHUF, 0), (300, 64, 200, EPI_F32, 0), (768, 512, 4096, EPI_F32, 2),
    (512, 256, 640, EPI_F32, 2), (4096, 1024, 1000, EPI_F32, 2), (256, 128, 64, EPI_BF16, 0),
]


def _plan(M, N, K, kind, acc):
    L = _lib.lib()
    out = (ctypes.c_int * 9)()
    assert L.pk_gemm_plan(M, N, K, kind, acc, out) == 0, L.pk_last_error()
    keys = ["pair", "BN", "mt", "nt", "splits", "kbps", "sk_units", "group_m", "workers"]
    return dict(zip(keys, list(out)))


@pytest.mark.parametrize("M,N,K,kind,acc", SHAPES)
def test_every_k_block_of_every_tile_is_covered_exactly_once(M, N, K, kind, acc):
    L = _lib.lib()
    p = _plan(M, N, K, kind, acc)
    num_kb = (K + 63) // 64
    bm = 256 if p["pair"] else 128
    assert p["mt"] == (M + bm - 1) // bm and p["nt"] * p["BN"] == N
    cover = np.zeros((p["mt"], p["nt"], num_kb), dtype=np.int32)
    buf = (ctypes.c_int * (4 * 4096))()
    loads = []
    for w in range(p["workers"]):
        r = L.pk_gemm_plan_walk(M, N, K, kind, acc, w, buf, 4096)
        assert r <= 0, L.pk_last_error()
        items = np.array(buf[: 4 * (-r)], dtype=np.int64).reshape(-1, 4)
        loads.append(int((items[:, 3] - items[:, 2]).sum()))
        for mb, nb, k0, k1 in items:
            assert 0 <= mb < p["mt"] and 0 <= nb < p["nt"] and 0 <= k0 < k1 <= num_kb
            cover[mb, nb, k0:k1] += 1
    assert (cover == 1).all(), f"coverage min {cover.min()} max {cover.max()} for plan {p}"
    if p["sk_units"] > 0:   # stream-K: every CTA but the last carries the same number of k-blocks
        assert acc == 2 and max(loads) == p["sk_units"] and min(loads[:-1]) == p["sk_units"]


def test_weight_gradient_shapes_take_stream_k_and_small_n_takes_column_fastest_raster():
    p = _plan(4096, 1024, 12544, EPI_F32, 2)
    assert p["sk_units"] > 0 and p["workers"] <= 132
    q = _plan(12544, 1024, 4096, EPI_RESID, 0)        # weights (8 MB) stay L2-resident: column blocks adjacent
    assert q["group_m"] == 1 and q["sk_units"] == 0
    d = _plan(12544, 16384, 4096, EPI_PIXSHUF, 0)     # 134 MB of weights: groups of 8 row blocks
    assert d["group_m"] == 8
