"""Host-side checks of painter_b200.panoptic (no GPU): the instance palette against the reference's generator, the
refusal of bad inputs before any device work, and ptxas's report on the panoptic kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ref_loader
from painter_b200 import build, panoptic as pn


@pytest.mark.skipif(not ref_loader.available(), reason="reference checkout / staged copy not found")
def test_instance_palette_equals_the_reference_generator():
    import _panoptic_eval as pe
    want = np.asarray(list(pe.palette_dict().values()), dtype=np.uint8)
    got = pn.instance_palette()
    assert got.dtype == np.uint8 and got.shape == (6400, 3)
    np.testing.assert_array_equal(got, want)


@pytest.fixture
def no_device(monkeypatch):
    """Any upload or library call fails the test: the inputs must be refused before."""
    def fail(*_a, **_k):
        raise AssertionError("device work before validation")
    monkeypatch.setattr(pn._se, "upload", fail)
    monkeypatch.setattr(pn, "lib", fail)
    monkeypatch.setattr(pn, "_device_of", lambda d: __import__("torch").device("cuda", 0))


IMG = np.zeros((4, 5, 3), dtype=np.uint8)


@pytest.mark.parametrize("dist_thr", [0.0, -1.0, float("nan"), float("inf"), [], [19.0] * 5, [16.0, 0.0], "19", True])
def test_bad_thresholds_are_refused(no_device, dist_thr):
    with pytest.raises(ValueError, match="dist_thr"):
        pn.decode_instances([IMG], dist_thr=dist_thr)


def test_bad_post_type_is_refused(no_device):
    with pytest.raises(ValueError, match="post_type"):
        pn.decode_instances([IMG], post_type="soft")


@pytest.mark.parametrize("img", [np.zeros((4, 5), np.uint8), np.zeros((4, 5, 4), np.uint8),
                                 np.zeros((4, 5, 3), np.float32), np.zeros((0, 5, 3), np.uint8)])
def test_bad_images_are_refused(no_device, img):
    with pytest.raises(ValueError):
        pn.decode_instances([img])


def test_empty_batch_is_refused(no_device):
    with pytest.raises(ValueError):
        pn.decode_instances([])


def test_bad_topk_is_refused(no_device):
    for k in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match="topk"):
            pn.decode_instances([IMG], topk=k)


def test_non_cuda_device_is_refused():
    with pytest.raises(ValueError, match="CUDA"):
        pn.decode_instances([IMG], device="cpu")


@pytest.mark.parametrize("palette", [np.zeros((79, 3)), np.zeros((201, 3)), np.zeros((100, 4)), np.zeros(3),
                                     np.full((100, 3), 256)])
def test_bad_semantic_palettes_are_refused(no_device, palette):
    with pytest.raises(ValueError, match="palette"):
        pn.classify_instances([], [], palette)
    with pytest.raises(ValueError, match="palette"):
        pn.panoptic_merge([], [], palette)


def test_ragged_instance_semantic_pairs_are_refused(no_device):
    pal = np.zeros((133, 3), np.uint8)
    with pytest.raises(ValueError):
        pn.classify_instances([], [IMG], pal)
    with pytest.raises(ValueError):
        pn.panoptic_merge([], [IMG], pal)


def test_bad_merge_thresholds_are_refused(no_device):
    pal = np.zeros((133, 3), np.uint8)
    for kw in ({"overlap_threshold": "0.5"}, {"stuff_area_thresh": float("nan")}, {"instances_score_thresh": None}):
        with pytest.raises(ValueError):
            pn.panoptic_merge([], [], pal, **kw)


def test_mask_bounds_follow_the_fp32_distance():
    d = np.arange(766, dtype=np.float32) * np.float32(1.0 / 3.0)
    for t in (0.2, 16.0, 16.5, 19.0, 255.0, 300.0):
        b = pn._bounds([t])[0]
        assert np.all(d[:b] < np.float32(t)) and np.all(d[b:] >= np.float32(t))


def test_panoptic_kernels_do_not_spill():
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc (CUDA toolkit) not found")
    r = subprocess.run([nvcc, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, "panoptic.cu"), "-o",
                        os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    report, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(_ZN2pk[^']*)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            report[name] = tuple(int(g) for g in m.groups())
            name = None
    assert len(report) == 18, sorted(report)
    assert all(v == (0, 0, 0) for v in report.values()), report
