"""Host-side checks of painter_b200.task_metrics (no GPU): the scores computed from a confusion matrix, the refusal of
bad inputs before any device work, and ptxas's report on the metric kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from painter_b200 import build, task_metrics as tm


def _matrix(K, cells):
    m = np.zeros((K + 1, K + 1), dtype=np.int64)
    for (pred, gt), v in cells.items():
        m[pred, gt] = v
    return m


def test_scores_of_a_hand_built_matrix():
    # K = 4.  Class 2 is absent from the ground truth and never predicted, class 3 is only predicted (on class-0
    # pixels); the ignore column (gt = K) holds pixels predicted as 0 and 2, which count nowhere.
    m = _matrix(4, {(0, 0): 5, (1, 0): 1, (3, 0): 2, (1, 1): 4, (0, 1): 2, (0, 4): 7, (2, 4): 4})
    r = tm.semseg_scores(m)
    iou0, iou1 = 5 / (8 + 7 - 5), 4 / (6 + 5 - 4)
    acc0, acc1 = 5 / 8, 4 / 6
    assert r["mIoU"] == pytest.approx(100 * (iou0 + iou1) / 2, rel=1e-15)
    assert r["fwIoU"] == pytest.approx(100 * (iou0 * 8 / 14 + iou1 * 6 / 14), rel=1e-15)
    assert r["mACC"] == pytest.approx(100 * (acc0 + acc1) / 2, rel=1e-15)
    assert r["pACC"] == pytest.approx(100 * 9 / 14, rel=1e-15)
    np.testing.assert_allclose(r["IoU"][:2], [100 * iou0, 100 * iou1], rtol=1e-15)
    np.testing.assert_allclose(r["ACC"][:2], [100 * acc0, 100 * acc1], rtol=1e-15)
    assert np.isnan(r["IoU"][2:]).all() and np.isnan(r["ACC"][2:]).all()


def test_scores_of_a_perfect_prediction_with_an_absent_class():
    m = _matrix(3, {(0, 0): 10, (2, 2): 30, (1, 3): 5})
    r = tm.semseg_scores(m)
    assert r["mIoU"] == r["fwIoU"] == r["mACC"] == r["pACC"] == 100.0
    assert np.isnan(r["IoU"][1]) and np.isnan(r["ACC"][1])


def test_scores_of_ignore_only_pixels_are_undefined():
    m = _matrix(3, {(0, 3): 10, (2, 3): 4})
    with np.errstate(invalid="ignore", divide="ignore"):
        r = tm.semseg_scores(m)
    assert np.isnan(r["mIoU"]) and np.isnan(r["mACC"]) and np.isnan(r["pACC"])
    assert r["fwIoU"] == 0.0                # a sum over no valid class
    assert np.isnan(r["IoU"]).all() and np.isnan(r["ACC"]).all()


@pytest.fixture
def no_device(monkeypatch):
    """Any upload or library call fails the test: the inputs must be refused before."""
    def fail(*_a, **_k):
        raise AssertionError("device work before validation")
    monkeypatch.setattr(tm._se, "upload", fail)
    monkeypatch.setattr(tm, "lib", fail)


PAL = [(255, 255, 255), (0, 0, 0), (128, 64, 32)]


@pytest.mark.parametrize("palette", [np.zeros((0, 3)), np.zeros((201, 3)), np.zeros((4, 4)), np.zeros(3),
                                     [(1.5, 0, 0)], [(256, 0, 0)], [(-1, 0, 0)]])
def test_bad_palettes_are_refused(no_device, palette):
    with pytest.raises(ValueError):
        tm.SemSegMeter(palette)
    with pytest.raises(ValueError):
        tm.palette_classes(None, palette)


def test_palette_limits_are_accepted(no_device):
    tm.SemSegMeter(np.zeros((1, 3)))
    tm.SemSegMeter(np.full((200, 3), 255.0))


def test_bad_dist_type_is_refused(no_device):
    with pytest.raises(ValueError, match="dist_type"):
        tm.SemSegMeter(PAL, dist_type="euclid")
    with pytest.raises(ValueError, match="dist_type"):
        tm.palette_classes(None, PAL, dist_type="l2")


def test_semseg_shapes_that_disagree_are_refused(no_device):
    m = tm.SemSegMeter(PAL)
    good = np.zeros((4, 5, 3), np.uint8)
    for pred, gt in [(good, np.zeros((4, 6), np.uint8)), (good, np.zeros((5, 5), np.uint8)),
                     (np.zeros((4, 5), np.uint8), np.zeros((4, 5), np.uint8)),
                     (np.zeros((4, 5, 4), np.uint8), np.zeros((4, 5), np.uint8))]:
        with pytest.raises(ValueError, match="disagree"):
            m.update([good, pred], [np.zeros((4, 5), np.uint8), gt])
    with pytest.raises(ValueError):
        m.update([good], [])
    with pytest.raises(ValueError, match="uint8"):
        m.update([good], [np.zeros((4, 5), np.int64)])
    with pytest.raises(ValueError, match="uint8"):
        m.update([good.astype(np.float32)], [np.zeros((4, 5), np.uint8)])


def test_semseg_labels_outside_the_palette_are_refused(no_device):
    m = tm.SemSegMeter(PAL, ignore_label=255)
    gt = np.zeros((4, 5), np.uint8)
    gt[0, 0], gt[1, 1] = 255, 2           # the ignore label and the last class are fine ...
    gt_bad = gt.copy()
    gt_bad[3, 4] = 3                      # ... class 3 does not exist
    with pytest.raises(ValueError, match="labels >= 3"):
        m.update([np.zeros((4, 5, 3), np.uint8)], [gt_bad])
    m7 = tm.SemSegMeter(PAL, ignore_label=7)
    with pytest.raises(ValueError, match="labels >= 3"):
        m7.update([np.zeros((4, 5, 3), np.uint8)], [gt])          # 255 is not this meter's ignore label
    with pytest.raises(ValueError, match="ignore_label"):
        tm.SemSegMeter(PAL, ignore_label=256)


def test_depth_bad_inputs_are_refused(no_device):
    with pytest.raises(ValueError, match="min_depth"):
        tm.DepthMeter(min_depth=10.0, max_depth=1.0)
    m = tm.DepthMeter()
    with pytest.raises(ValueError, match="disagree"):
        m.update([np.zeros((480, 640), np.int32)], [np.zeros((480, 641), np.uint16)])
    with pytest.raises(ValueError, match="uint16"):
        m.update([np.zeros((480, 640), np.int32)], [np.zeros((480, 640), np.int32)])
    with pytest.raises(ValueError, match="int32"):
        m.update([np.zeros((480, 640), np.float32)], [np.zeros((480, 640), np.uint16)])


def test_restoration_bad_inputs_are_refused(no_device):
    x, g = np.zeros((9, 8, 3)), np.zeros((9, 8, 3), np.uint8)
    with pytest.raises(ValueError, match="7 x 7"):
        tm.restoration_scores([x, np.zeros((6, 8, 3))], [g, np.zeros((6, 8, 3), np.uint8)])
    with pytest.raises(ValueError, match="disagree"):
        tm.restoration_scores([x], [np.zeros((9, 9, 3), np.uint8)])
    with pytest.raises(ValueError, match="float64"):
        tm.restoration_scores([x.astype(np.float32)], [g])
    with pytest.raises(ValueError, match="CUDA"):
        tm.restoration_scores([x], [g], device="cpu")


def test_metric_kernels_do_not_spill():
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc (CUDA toolkit) not found")
    r = subprocess.run([nvcc, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, "metrics.cu"), "-o",
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
    # palette decode and confusion matrix for each of the three distances, depth errors, restoration scores
    assert len(report) == 8, report
    assert all(v == (0, 0, 0) for v in report.values()), report
