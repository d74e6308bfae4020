"""Host-side checks of painter_b200.pose (no GPU): the palette and COCO constants against the staged reference files,
box_center_scale against the restated bbox_xywh2cs, the refusal of bad inputs before any device work, hand-computed
cases of the restated mmpose functions, and ptxas's report on the pose kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import mmpose_ref as mr
from oracle import ref_loader
from painter_b200 import build, pose

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="reference checkout / staged copy not found")


@needs_ref
def test_keypoint_palette_equals_the_reference_colours():
    import _pose_eval as pe
    got = pose.keypoint_palette()
    assert got.dtype == np.uint8 and got.shape == (18, 2)
    np.testing.assert_array_equal(got, np.asarray(pe.palette(), dtype=np.uint8))


@needs_ref
def test_coco_constants_equal_the_config(tmp_path):
    import _pose_eval as pe
    info = pe.coco_info()
    ann = mr.write_image_list(str(tmp_path / "ann.json"), {"x.jpg": 1})
    ds = mr.TopDownCocoDataset(ann, "", pe.DATA_CFG, [], dataset_info=info)
    assert ds.ann_info["flip_pairs"] == pose.COCO_FLIP_PAIRS
    assert np.array(pose.COCO_SIGMAS).dtype == np.float64
    np.testing.assert_array_equal(np.array(pose.COCO_SIGMAS), np.array(info["sigmas"]))


def test_box_center_scale_equals_bbox_xywh2cs():
    rng = np.random.default_rng(0)
    boxes = [[10.0, 20.0, 300.0, 100.0],          # wide
             [5.5, 7.25, 40.0, 200.0],            # tall
             [0.0, 0.0, 75.0, 100.0],             # exactly 3:4
             [1.0, 2.0, 150.0, 200.0]]
    boxes += rng.uniform(0.1, 400.0, size=(200, 4)).tolist()         # fractional
    c, s = pose.box_center_scale(boxes)
    assert c.dtype == np.float32 and s.dtype == np.float32
    aspect = np.array([192, 256])[0] / np.array([192, 256])[1]          # the pipeline's image_size is an int array
    for i, b in enumerate(boxes):
        rc, rs = mr.bbox_xywh2cs(b, aspect_ratio=aspect, padding=1.25)
        assert rc.dtype == np.float32 and rs.dtype == np.float32
        assert c[i].tobytes() == rc.tobytes() and s[i].tobytes() == rs.tobytes(), (b, c[i], rc, s[i], rs)


@pytest.fixture
def no_device(monkeypatch):
    """Any upload or library call fails the test: the inputs must be refused before."""
    def fail(*_a, **_k):
        raise AssertionError("device work before validation")
    monkeypatch.setattr(pose._se, "upload", fail)
    monkeypatch.setattr(pose, "lib", fail)
    monkeypatch.setattr(pose, "_device_of", lambda d: __import__("torch").device("cuda", 0))


IMG = np.zeros((256, 192, 3), dtype=np.uint8)
CS = np.ones((1, 2), dtype=np.float32)


@pytest.mark.parametrize("kw", [
    dict(preds=[]),
    dict(preds=[IMG, IMG]),                                           # 2 images, 1 centre
    dict(preds=[np.zeros((256, 192), np.uint8)]),
    dict(preds=[np.zeros((256, 192, 4), np.uint8)]),
    dict(preds=[IMG.astype(np.float32)]),
    dict(preds=[np.zeros((2, 192, 3), np.uint8)]),                    # smaller than 3 x 3
    dict(preds=[np.zeros((256, 2, 3), np.uint8)]),
    dict(flipped=[IMG, IMG]),                                         # flipped not pairing with preds
    dict(flipped=[np.zeros((128, 192, 3), np.uint8)]),                # flipped of another size
    dict(centers=CS.astype(np.float64)),
    dict(centers=np.ones((1, 3), np.float32)),
    dict(scales=np.zeros((1, 2), np.float32)),                        # non-positive scales
    dict(scales=-CS),
    dict(scales=np.full((1, 2), np.nan, np.float32)),
    dict(flip_pairs=[[1, 17]]),                                       # outside [0, 17)
    dict(flip_pairs=[[-1, 2]]),
    dict(flip_pairs=[[1, 2], [2, 3]]),                                # repeated
    dict(flip_pairs=[[1, 1]]),
    dict(flip_pairs=[[1, 2, 3]]),
])
def test_bad_decode_inputs_are_refused(no_device, kw):
    args = dict(preds=[IMG], centers=CS, scales=CS)
    args.update(kw)
    with pytest.raises(ValueError):
        pose.decode_keypoints(**args)


def test_batch_of_different_sizes_is_refused(no_device):
    with pytest.raises(ValueError, match="batch"):
        pose.decode_keypoints([IMG, np.zeros((128, 96, 3), np.uint8)], np.ones((2, 2), np.float32),
                              np.ones((2, 2), np.float32))


def _results_args(n=3, **kw):
    a = dict(keypoints=np.zeros((n, 17, 3), np.float32), centers=np.ones((n, 2), np.float32),
             scales=np.ones((n, 2), np.float32), box_scores=np.ones(n), image_ids=np.arange(n),
             bbox_ids=np.arange(n))
    a.update(kw)
    return a


@pytest.mark.parametrize("kw", [
    dict(keypoints=np.zeros((2, 17, 3), np.float32)),                 # mismatched lengths
    dict(keypoints=np.zeros((3, 17, 2), np.float32)),
    dict(keypoints=np.zeros((3, 17, 3), np.float64)),
    dict(centers=np.ones((2, 2), np.float32)),
    dict(scales=np.zeros((3, 2), np.float32)),
    dict(box_scores=np.ones(4)),
    dict(box_scores=np.array([1.0, np.nan, 1.0])),
    dict(box_scores=np.array([1.0, 1e39, 1.0])),                      # finite in float64, inf as float32
    dict(keypoints=np.full((3, 17, 3), np.inf, np.float32)),
    dict(keypoints=np.full((3, 17, 3), np.nan, np.float32)),
    dict(image_ids=np.arange(2)),
    dict(image_ids=np.arange(3.0)),
    dict(bbox_ids=np.arange(4)),
    dict(bbox_ids=np.array(["a", "b", "c"])),
    dict(vis_thr="0.2"),
    dict(oks_thr=float("nan")),
    dict(sigmas=[0.1] * 16),
    dict(sigmas=[0.0] * 17),
])
def test_bad_result_inputs_are_refused(no_device, kw):
    with pytest.raises(ValueError):
        pose.pose_results(**_results_args(**kw))


def test_more_than_1024_boxes_in_one_image_are_refused(no_device):
    n = 1100
    args = _results_args(n, image_ids=np.zeros(n, np.int64), bbox_ids=np.arange(n))
    with pytest.raises(ValueError, match="1024"):
        pose.pose_results(**args)


def test_repeated_bbox_ids_are_removed_before_the_limit(no_device, monkeypatch):
    # 1100 rows, but only 1000 distinct ids: passes validation and reaches the device (the upload stand-in)
    n = 1100
    args = _results_args(n, image_ids=np.zeros(n, np.int64), bbox_ids=np.arange(n) % 1000)
    with pytest.raises(AssertionError, match="device work"):
        pose.pose_results(**args)


def test_groups_follow_sort_and_unique_bboxes():
    rng = np.random.default_rng(1)
    n = 300
    image_ids = rng.integers(0, 12, n) * 7 + 100
    bbox_ids = rng.integers(0, 80, n)
    pos, table, ids = pose._groups(image_ids, bbox_ids)
    kpts = {}
    for i in range(n):
        kpts.setdefault(int(image_ids[i]), []).append({"bbox_id": int(bbox_ids[i]), "pos": i})
    want = mr.TopDownCocoDataset._sort_and_unique_bboxes(kpts)
    assert [int(v) for v in ids] == list(want.keys())
    for (start, count), (img, people) in zip(table, want.items()):
        assert [int(p) for p in pos[start:start + count]] == [p["pos"] for p in people]


# ---------------------------------------------------------------------------------------------------------------------
# The restated mmpose functions on hand-computed cases.

def _decode_one(hm, center=(0.0, 0.0), scale=(0.96, 1.28)):
    c = np.array([center], np.float32)
    s = np.array([scale], np.float32)
    return mr.keypoints_from_heatmaps(hm[None, None].astype(np.float32), c, s)


def test_keypoints_from_heatmaps_hand_cases():
    H, W = 6, 5                                         # S = (192, 256): step 192 / 5 = 38.4, 256 / 6
    # interior peak with a larger right and lower neighbour: +0.25 in x and y
    hm = np.zeros((H, W), np.float32)
    hm[3, 2], hm[3, 3], hm[3, 1], hm[4, 2], hm[2, 2] = 1.0, 0.5, 0.25, 0.5, 0.25
    p, m = _decode_one(hm)
    sx, sy = np.float32(192.0) / np.float32(W), np.float32(256.0) / np.float32(H)
    assert m[0, 0, 0] == np.float32(1.0)
    assert p[0, 0, 0] == np.float32(np.float32(2.25) * sx) - np.float32(96.0)
    assert p[0, 0, 1] == np.float32(np.float32(3.25) * sy) - np.float32(128.0)
    # px = 1 is not inside (1 < px is strict): no shift
    hm = np.zeros((H, W), np.float32)
    hm[3, 1], hm[3, 2] = 1.0, 0.5
    p, _ = _decode_one(hm)
    assert p[0, 0, 0] == np.float32(np.float32(1.0) * sx) - np.float32(96.0)
    # maxval 0: both coordinates -1
    p, m = _decode_one(np.zeros((H, W), np.float32))
    assert m[0, 0, 0] == 0.0
    assert p[0, 0, 0] == np.float32(np.float32(-1.0) * sx) - np.float32(96.0)
    assert p[0, 0, 1] == np.float32(np.float32(-1.0) * sy) - np.float32(128.0)
    # a flat top: the first maximum in row-major order
    hm = np.zeros((H, W), np.float32)
    hm[2, 3] = hm[3, 2] = hm[3, 3] = 0.5
    p, _ = _decode_one(hm)
    assert p[0, 0, 0] == np.float32(np.float32(3.0) * sx) - np.float32(96.0)      # (3, 2): right 0, left 0
    assert p[0, 0, 1] == np.float32(np.float32(2.25) * sy) - np.float32(128.0)    # below 0.5 > above 0


def test_flip_back_and_shift():
    hm = np.arange(2 * 3 * 4, dtype=np.float32).reshape(1, 2, 3, 4)
    out = mr.flip_back(hm, [[0, 1]])
    np.testing.assert_array_equal(out[0, 0], hm[0, 1, :, ::-1])
    out[:, :, :, 1:] = out[:, :, :, :-1]
    np.testing.assert_array_equal(out[0, 0, :, 0], hm[0, 1, :, 3])
    np.testing.assert_array_equal(out[0, 0, :, 1:], hm[0, 1, :, ::-1][:, :-1])


def _person(x, y, score, area=10000.0):
    kp = np.zeros((17, 3), np.float32)
    kp[:, 0], kp[:, 1], kp[:, 2] = x + np.arange(17), y + 2 * np.arange(17), 0.9
    return {"keypoints": kp, "score": np.float32(score), "area": np.float32(area)}


def test_oks_of_identical_and_distant_poses():
    a = _person(100, 100, 1.0)
    d = np.array([a["keypoints"].flatten(), _person(400, 100, 1.0)["keypoints"].flatten()])
    ious = mr.oks_iou(a["keypoints"].flatten(), d, a["area"], np.array([a["area"], a["area"]]),
                      sigmas=np.array(pose.COCO_SIGMAS))
    assert ious.dtype == np.float32 and ious[0] == np.float32(1.0) and 0 <= ious[1] < 1e-30
    # one joint off by (3, 4): e = 25 / (2 sigma)^2 / (area + 2^-52) / 2, averaged with 16 ones
    b = a["keypoints"].copy()
    b[5, 0] += 3
    b[5, 1] += 4
    e = 25.0 / (2 * 0.079) ** 2 / (10000.0 + 2.0 ** -52) / 2
    got = mr.oks_iou(a["keypoints"].flatten(), b.flatten()[None], a["area"], np.array([a["area"]]),
                     sigmas=np.array(pose.COCO_SIGMAS))[0]
    assert got == np.float32((16 + np.exp(-e)) / 17)


def test_oks_nms_hand_cases():
    sig = np.array(pose.COCO_SIGMAS)
    people = [_person(100, 100, 0.5), _person(100.5, 100, 0.9), _person(300, 100, 0.7), _person(300.2, 100, 0.2)]
    keep = mr.oks_nms(people, 0.9, sigmas=sig)
    assert list(keep) == [1, 2]
    # equal scores: with the stable order reversed, the later box comes first
    tied = [_person(100, 100, 0.0), _person(100.1, 100, 0.0), _person(500, 100, 0.0)]
    assert list(mr.oks_nms(tied, 0.9, sigmas=sig, kind="stable")) == [2, 1]


def test_pose_kernels_do_not_spill():
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc (CUDA toolkit) not found")
    r = subprocess.run([nvcc, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, "pose.cu"), "-o",
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
    assert len(report) == 2, sorted(report)
    assert all(v == (0, 0, 0) for v in report.values()), report
