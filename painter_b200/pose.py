"""COCO human pose post-processing on the GPU (kernels in csrc/pose.cu): the steps Painter's offline pose evaluation
(eval/mmpose_custom, configs/coco_256x192_test_offline.py) runs on the painted person crops and their flipped
paintings, computed from painter_inference.run_batch's device outputs without writing or reading PNG files.

    keypoint_palette     define_colors_gb_mean_sep(17) (data/pipelines/custom_transform.py) and the background
    COCO_FLIP_PAIRS      the flip pairs configs/_base_/coco.py's `swap` names give
    COCO_SIGMAS          configs/_base_/coco.py's sigmas
    box_center_scale     TopDownGetBboxCenterScale(padding=1.25): bbox_xywh2cs with the config's 192 x 256 input
    decode_keypoints     TopDownCustom.forward_pseudo_test (model/top_down.py): colour-decoded heatmaps, flip_back, the
                         one-pixel shift and the average; then the head's decode (keypoints_from_heatmaps with
                         post_process 'default', transform_preds)
    pose_results         TopDownCocoDatasetCustom.evaluate (data/topdown_coco_dataset.py) up to the JSON it writes:
                         de-duplication by bbox_id, rescoring, oks_nms per image, the result dicts

Every call validates its host-side inputs (ValueError) before any device work.  decode_keypoints makes one upload and
one launch per batch (plus the zeroing of its workspace); pose_results one upload, one launch and one download for the
whole dataset.  No heatmap is written to memory.  Results are bitwise reproducible; DESIGN.md records the arithmetic.
"""
import ctypes

import numpy as np
import torch

from ._lib import check, lib
from . import seggpt_engine as _se
from .panoptic import _device_of, _images, _pad16, _ptr
from .seggpt_engine import _stream

NUM_JOINTS = 17
MAX_BOXES_PER_IMAGE = 1024             # include/painter_b200.h PK_POSE_MAX_BOXES
_FIELDS = 4                            # PK_POSE_FIELDS
_ROW = 53                              # PK_POSE_ROW: position, score, 51 keypoint floats

# configs/_base_/coco.py: the pairs of keypoint_info's `swap` names, and the sigmas as written there
COCO_FLIP_PAIRS = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
COCO_SIGMAS = [0.026, 0.025, 0.025, 0.035, 0.035, 0.079, 0.079, 0.072, 0.072, 0.062, 0.062, 0.107, 0.107, 0.087,
               0.087, 0.089, 0.089]


def keypoint_palette():
    """uint8 [18, 2]: the (G, B) colours of define_colors_gb_mean_sep(17) in its dict order (G steps down from 255 by
    51 every 5 joints, B by 51 within them), then the background (0, 0): TopDownCustom.colors."""
    loc = np.arange(NUM_JOINTS)
    per = int(NUM_JOINTS ** 0.5) + 1                   # 5 steps per channel
    step = 256 // per                                  # 51
    gb = np.stack([255 - loc // per * step, 255 - loc % per * step], axis=1)
    return np.concatenate([gb, np.zeros((1, 2), dtype=gb.dtype)]).astype(np.uint8)


def box_center_scale(boxes_xywh, image_size=(192, 256), padding=1.25):
    """bbox_xywh2cs as TopDownGetBboxCenterScale(padding) applies it: per [x, y, w, h] box, the centre computed in
    double and stored as float32; w or h widened to the aspect ratio image_size[0] / image_size[1] in double; the
    scale [w, h] as float32 / 200, times padding, in float32.  Returns (centers, scales), float32 [N, 2] each."""
    b = np.asarray(boxes_xywh)
    if b.ndim != 2 or b.shape[1] != 4 or b.shape[0] < 1 or b.dtype.kind not in "fiu":
        raise ValueError(f"box_center_scale: boxes must be a real [N >= 1, 4] array, got {b.shape} {b.dtype}")
    b = b.astype(np.float64)
    if not np.all(np.isfinite(b)) or not np.all(b[:, 2:] > 0):
        raise ValueError("box_center_scale: boxes must be finite with positive width and height")
    if len(image_size) != 2 or min(image_size) <= 0:
        raise ValueError(f"box_center_scale: image_size must be (w, h) > 0, got {image_size!r}")
    if isinstance(padding, bool) or not isinstance(padding, (int, float, np.integer, np.floating)) or \
            not np.isfinite(padding) or padding <= 0:
        raise ValueError(f"box_center_scale: padding must be a positive number, got {padding!r}")
    aspect = float(image_size[0]) / float(image_size[1])
    x, y, w, h = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    centers = np.stack([x + w * 0.5, y + h * 0.5], axis=1).astype(np.float32)
    wide, tall = w > aspect * h, w < aspect * h
    h2 = np.where(wide, w * 1.0 / aspect, h)
    w2 = np.where(tall & ~wide, h * aspect, w)
    scales = np.stack([w2, h2], axis=1).astype(np.float32) / np.float32(200.0)
    return centers, scales * np.float32(padding)


def _pair_table(flip_pairs):
    swap = np.arange(NUM_JOINTS, dtype=np.int32)
    seen = set()
    try:
        pairs = [tuple(p) for p in flip_pairs]
    except TypeError:
        raise ValueError(f"flip_pairs must be a list of index pairs, got {flip_pairs!r}") from None
    for p in pairs:
        if len(p) != 2 or any(isinstance(v, bool) or not isinstance(v, (int, np.integer)) for v in p):
            raise ValueError(f"flip_pairs: {p!r} is not a pair of integers")
        a, b = int(p[0]), int(p[1])
        if not (0 <= a < NUM_JOINTS and 0 <= b < NUM_JOINTS) or a == b or a in seen or b in seen:
            raise ValueError(f"flip_pairs: pair {p!r} is outside [0, {NUM_JOINTS}) or repeats a joint")
        seen.update((a, b))
        swap[a], swap[b] = b, a
    return swap


def _host_f32(a, n, cols, what):
    if torch.is_tensor(a):
        if a.is_cuda:
            raise ValueError(f"{what} must be a host array")
        a = a.numpy()
    a = np.asarray(a)
    if a.dtype != np.float32 or a.shape != (n, cols):
        raise ValueError(f"{what} must be float32 [{n}, {cols}], got {a.dtype} {a.shape}")
    if not np.all(np.isfinite(a)):
        raise ValueError(f"{what} must be finite")
    return np.ascontiguousarray(a)


def _centers_scales(centers, scales, n):
    c = _host_f32(centers, n, 2, "centers")
    s = _host_f32(scales, n, 2, "scales")
    if not np.all(s > 0):
        raise ValueError("scales must be positive")
    return c, s


def _image_rows(images, dev, what, hw=None):
    """panoptic._images' checks (uint8 [H, W, 3] device tensors read in place, or host arrays staged in the upload),
    and one size for the whole batch, at least 3 x 3: (addresses, staged flags, staged arrays, (H, W))."""
    rows, staged, sizes = _images(images, dev, what)
    if hw is None:
        hw = sizes[0]
        if min(hw) < 3:
            raise ValueError(f"{what}: images must be at least 3 x 3, got {hw}")
    for i, sz in enumerate(sizes):
        if sz != hw:
            raise ValueError(f"{what}: image {i} is {sz}, the batch is {hw}")
    return rows[:, 0], rows[:, 1], staged, hw


def decode_keypoints(preds, centers, scales, flipped=None, flip_pairs=COCO_FLIP_PAIRS, device="cuda"):
    """Keypoints of N painted person crops: preds (and flipped, the paintings of the flipped crops) are N uint8
    [H, W, 3] RGB images of one size (run_batch(task="nearest") device tensors, or host arrays); centers / scales
    float32 [N, 2] (box_center_scale).  Equals TopDownCustom.forward_pseudo_test followed by the head's decode under
    the offline config: flip test exactly when `flipped` is given, shift_heatmap, post_process 'default', heatmap size
    W x H.  Returns a device float32 [N, 17, 3] of (x, y, maxval)."""
    n = len(preds)
    if flipped is not None and len(flipped) != n:
        raise ValueError(f"decode_keypoints: {n} images and {len(flipped)} flipped images")
    swap = _pair_table(flip_pairs)
    c, s = _centers_scales(centers, scales, n)
    dev = _device_of(device)
    addr, flag, staged, hw = _image_rows(preds, dev, "decode_keypoints")
    rows = np.zeros((n, _FIELDS), dtype=np.int64)
    rows[:, 0], rows[:, 1], rows[:, 3] = addr, flag, 2
    fstaged = []
    if flipped is not None:
        faddr, fflag, fstaged, _ = _image_rows(flipped, dev, "decode_keypoints (flipped)", hw=hw)
        rows[:, 2], rows[:, 3] = faddr, fflag
    cs = np.ascontiguousarray(np.concatenate([c, s], axis=1))
    # one upload: the table, centres / scales, then the staged images (their rows get byte offsets from the table)
    arrays, end = [rows, cs], 0
    for a in arrays:
        end += _pad16(a.nbytes)
    for col, items in ((0, staged), (2, fstaged)):
        for i, a in items:
            rows[i, col] = end
            arrays.append(a)
            end += _pad16(a.nbytes)
    tab, cs_d = _se.upload(arrays, dev)[:2]
    H, W = hw
    ws = torch.zeros(n * NUM_JOINTS * 2 + n, dtype=torch.int32, device=dev)     # argmax keys, per-box counters
    keys = ws[:n * NUM_JOINTS * 2]
    done = ws[n * NUM_JOINTS * 2:]
    out = torch.empty((n, NUM_JOINTS, 3), dtype=torch.float32, device=dev)
    pal = keypoint_palette()
    check(lib().pk_pose_decode(_ptr(tab), _ptr(tab), n, H, W, pal.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
                               swap.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), _ptr(cs_d), _ptr(keys), _ptr(done),
                               _ptr(out), _stream()), "pk_pose_decode")
    return out


def _ids(a, n, what):
    a = a.numpy() if torch.is_tensor(a) else np.asarray(a)
    if a.shape != (n,) or a.dtype.kind not in "iu":
        raise ValueError(f"{what} must be integers [{n}], got {a.dtype} {a.shape}")
    return a.astype(np.int64)


def _threshold(v, what):
    if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not np.isfinite(v):
        raise ValueError(f"{what} must be a finite number, got {v!r}")
    return np.float32(v)


def _groups(image_ids, bbox_ids):
    """_sort_and_unique_bboxes on ids alone: the images in order of their first box; within each, the positions
    sorted stably by bbox_id with repeated ids dropped (the first kept).  Returns (positions int32 [M], table int32
    [n_img, 2] of (start, count), the image ids)."""
    n = len(image_ids)
    uniq, first, inv = np.unique(image_ids, return_index=True, return_inverse=True)
    rank = np.empty(len(uniq), dtype=np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(len(uniq))
    img_rank = rank[inv.reshape(-1)]
    order = np.lexsort((np.arange(n), bbox_ids, img_rank))
    r, b = img_rank[order], bbox_ids[order]
    dup = np.zeros(n, dtype=bool)
    dup[1:] = (r[1:] == r[:-1]) & (b[1:] == b[:-1])
    pos, r = order[~dup], r[~dup]
    counts = np.bincount(r, minlength=len(uniq))
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    table = np.stack([starts, counts], axis=1).astype(np.int32)
    return pos.astype(np.int32), table, uniq[np.argsort(rank)]


def pose_results(keypoints, centers, scales, box_scores, image_ids, bbox_ids, vis_thr=0.2, oks_thr=0.9,
                 sigmas=COCO_SIGMAS, device="cuda"):
    """The COCO keypoint results of a whole dataset, as TopDownCocoDatasetCustom.evaluate writes them to
    result_keypoints.json (rle_score off, OKS NMS without soft NMS): keypoints float32 [N, 17, 3] (decode_keypoints'
    outputs of every batch in order, concatenated; device or host), centers / scales float32 [N, 2], box_scores [N]
    (stored as float32, as the head's decode does), image_ids / bbox_ids integers [N].  Per image (in order of its
    first box): the boxes sorted by bbox_id with repeated ids dropped, each rescored by the float32 mean of its joint
    scores above vis_thr times its box score, then oks_nms(oks_thr, sigmas) on the scores in descending order, equal
    scores the larger bbox_id first.  Returns the list of dicts (image_id, category_id 1, keypoints as 51 floats,
    score, center, scale) in image order and each image's keep order.  Host keypoints and the float32 box scores must
    be finite; device keypoints are read as they are, and any scores, NaN included, get the order numpy's argsort
    gives them (NaN above every number), with a NaN OKS suppressing, as the reference's `oks <= thr` test does."""
    n = len(box_scores) if hasattr(box_scores, "__len__") else -1
    if n < 1:
        raise ValueError("pose_results: box_scores must be a non-empty sequence")
    if torch.is_tensor(keypoints) and keypoints.is_cuda:
        dev = _device_of(device)
        if keypoints.dtype != torch.float32 or tuple(keypoints.shape) != (n, NUM_JOINTS, 3) or \
                not keypoints.is_contiguous() or keypoints.device != dev:
            raise ValueError(f"pose_results: keypoints must be a contiguous float32 [{n}, {NUM_JOINTS}, 3] tensor on "
                             f"{dev}, got {keypoints.dtype} {tuple(keypoints.shape)} on {keypoints.device}")
        kp_host = None
    else:
        kp_host = keypoints.numpy() if torch.is_tensor(keypoints) else np.asarray(keypoints)
        if kp_host.dtype != np.float32 or kp_host.shape != (n, NUM_JOINTS, 3):
            raise ValueError(f"pose_results: keypoints must be float32 [{n}, {NUM_JOINTS}, 3], got {kp_host.dtype} "
                             f"{kp_host.shape}")
        if not np.all(np.isfinite(kp_host)):
            raise ValueError("pose_results: keypoints must be finite")
        kp_host = np.ascontiguousarray(kp_host)
    c, s = _centers_scales(centers, scales, n)
    bs = box_scores.numpy() if torch.is_tensor(box_scores) else np.asarray(box_scores)
    if bs.shape != (n,) or bs.dtype.kind not in "fiu" or not np.all(np.isfinite(bs)):
        raise ValueError(f"pose_results: box_scores must be finite numbers [{n}]")
    bs = bs.astype(np.float32)
    if not np.all(np.isfinite(bs)):
        raise ValueError("pose_results: box_scores must be finite as float32 (|score| < 3.4e38)")
    img_ids = _ids(image_ids, n, "image_ids")
    box_ids = _ids(bbox_ids, n, "bbox_ids")
    vis = _threshold(vis_thr, "vis_thr")
    thr = _threshold(oks_thr, "oks_thr")
    sg = np.asarray(sigmas, dtype=np.float64) if np.ndim(sigmas) == 1 else np.zeros(0)
    if sg.shape != (NUM_JOINTS,) or not np.all(np.isfinite(sg)) or not np.all(sg > 0):
        raise ValueError(f"pose_results: sigmas must be {NUM_JOINTS} positive numbers")
    pos, table, order_ids = _groups(img_ids, box_ids)
    max_count = int(table[:, 1].max())
    if max_count > MAX_BOXES_PER_IMAGE:
        worst = order_ids[int(np.argmax(table[:, 1]))]
        raise ValueError(f"pose_results: image {worst} has {max_count} boxes after de-duplication (at most "
                         f"{MAX_BOXES_PER_IMAGE})")
    dev = _device_of(device)
    var = (sg * 2) ** 2                                # oks_iou's `vars`
    areas = np.prod(s * 200.0, axis=1)                 # the head's decode: float32 (s0 * 200) * (s1 * 200)
    n_img = table.shape[0]
    extra = [kp_host.reshape(n, -1)] if kp_host is not None else []
    views = _se.upload([table, pos, bs, areas] + extra, dev)
    tab_d, pos_d, bs_d, areas_d = views[:4]
    kp_d = views[4] if kp_host is not None else keypoints
    M = len(pos)
    out = torch.empty(M * _ROW + n_img, dtype=torch.int32, device=dev)
    L = lib()
    check(L.pk_pose_nms(_ptr(tab_d), n_img, max_count, _ptr(pos_d), _ptr(kp_d), _ptr(bs_d), _ptr(areas_d),
                        var.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), ctypes.c_float(vis),
                        ctypes.c_float(thr), _ptr(out), _ptr(out[M * _ROW:]), _stream()), "pk_pose_nms")
    host = out.cpu().numpy()
    rows = host[:M * _ROW].reshape(M, _ROW)
    counts = host[M * _ROW:]
    results = []
    for (start, _), k in zip(table, counts):
        for row in rows[start:start + k]:
            p = int(row[0])
            results.append({"image_id": int(img_ids[p]), "category_id": 1,
                            "keypoints": row[2:].view(np.float32).tolist(),
                            "score": float(row[1:2].view(np.float32)[0]),
                            "center": c[p].tolist(), "scale": s[p].tolist()})
    return results
