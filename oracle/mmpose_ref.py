"""TEST INFRASTRUCTURE: a CPU restatement of the mmpose 0.29 pieces that Painter/eval/mmpose_custom calls but this
environment does not have (mmpose and mmcv are not installed).  Written from their documented behaviour under the
offline config (configs/coco_256x192_test_offline.py), with NumPy 2 (NEP 50) promotion:

    flip_back                       swap each flip pair's channels, then reverse the width
    _get_max_preds                  first maximum per heatmap; coordinates -1 where the maximum is <= 0
    keypoints_from_heatmaps         post_process 'default' only: +-0.25 towards the larger neighbour, transform_preds
    transform_preds                 crop coordinates back to the image (no UDP)
    bbox_xywh2cs                    box centre and scale, widened to the aspect ratio
    TopdownHeatmapHead.decode       the head's decode: keypoints and the per-box [c, s, area, score] rows
    oks_iou / oks_nms               object keypoint similarity and the greedy NMS on it
    TopDown                         stand-in detector base class (keypoint head, test_cfg)
    TopDownCocoDataset              stand-in dataset base class: _sort_and_unique_bboxes, _write_coco_keypoint_results

Used by tests/_pose_eval.py (as the stand-in modules the unmodified reference files import), tests/test_pose_host.py
and scripts/pose_post.py; nothing in painter_b200/ imports it.
"""
import json
import os
import warnings

import numpy as np


def flip_back(output_flipped, flip_pairs, target_type="GaussianHeatmap"):
    """[N, K, H, W] heatmaps of flipped images back to the original orientation: channels of each pair exchanged,
    columns reversed (a reversed view)."""
    if output_flipped.ndim != 4:
        raise ValueError("flip_back expects [N, K, H, W] heatmaps")
    if target_type.lower() != "gaussianheatmap":
        raise NotImplementedError(target_type)
    back = output_flipped.copy()
    for a, b in flip_pairs:
        back[:, a] = output_flipped[:, b]
        back[:, b] = output_flipped[:, a]
    return back[..., ::-1]


def _get_max_preds(heatmaps):
    """(preds float32 [N, K, 2], maxvals [N, K, 1]): x = idx % W, y = idx // W of np.argmax's first maximum, both -1
    where the maximum is not positive."""
    N, K, _, W = heatmaps.shape
    flat = heatmaps.reshape(N, K, -1)
    idx = np.argmax(flat, axis=2).reshape(N, K, 1)
    maxvals = np.amax(flat, axis=2).reshape(N, K, 1)
    preds = np.tile(idx, (1, 1, 2)).astype(np.float32)
    preds[:, :, 0] = preds[:, :, 0] % W
    preds[:, :, 1] = preds[:, :, 1] // W
    preds = np.where(np.tile(maxvals, (1, 1, 2)) > 0.0, preds, -1)
    return preds, maxvals


def transform_preds(coords, center, scale, output_size, use_udp=False):
    """Heatmap coordinates [K, 2] to image coordinates: x * (S / W) + c - S / 2 with S = scale * 200."""
    if use_udp:
        raise NotImplementedError("use_udp")
    size = scale * 200.0
    step_x = size[0] / output_size[0]
    step_y = size[1] / output_size[1]
    out = np.ones_like(coords)
    out[:, 0] = coords[:, 0] * step_x + center[0] - size[0] * 0.5
    out[:, 1] = coords[:, 1] * step_y + center[1] - size[1] * 0.5
    return out


def keypoints_from_heatmaps(heatmaps, center, scale, unbiased=False, post_process="default", kernel=11,
                            valid_radius_factor=0.0546875, use_udp=False, target_type="GaussianHeatmap"):
    """(preds [N, K, 2], maxvals [N, K, 1]) of float32 heatmaps [N, K, H, W]; post_process 'default' only."""
    if unbiased or use_udp or post_process != "default":
        raise NotImplementedError("only post_process='default' without unbiased decoding or UDP")
    heatmaps = heatmaps.copy()
    N, K, H, W = heatmaps.shape
    preds, maxvals = _get_max_preds(heatmaps)
    for n in range(N):
        for k in range(K):
            hm = heatmaps[n][k]
            px, py = int(preds[n][k][0]), int(preds[n][k][1])
            if 1 < px < W - 1 and 1 < py < H - 1:
                diff = np.array([hm[py][px + 1] - hm[py][px - 1], hm[py + 1][px] - hm[py - 1][px]])
                preds[n][k] += np.sign(diff) * .25
    for n in range(N):
        preds[n] = transform_preds(preds[n], center[n], scale[n], [W, H], use_udp=use_udp)
    return preds, maxvals


def bbox_xywh2cs(bbox, aspect_ratio, padding=1., pixel_std=200.):
    """(center float32 [2], scale float32 [2]) of an [x, y, w, h] box."""
    x, y, w, h = bbox[:4]
    center = np.array([x + w * 0.5, y + h * 0.5], dtype=np.float32)
    if w > aspect_ratio * h:
        h = w * 1.0 / aspect_ratio
    elif w < aspect_ratio * h:
        w = h * aspect_ratio
    scale = np.array([w, h], dtype=np.float32) / pixel_std
    return center, scale * padding


class TopdownHeatmapHead:
    """The part of TopdownHeatmapSimpleHead that forward_pseudo_test uses: target_type, test_cfg and decode."""

    def __init__(self, test_cfg=None, target_type="GaussianHeatmap"):
        self.test_cfg = dict(test_cfg or {})
        self.target_type = target_type

    def decode(self, img_metas, output, **kwargs):
        n = len(img_metas)
        bbox_ids = [] if "bbox_id" in img_metas[0] else None
        c = np.zeros((n, 2), dtype=np.float32)
        s = np.zeros((n, 2), dtype=np.float32)
        paths = []
        score = np.ones(n)
        for i, meta in enumerate(img_metas):
            c[i, :] = meta["center"]
            s[i, :] = meta["scale"]
            paths.append(meta["image_file"])
            if "bbox_score" in meta:
                score[i] = np.array(meta["bbox_score"]).reshape(-1)[0]
            if bbox_ids is not None:
                bbox_ids.append(meta["bbox_id"])
        cfg = self.test_cfg
        preds, maxvals = keypoints_from_heatmaps(
            output, c, s, unbiased=cfg.get("unbiased_decoding", False), post_process=cfg.get("post_process", "default"),
            kernel=cfg.get("modulate_kernel", 11), use_udp=cfg.get("use_udp", False), target_type=self.target_type)
        all_preds = np.zeros((n, preds.shape[1], 3), dtype=np.float32)
        all_boxes = np.zeros((n, 6), dtype=np.float32)
        all_preds[:, :, 0:2] = preds[:, :, 0:2]
        all_preds[:, :, 2:3] = maxvals
        all_boxes[:, 0:2] = c[:, 0:2]
        all_boxes[:, 2:4] = s[:, 0:2]
        all_boxes[:, 4] = np.prod(s * 200.0, axis=1)
        all_boxes[:, 5] = score
        return {"preds": all_preds, "boxes": all_boxes, "image_paths": paths, "bbox_ids": bbox_ids}


def oks_iou(g, d, a_g, a_d, sigmas=None, vis_thr=None):
    """float32 OKS of keypoint row g [K * 3] against each row of d [n, K * 3] (areas a_g, a_d)."""
    if sigmas is None:
        sigmas = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89,
                           .89]) / 10.0
    var = (sigmas * 2) ** 2
    xg, yg, vg = g[0::3], g[1::3], g[2::3]
    ious = np.zeros(len(d), dtype=np.float32)
    for i in range(len(d)):
        xd, yd, vd = d[i, 0::3], d[i, 1::3], d[i, 2::3]
        dx, dy = xd - xg, yd - yg
        e = (dx ** 2 + dy ** 2) / var / ((a_g + a_d[i]) / 2 + np.spacing(1)) / 2
        if vis_thr is not None:
            e = e[list(vg > vis_thr) and list(vd > vis_thr)]
        ious[i] = np.sum(np.exp(-e)) / e.shape[0] if e.shape[0] != 0 else 0.0
    return ious


def oks_nms(kpts_db, thr, sigmas=None, vis_thr=None, score_per_joint=False, kind=None):
    """Indices kept by greedy OKS NMS over dicts with 'score', 'keypoints' and 'area', highest score first.
    kind: np.argsort's kind for the score order (None: NumPy's default, as mmpose; "stable" defines ties)."""
    if len(kpts_db) == 0:
        return []
    if score_per_joint:
        scores = np.array([k["score"].mean() for k in kpts_db])
    else:
        scores = np.array([k["score"] for k in kpts_db])
    kpts = np.array([k["keypoints"].flatten() for k in kpts_db])
    areas = np.array([k["area"] for k in kpts_db])
    order = (scores.argsort() if kind is None else scores.argsort(kind=kind))[::-1]
    keep = []
    while len(order) > 0:
        i = order[0]
        keep.append(i)
        ovr = oks_iou(kpts[i], kpts[order[1:]], areas[i], areas[order[1:]], sigmas, vis_thr)
        order = order[np.where(ovr <= thr)[0] + 1]
    return np.array(keep)


def soft_oks_nms(*_a, **_k):
    raise NotImplementedError("soft OKS NMS is not used by the offline config")


class TopDown:
    """Stand-in detector base class: keeps the keypoint head and test_cfg, as TopDownCustom's methods read them."""

    def __init__(self, backbone=None, neck=None, keypoint_head=None, train_cfg=None, test_cfg=None, pretrained=None,
                 loss_pose=None):
        self.test_cfg = dict(test_cfg or {})
        self.keypoint_head = keypoint_head if keypoint_head is not None else TopdownHeatmapHead(self.test_cfg)
        self.with_neck = neck is not None

    @property
    def with_keypoint(self):
        return self.keypoint_head is not None


class _Coco:
    def __init__(self, ann_file):
        with open(ann_file) as f:
            self.dataset = json.load(f)


class TopDownCocoDataset:
    """Stand-in dataset base class: what evaluate() reads from a COCO keypoint dataset whose annotation file lists the
    images (id, file_name), and the two restated helpers."""

    def __init__(self, ann_file, img_prefix, data_cfg, pipeline, dataset_info=None, test_mode=False):
        self.img_prefix = img_prefix
        self.coco = _Coco(ann_file)
        self.name2id = {im["file_name"]: im["id"] for im in self.coco.dataset["images"]}
        self.ann_info = {"num_joints": data_cfg["num_joints"], "image_size": np.array(data_cfg["image_size"])}
        self.use_nms = data_cfg.get("use_nms", True)
        self.soft_nms = data_cfg["soft_nms"]
        self.oks_thr = data_cfg["oks_thr"]
        self.vis_thr = data_cfg["vis_thr"]
        self.sigmas = np.array(dataset_info["sigmas"])
        self.classes = ["person"]
        self._class_to_coco_ind = {"person": 1}
        names = {v["name"]: k for k, v in dataset_info["keypoint_info"].items()}
        pairs = []
        for k, v in dataset_info["keypoint_info"].items():
            if v["swap"] and [names[v["swap"]], k] not in pairs:
                pairs.append([k, names[v["swap"]]])
        self.ann_info["flip_pairs"] = pairs

    @staticmethod
    def _sort_and_unique_bboxes(kpts, key="bbox_id"):
        """Per image: sort by `key` (stable), then drop each entry whose key equals its predecessor's."""
        for img_id in kpts:
            people = sorted(kpts[img_id], key=lambda x: x[key])
            unique = people[:1]
            for p in people[1:]:
                if p[key] != unique[-1][key]:
                    unique.append(p)
            kpts[img_id] = unique
        return kpts

    def _write_coco_keypoint_results(self, keypoints, res_file):
        """One dict per kept person of every image, in order: image_id, category_id, keypoints (K * 3 floats), score,
        center, scale; written as JSON."""
        cat_id = self._class_to_coco_ind[self.classes[0]]
        K = self.ann_info["num_joints"]
        results = []
        for img_kpts in keypoints:
            if len(img_kpts) == 0:
                continue
            rows = np.array([p["keypoints"] for p in img_kpts]).reshape(-1, K * 3)
            for p, row in zip(img_kpts, rows):
                results.append({"image_id": p["image_id"], "category_id": cat_id, "keypoints": row.tolist(),
                                "score": float(p["score"]), "center": p["center"].tolist(),
                                "scale": p["scale"].tolist()})
        with open(res_file, "w") as f:
            json.dump(results, f, sort_keys=True, indent=4)


def write_image_list(path, images):
    """A COCO annotation file that lists `images` ({file_name: id}) and has no annotations."""
    with open(path, "w") as f:
        json.dump({"images": [{"id": int(i), "file_name": nm} for nm, i in images.items()]}, f)
    return path


def quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)
