"""COCO pose post-processing on the GPU (painter_b200.pose) against the unmodified reference TopDownCustom and
TopDownCocoDatasetCustom (tests/_pose_eval.py) on seeded synthetic painted crops."""
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import _pose_eval as pe
from oracle import mmpose_ref as mr
from oracle import ref_loader
from painter_b200 import pose

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_loader.available(), reason="reference checkout / staged copy not found")]

BATCH = 32                              # the offline config's samples_per_gpu


def _crops(seed, n):
    rng = np.random.default_rng(seed)
    pairs = [pe.painted_pair(rng) for _ in range(n)]
    boxes = pe.boxes_for(rng, n)
    c, s = pose.box_center_scale(boxes)
    return [p for p, _ in pairs], [f for _, f in pairs], c, s, rng.uniform(0.2, 1.0, n)


def _names(n, stem="000000000785"):
    return [f"{stem}_box{i}_image.png" for i in range(n)]


def _reference(tmp_path, preds, flipped, c, s, scores, bbox_ids, names):
    """forward_pseudo_test in batches of 32 on PNG files: the list of per-batch results."""
    paths = pe.write_pngs(str(tmp_path), names, preds, flipped)
    mdl = pe.model(flip_test=flipped is not None)
    out = []
    for b in range(0, len(paths), BATCH):
        sl = slice(b, b + BATCH)
        out.append(pe.forward_pseudo_test(mdl, paths[sl], c[sl], s[sl], scores[sl], bbox_ids[sl],
                                          pose.COCO_FLIP_PAIRS))
    return out


def _decode_batches(preds, flipped, c, s, to_device=True):
    outs = []
    for b in range(0, len(preds), BATCH):
        sl = slice(b, b + BATCH)
        p = [torch.from_numpy(a).cuda() for a in preds[sl]] if to_device else preds[sl]
        f = None if flipped is None else ([torch.from_numpy(a).cuda() for a in flipped[sl]] if to_device
                                          else flipped[sl])
        outs.append(pose.decode_keypoints(p, c[sl], s[sl], flipped=f))
    return torch.cat(outs)


@pytest.mark.parametrize("n", [1, 7, 64])
@pytest.mark.parametrize("flip", [True, False])
def test_decode_matches_forward_pseudo_test(tmp_path, n, flip):
    preds, flipped, c, s, scores = _crops(10 + n, n)
    flipped = flipped if flip else None
    ref = _reference(tmp_path, preds, flipped, c, s, scores, np.arange(n), _names(n))
    want = np.concatenate([r["preds"] for r in ref])
    for to_device in (True, False):
        got = _decode_batches(preds, flipped, c, s, to_device).cpu().numpy()
        assert got.dtype == np.float32 and got.shape == (n, 17, 3)
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert len(bad) == 0, (to_device, bad[:8], got[tuple(bad[0])], want[tuple(bad[0])])
    maxvals = want[:, :, 2]
    assert np.any(maxvals == 0) and np.any(maxvals > 0)
    if n == 7:
        one = torch.cat([pose.decode_keypoints([torch.from_numpy(preds[i]).cuda()], c[i:i + 1], s[i:i + 1],
                                               flipped=None if flipped is None else [flipped[i]])
                         for i in range(n)])
        assert torch.equal(one, pose.decode_keypoints(preds, c, s, flipped=flipped))
    if n == 64:
        # the generator gives joints whose maximum is exactly fl32(0.2) (R = 51)
        assert np.any(maxvals == np.float32(0.2))


def _rescored(kp, box_score, vis_thr=0.2):
    """The rescoring loop of TopDownCocoDatasetCustom.evaluate, under NumPy 2."""
    kpt_score, valid = 0, 0
    for j in range(17):
        t = kp[j][2]
        if t > vis_thr:
            kpt_score = kpt_score + t
            valid = valid + 1
    if valid != 0:
        kpt_score = kpt_score / valid
    return kpt_score * box_score


def _check_construction(kp, areas, box_scores, image_ids, bbox_ids):
    """The comparison is exact only where NumPy's sort and the fp32 OKS threshold are unambiguous: tie-free scores
    per image and every OKS at least 1e-6 from fl32(0.9).  Suppression must happen."""
    pos, table, _ = pose._groups(image_ids, bbox_ids)
    thr, suppressed = np.float32(0.9), 0
    for start, cnt in table:
        idx = pos[start:start + cnt]
        sc = [_rescored(kp[i], box_scores[i]) for i in idx]
        assert len(set(float(v) for v in sc)) == len(sc), "construction: tied scores"
        for a in range(cnt):
            o = mr.oks_iou(kp[idx[a]].flatten(), kp[idx].reshape(cnt, -1), areas[idx[a]], areas[idx],
                           sigmas=np.array(pose.COCO_SIGMAS))
            o = np.delete(o, a)
            assert np.all(np.abs(o.astype(np.float64) - float(thr)) >= 1e-6), "construction: OKS near 0.9"
            suppressed += int(np.sum(o > thr))
    assert suppressed > 0, "construction: nothing is suppressed"


def test_pose_results_match_evaluate(tmp_path):
    preds, flipped, c, s, scores, image_ids, bbox_ids, names = pe.dataset_stream(5)
    ref = _reference(tmp_path, preds, flipped, c, s, scores, bbox_ids, names)
    kp_ref = np.concatenate([r["preds"] for r in ref])
    boxes_ref = np.concatenate([r["boxes"] for r in ref])
    _check_construction(kp_ref, boxes_ref[:, 4], boxes_ref[:, 5], image_ids, bbox_ids)
    assert max(np.bincount(image_ids - image_ids.min())) > 16
    ann = mr.write_image_list(str(tmp_path / "ann.json"), {f"{i:012d}.jpg": int(i) for i in set(image_ids)})
    ds = pe.dataset(ann, str(tmp_path / "crops") + "/")
    mr.quiet(ds.evaluate, ref, res_folder=str(tmp_path))
    with open(tmp_path / "result_keypoints.json") as f:
        want = json.load(f)
    kp = _decode_batches(preds, flipped, c, s)
    got = pose.pose_results(kp, c, s, scores, image_ids, bbox_ids)
    assert len(got) == len(want) and len(got) < len(set(bbox_ids.tolist()))
    for g, w in zip(got, want):
        assert g == w, (g, w)


def test_score_ties_follow_the_reversed_stable_order():
    rng = np.random.default_rng(3)
    n = 14
    base = rng.uniform(0, 150, (17, 2)).astype(np.float32)
    kp = np.zeros((n, 17, 3), np.float32)
    for i in range(n):
        kp[i, :, :2] = base + rng.normal(0, [0.5, 8.0][i % 2], (17, 2)).astype(np.float32)
        kp[i, :, 2] = rng.uniform(0.0, 1.0, 17) if i % 3 else rng.uniform(0.0, 0.2, 17)    # none above 0.2
    box_scores = np.where(np.arange(n) % 4 == 1, 0.0, 0.8)                                    # more zeros, and equal
    c, s = pose.box_center_scale(pe.boxes_for(rng, n))
    bbox_ids = rng.permutation(n) + 40
    image_ids = np.full(n, 9, np.int64)
    got = pose.pose_results(torch.from_numpy(kp).cuda(), c, s, box_scores, image_ids, bbox_ids)
    # the reference flow with oks_nms's sort made stable
    order = np.argsort(bbox_ids, kind="stable")
    db = []
    for i in order:
        db.append({"keypoints": kp[i], "score": _rescored(kp[i], np.float32(box_scores[i])),
                   "area": np.prod(s[i] * 200.0), "i": i})
    assert sum(1 for d in db if d["score"] == 0) >= 3
    keep = mr.oks_nms(db, 0.9, sigmas=np.array(pose.COCO_SIGMAS), kind="stable")
    assert len(got) == len(keep) and 1 < len(keep) < n
    for g, k in zip(got, keep):
        d = db[k]
        assert g["keypoints"] == d["keypoints"].reshape(-1).tolist() and g["score"] == float(d["score"])
        assert g["center"] == c[d["i"]].tolist() and g["image_id"] == 9


def test_run_batch_outputs_feed_decode_directly(tmp_path):
    from oracle import painter_oracle as po
    from _common import build_model
    from painter_b200 import painter_inference as pi
    model, _ = build_model(po.PainterConfig(), 1)
    model.eval()
    rng = np.random.RandomState(12)
    n = 4
    canv = [(rng.randn(896, 448, 3), rng.randn(896, 448, 3)) for _ in range(2 * n)]
    paths = [str(tmp_path / f"p{i}.png") for i in range(2 * n)]
    outs = pi.run_batch([x[0] for x in canv], [x[1] for x in canv], [(192, 256)] * (2 * n), model,
                        torch.device("cuda"), "nearest", out_paths=paths)
    c, s = pose.box_center_scale(pe.boxes_for(np.random.default_rng(0), n))
    ours = pose.decode_keypoints(outs[:n], c, s, flipped=outs[n:])
    files = [np.array(Image.open(p).convert("RGB")) for p in paths]
    theirs = pose.decode_keypoints(files[:n], c, s, flipped=files[n:])
    assert torch.equal(ours, theirs)
    model.__dict__.pop("_pk_graphed", None)


def test_two_runs_are_bit_identical():
    preds, flipped, c, s, scores = _crops(21, 40)
    dev = [torch.from_numpy(a).cuda() for a in preds]
    fdev = [torch.from_numpy(a).cuda() for a in flipped]
    a = pose.decode_keypoints(dev, c, s, flipped=fdev)
    b = pose.decode_keypoints(dev, c, s, flipped=fdev)
    assert torch.equal(a, b)
    ids = np.arange(40) % 3
    r1 = pose.pose_results(a, c, s, scores, ids, np.arange(40))
    r2 = pose.pose_results(b, c, s, scores, ids, np.arange(40))
    assert r1 == r2


def test_non_finite_device_scores_rank_like_numpy():
    """Device keypoints are not validated: inf joint scores with a zero box score rescore to NaN, and a NaN
    coordinate gives NaN OKS.  The order is still total (NaN above every number, later boxes first among equals) and
    a NaN OKS suppresses, as in the reference flow with a stable sort."""
    rng = np.random.default_rng(4)
    n = 12
    base = rng.uniform(0, 150, (17, 2)).astype(np.float32)
    kp = np.zeros((n, 17, 3), np.float32)
    for i in range(n):
        kp[i, :, :2] = base + rng.normal(0, 20.0, (17, 2)).astype(np.float32)
        kp[i, :, 2] = rng.uniform(0.0, 1.0, 17)
    kp[[2, 5, 9], 3, 2] = np.inf                                        # rescored inf, or NaN with a zero box score
    kp[7, 4, 0] = np.nan                                                # NaN OKS against every other box
    box_scores = np.full(n, 0.7)
    box_scores[[5, 9]] = 0.0
    c, s = pose.box_center_scale(pe.boxes_for(rng, n))
    bbox_ids = np.arange(n) + 10
    got = pose.pose_results(torch.from_numpy(kp).cuda(), c, s, box_scores, np.zeros(n, np.int64), bbox_ids)
    with np.errstate(all="ignore"):
        db = [{"keypoints": kp[i], "score": _rescored(kp[i], np.float32(box_scores[i])),
               "area": np.prod(s[i] * 200.0), "i": i} for i in range(n)]
        assert sum(np.isnan(d["score"]) for d in db) == 2
        keep = mr.oks_nms(db, 0.9, sigmas=np.array(pose.COCO_SIGMAS), kind="stable")
    assert len(got) == len(keep) >= 2
    for g, k in zip(got, keep):
        d = db[k]
        assert np.array(g["keypoints"], np.float32).tobytes() == d["keypoints"].tobytes()
        assert g["score"] == float(d["score"]) or (np.isnan(g["score"]) and np.isnan(d["score"]))
