"""COCO panoptic post-processing on the GPU (painter_b200.panoptic) against the unmodified reference evaluators
(tests/_panoptic_eval.py) on seeded synthetic painted images."""
import numpy as np
import pytest
import torch
from PIL import Image

import _panoptic_eval as pe
import _task_eval
from oracle import ref_loader
from painter_b200 import panoptic as pn

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_loader.available(), reason="reference checkout / staged copy not found")]

SIZES = [(480, 640), (427, 640), (640, 480)]


def _images(seed, blobs=4, jitter=8):
    rng = np.random.default_rng(seed)
    pal = pn.instance_palette().astype(np.int32)
    return [pe.instance_image(rng, h, w, pal, blobs=blobs, jitter=jitter) for h, w in SIZES]


def _write(tmp_path, imgs, tag):
    paths = []
    for i, a in enumerate(imgs):
        p = tmp_path / f"{tag}{i}.png"
        Image.fromarray(a).save(p)
        paths.append(str(p))
    return paths


def _groups(masks, scores):
    """{mask bytes: sorted scores} of a set of instances."""
    out = {}
    m = masks.bool().cpu().numpy()
    for k in range(m.shape[0]):
        out.setdefault(np.packbits(m[k]).tobytes(), []).append(float(scores[k]))
    return {k: sorted(v) for k, v in out.items()}


def _same_instances(ours, ref_inst, rel=1e-5):
    g_ours = _groups(ours.masks, ours.scores.cpu().numpy())
    g_ref = _groups(ref_inst.pred_masks, ref_inst.scores.float().cpu().numpy())
    assert g_ours.keys() == g_ref.keys()
    for k in g_ref:
        np.testing.assert_allclose(g_ours[k], g_ref[k], rtol=rel, atol=2.4e-7)   # 1 - m / max: ulps of 1.0


@pytest.mark.parametrize("dist_thr,keep_all", [(19.0, False), (19.0, True), (16.0, False), ([16.0, 19.0], False),
                                               ([16.0, 19.0], True)])
def test_decode_matches_threshold_postprocess(tmp_path, dist_thr, keep_all):
    imgs = _images(1)
    paths = _write(tmp_path, imgs, "inst")
    ev = pe.inst_evaluator(dist_thr=dist_thr)
    ours = pn.decode_instances([torch.from_numpy(a).cuda() for a in imgs], dist_thr=dist_thr, keep_all=keep_all)
    for o, p, a in zip(ours, paths, imgs):
        ref = ev.post_process_segm_output_by_threshold(p, dist_thr_list=ev.dist_thr_list, keep_all=keep_all)
        r = ref["instances"]
        assert o.image_size == a.shape[:2] and len(o) == len(r.scores)
        _same_instances(o, r)
        assert torch.equal(o.classes.cpu(), r.pred_classes.to(torch.int64).cpu())


def test_decode_empty_prediction(tmp_path):
    imgs = [np.full((h, w, 3), 128, dtype=np.uint8) for h, w in SIZES[:2]]   # 128 is no location colour's channel
    paths = _write(tmp_path, imgs, "empty")
    ev = pe.inst_evaluator(dist_thr=0.2)
    ours = pn.decode_instances(imgs, dist_thr=0.2)
    for o, p in zip(ours, paths):
        r = ev.post_process_segm_output_by_threshold(p, dist_thr_list=[0.2])["instances"]
        assert len(o) == 1 and len(r.scores) == 1
        assert not o.masks.any() and float(o.scores[0]) == 0.0 and int(o.classes[0]) == 0
        assert float(r.scores[0]) == 0.0 and not r.pred_masks.any()


def test_decode_minmax(tmp_path):
    imgs = _images(2, blobs=6, jitter=3)
    paths = _write(tmp_path, imgs, "mm")
    ev = pe.inst_evaluator(post_type="minmax")
    ours = pn.decode_instances([torch.from_numpy(a).cuda() for a in imgs], post_type="minmax")
    for o, p in zip(ours, paths):
        r = ev.post_process_segm_output_by_minmax(p)[0]["instances"]
        assert torch.equal(o.masks.cpu(), r.pred_masks.bool().cpu())
        np.testing.assert_allclose(o.scores.cpu().numpy(), r.scores.cpu().numpy(), rtol=1e-5, atol=2.4e-7)
        assert torch.equal(o.classes.cpu(), r.pred_classes.to(torch.int64).cpu())


@pytest.mark.parametrize("class_aware", [False, True])
def test_matrix_nms_on_explicit_masks(class_aware):
    g = torch.Generator().manual_seed(3)
    n, h, w = 2100, 48, 64
    # random rectangles: overlaps of every size
    masks = torch.zeros(n, h, w, dtype=torch.bool)
    y0 = torch.randint(0, h - 4, (n,), generator=g)
    x0 = torch.randint(0, w - 4, (n,), generator=g)
    hh = torch.randint(2, 24, (n,), generator=g)
    ww = torch.randint(2, 24, (n,), generator=g)
    for k in range(n):
        masks[k, y0[k]:y0[k] + hh[k], x0[k]:x0[k] + ww[k]] = True
    scores = (torch.randperm(n, generator=g).float() + 1) / (n + 1)          # distinct, separated by 1 / (n + 1)
    labels = torch.randint(0, 5, (n,), generator=g) if class_aware else torch.ones(n, dtype=torch.int64)
    md, sd, ld = masks.cuda(), scores.cuda(), labels.cuda()
    rs, rl, rm, rk = pe.mask_matrix_nms()(md, ld, sd, filter_thr=-1, nms_pre=-1, max_num=100, kernel="gaussian",
                                          sigma=2.0, mask_area=None)
    os_, ok = pn.matrix_nms(md, ld if class_aware else None, sd)
    ref_s = rs.cpu().numpy()
    np.testing.assert_allclose(os_.cpu().numpy(), ref_s, rtol=1e-5)
    # the kept indices agree wherever the reference's decayed scores are separated from their neighbours
    gap = np.diff(ref_s.astype(np.float64))
    sep = np.ones(len(ref_s), dtype=bool)
    close = np.abs(gap) <= 1e-4 * np.abs(ref_s[1:])
    sep[1:] &= ~close
    sep[:-1] &= ~close
    assert sep.sum() > len(ref_s) // 2, "too few separated scores: the construction does not test the order"
    np.testing.assert_array_equal(ok.cpu().numpy()[sep], rk.cpu().numpy()[sep])


def _coco_palette():
    return np.asarray(_task_eval.coco_palette(), dtype=np.uint8)


def _sem_images(seed):
    rng = np.random.default_rng(seed)
    pal = _coco_palette().astype(np.int32)
    return [pe.semantic_image(rng, h, w, pal) for h, w in SIZES]


@pytest.mark.parametrize("with_nms", [False, True])
def test_classify_matches_merge_inst_semseg(tmp_path, with_nms):
    imgs, sems = _images(4), _sem_images(5)
    ipaths, spaths = _write(tmp_path, imgs, "inst"), _write(tmp_path, sems, "sem")
    pal = _coco_palette()
    ev_inst = pe.inst_evaluator(dist_thr=19.0)
    ev = pe.instance_evaluator(ev_inst, pe.semseg_evaluator(pal.tolist()), with_nms)
    dec = pn.decode_instances([torch.from_numpy(a).cuda() for a in imgs], dist_thr=19.0, keep_all=with_nms)
    ours = pn.classify_instances(dec, [torch.from_numpy(a).cuda() for a in sems], pal, with_nms=with_nms)
    for o, ip, sp in zip(ours, ipaths, spaths):
        r = ev.merge_inst_semseg_result({"inst_file": ip, "semseg_file": sp})
        _same_instances(o, r)
        got = {np.packbits(m).tobytes(): int(c) for m, c in zip(o.masks.cpu().numpy(), o.classes.cpu().numpy())}
        want = {np.packbits(m).tobytes(): int(c) for m, c in zip(r.pred_masks.bool().cpu().numpy(),
                                                                r.pred_classes.cpu().numpy())}
        assert got == want


def test_panoptic_merge_matches_combine():
    sems = _sem_images(6)
    pal = _coco_palette()
    sem_ev = pe.semseg_evaluator(pal.tolist())
    rng = np.random.default_rng(7)
    insts, refs = [], []
    for (h, w), s in zip(SIZES, sems):
        n = 40
        masks = torch.zeros(n, h, w, dtype=torch.bool)
        for k in range(n):
            y0, x0 = rng.integers(0, h - 10), rng.integers(0, w - 10)
            masks[k, y0:y0 + rng.integers(5, h // 3), x0:x0 + rng.integers(5, w // 3)] = True
        scores = torch.from_numpy(rng.permutation(n).astype(np.float32) / n * 0.9 + 0.1)
        classes = torch.from_numpy(rng.integers(0, 80, n)).to(torch.int64)
        insts.append(pn.Instances((h, w), masks.cuda(), scores.cuda(), classes.cuda()))
        ri = pe.Instances((h, w))
        ri.pred_masks, ri.scores, ri.pred_classes = masks.float().cuda(), scores.cuda(), classes.cuda()
        refs.append(ri)
    ours = pn.panoptic_merge(insts, [torch.from_numpy(s).cuda() for s in sems], pal, overlap_threshold=0.5,
                             stuff_area_thresh=4096, instances_score_thresh=0.3)
    for (pmap, info), ri, s in zip(ours, refs, sems):
        sem_map, _ = sem_ev.post_process_segm_output(s)
        rmap, rinfo = pe.pano_eval().combine_semantic_and_instance_outputs_custom(
            ri, torch.from_numpy(sem_map).cuda(), 0.5, 4096, 0.3)
        assert torch.equal(pmap.cpu(), rmap.cpu())
        assert info == rinfo


def test_end_to_end_device_outputs_equal_png_files(tmp_path):
    from oracle import painter_oracle as po
    from _common import build_model
    from painter_b200 import painter_inference as pi
    model, _ = build_model(po.PainterConfig(), 1)
    model.eval()
    rng = np.random.RandomState(11)
    sizes = [(640, 480), (640, 427), (301, 523)]
    canv = [(rng.randn(896, 448, 3), rng.randn(896, 448, 3)) for _ in sizes]
    paths = [str(tmp_path / f"n{i}.png") for i in range(len(sizes))]
    outs = pi.run_batch([c[0] for c in canv], [c[1] for c in canv], sizes, model, torch.device("cuda"), "nearest",
                        out_paths=paths)
    ours = pn.decode_instances(outs, dist_thr=19.0)
    theirs = pn.decode_instances([np.array(Image.open(p).convert("RGB")) for p in paths], dist_thr=19.0)
    for a, b in zip(ours, theirs):
        assert torch.equal(a.masks, b.masks) and torch.equal(a.scores, b.scores)
    model.__dict__.pop("_pk_graphed", None)


def test_two_runs_are_bit_identical():
    imgs = [torch.from_numpy(a).cuda() for a in _images(8)]
    a = pn.decode_instances(imgs, dist_thr=[16.0, 19.0])
    b = pn.decode_instances(imgs, dist_thr=[16.0, 19.0])
    for x, y in zip(a, b):
        assert torch.equal(x.masks, y.masks) and torch.equal(x.scores, y.scores) and torch.equal(x.classes, y.classes)
