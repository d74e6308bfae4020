"""GPU parity of painter_b200.task_metrics against the UNMODIFIED reference evaluators (tests/_task_eval.py):

- palette_classes equals SemSegEvaluatorCustom.post_process_segm_output on every one of the 2^24 RGB colours, for the
  ADE20K and COCO palettes and the three distances (every tie between palette colours is among them);
- SemSegMeter's confusion matrix equals the evaluator's np.bincount on a ragged batch over several updates, and end to
  end from run_batch's device outputs against the PNG files the same call writes;
- DepthMeter equals eval_with_pngs.eval() (d1, d2, d3 bit for bit in float32, the rest to 1e-5 relative);
- restoration_scores equals a numpy + scipy restatement of skimage 0.19's PSNR / SSIM (1e-12);
- every result is bit-identical from run to run."""
import numpy as np
import pytest
import torch

from oracle import painter_oracle as po

from _common import build_model
from _refmods import have_reference

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not have_reference(), reason="reference tree not staged")

DISTS = ["abs", "square", "mean"]


def _palettes():
    import _task_eval
    return {"ade20k": _task_eval.ade20k_palette(), "coco": _task_eval.coco_palette()}


@pytest.fixture(scope="module")
def painter():
    model, _ = build_model(po.PainterConfig(), 1)
    model.eval()
    yield model
    model.__dict__.pop("_pk_graphed", None)
    torch.cuda.empty_cache()


@needs_ref
@pytest.mark.parametrize("kind", ["ade20k", "coco"])
@pytest.mark.parametrize("dist", DISTS)
def test_palette_classes_on_every_colour(kind, dist):
    import _task_eval
    from painter_b200.task_metrics import palette_classes
    palette = _palettes()[kind]
    assert len(palette) == {"ade20k": 150, "coco": 133}[kind]
    ref = _task_eval.semseg_decoder(kind, palette, dist)
    chunk = 1 << 20
    for c0 in range(0, 1 << 24, chunk):
        idx = torch.arange(c0, c0 + chunk, device="cuda", dtype=torch.int32)
        rgb = torch.stack([(idx >> 16) & 255, (idx >> 8) & 255, idx & 255], -1).to(torch.uint8).view(1024, 1024, 3)
        ours = palette_classes(rgb, palette, dist).cpu().numpy()
        want = ref(rgb.cpu().numpy())
        assert ours.shape == want.shape
        bad = np.flatnonzero(ours.astype(np.int64) != want)
        assert bad.size == 0, (kind, dist, c0, bad[:5], ours.reshape(-1)[bad[:5]], want.reshape(-1)[bad[:5]])


def _semseg_batch(rng, palette, sizes, K, ignore=255):
    """Predictions near palette colours (small jitter, so classes are hit) and label maps with the ignore label;
    the first image's first K labels are 0 .. K-1."""
    pal = np.asarray(palette, dtype=np.int64)
    preds, gts = [], []
    for i, (h, w) in enumerate(sizes):
        cls = rng.randint(0, K, size=(h, w))
        img = pal[cls] + rng.randint(-40, 41, size=(h, w, 3))
        preds.append(np.clip(img, 0, 255).astype(np.uint8))
        g = rng.randint(0, K, size=(h, w))
        g[rng.rand(h, w) < 0.1] = ignore
        if i == 0:
            g.reshape(-1)[:K] = np.arange(K)
        gts.append(g.astype(np.uint8))
    return preds, gts


def _ref_conf(decode, preds, gts, K, ignore=255):
    conf = np.zeros((K + 1) ** 2, dtype=np.int64)
    for p, g in zip(preds, gts):
        pred = decode(p).astype(np.int64)
        gt = g.astype(np.int64)
        gt[gt == ignore] = K
        conf += np.bincount((K + 1) * pred.reshape(-1) + gt.reshape(-1), minlength=conf.size)
    return conf.reshape(K + 1, K + 1)


@needs_ref
@pytest.mark.parametrize("kind,dist", [("ade20k", "abs"), ("coco", "square"), ("ade20k", "mean")])
def test_semseg_confusion_matches_bincount(kind, dist):
    import _task_eval
    from painter_b200.task_metrics import SemSegMeter
    palette = _palettes()[kind]
    K = len(palette)
    decode = _task_eval.semseg_decoder(kind, palette, dist)
    rng = np.random.RandomState(0)
    batches = [_semseg_batch(rng, palette, [(512, 683), (37, 53), (1, 1), (683, 512)], K),
               _semseg_batch(rng, palette, [(100, 33), (256, 256)], K),
               _semseg_batch(rng, palette, [(7, 900)], K)]
    results = []
    for _ in range(2):
        meter = SemSegMeter(palette, dist_type=dist)
        for j, (preds, gts) in enumerate(batches):
            # device predictions (as run_batch returns them) in the first update, host arrays after
            meter.update([torch.from_numpy(p).cuda() for p in preds] if j == 0 else preds, gts)
        results.append(meter.conf_matrix)
    want = _ref_conf(decode, [p for b in batches for p in b[0]], [g for b in batches for g in b[1]], K)
    assert (want[:-1, :-1].sum(0) > 0).all()          # every class is in the ground truth
    np.testing.assert_array_equal(results[0], want)
    np.testing.assert_array_equal(results[1], want)
    r0 = SemSegMeter(palette, dist_type=dist)
    r0.update(*batches[0])
    r0.reset()
    assert r0.conf_matrix.sum() == 0


@needs_ref
def test_semseg_end_to_end_from_run_batch(painter, tmp_path):
    import _task_eval
    from PIL import Image
    from painter_b200 import painter_inference as pi
    from painter_b200.task_metrics import SemSegMeter
    palette = _task_eval.ade20k_palette()
    K = len(palette)
    decode = _task_eval.semseg_decoder("ade20k", palette, "abs")
    rng = np.random.RandomState(3)
    sizes = [(683, 512), (512, 683), (301, 523), (64, 48)]
    canv = [(rng.randn(896, 448, 3), rng.randn(896, 448, 3)) for _ in sizes]
    paths = [str(tmp_path / f"p{i}.png") for i in range(len(sizes))]
    gts = []
    for w, h in sizes:
        g = rng.randint(0, K, size=(h, w)).astype(np.uint8)
        g[rng.rand(h, w) < 0.05] = 255
        gts.append(g)
    outs = pi.run_batch([c[0] for c in canv], [c[1] for c in canv], sizes, painter, torch.device("cuda"), "segm",
                        out_paths=paths)
    meter = SemSegMeter(palette)
    meter.update(outs, gts)
    want = _ref_conf(decode, [np.array(Image.open(p)) for p in paths], gts, K)
    np.testing.assert_array_equal(meter.conf_matrix, want)
    from painter_b200.task_metrics import semseg_scores
    ours, ref = meter.evaluate(), semseg_scores(want)
    for k in ("mIoU", "fwIoU", "mACC", "pACC"):
        assert ours[k] == ref[k], k
    np.testing.assert_array_equal(ours["IoU"], ref["IoU"])


def _depth_maps(rng, n, H=480, W=640):
    preds, gts = [], []
    for _ in range(n):
        p = rng.randint(0, 12001, size=(H, W)).astype(np.int32)       # 0 and < 1 (below min_depth), > 10000
        p[rng.rand(H, W) < 0.05] = 0
        g = rng.randint(0, 12001, size=(H, W)).astype(np.uint16)      # 0 and > max_depth: invalid
        g[rng.rand(H, W) < 0.1] = 0
        g[:8, :8] = 65535
        preds.append(p)
        gts.append(g)
    return preds, gts


@needs_ref
@pytest.mark.parametrize("eigen_crop", [True, False])
def test_depth_matches_eval_with_pngs(eigen_crop):
    import _task_eval
    from painter_b200.task_metrics import DepthMeter
    ref = _task_eval.depth_eval(eigen_crop=eigen_crop)
    rng = np.random.RandomState(1 + eigen_crop)
    preds, gts = _depth_maps(rng, 5)
    ref.gt_depths = [g.astype(np.float32) / 1000.0 for g in gts]
    ref.missing_ids = set()
    silog, log10, abs_rel, sq_rel, rms, log_rms, d1, d2, d3 = ref.eval([p.astype(np.float32) / 1000.0 for p in preds])
    runs = []
    for _ in range(2):
        m = DepthMeter(eigen_crop=eigen_crop)
        m.update([torch.from_numpy(p).cuda() for p in preds[:3]], gts[:3])
        m.update(preds[3:], gts[3:])
        runs.append(m.per_image())
    ours = runs[0]
    assert ours.shape == (5, 9)
    np.testing.assert_array_equal(runs[0], runs[1])
    for j, r in enumerate((d1, d2, d3)):
        np.testing.assert_array_equal(ours[:, j].astype(np.float32), r)
    for j, r in zip(range(3, 9), (abs_rel, sq_rel, rms, log_rms, silog, log10)):
        np.testing.assert_allclose(ours[:, j], r, rtol=1e-5, atol=0)
    ev = m.evaluate()
    assert list(ev) == ["d1", "d2", "d3", "AbsRel", "SqRel", "RMSE", "RMSElog", "SILog", "log10"]
    assert ev["RMSE"] == ours[:, 5].mean()


def _ref_restoration(restored, gt):
    """skimage 0.19 peak_signal_noise_ratio / structural_similarity(multichannel=True) as painter_inference_lol.py
    calls them, restated with numpy and scipy.ndimage.uniform_filter."""
    from scipy.ndimage import uniform_filter
    x, y = np.clip(restored, 0, 1), gt / 255.
    with np.errstate(divide="ignore"):
        psnr = 10 * np.log10(1.0 / np.mean((x - y) ** 2, dtype=np.float64))
    c1, c2, cov_norm = (0.01 * 2.0) ** 2, (0.03 * 2.0) ** 2, 49 / 48
    ssims = []
    for ch in range(3):
        X, Y = x[..., ch], y[..., ch]
        ux, uy = uniform_filter(X, size=7), uniform_filter(Y, size=7)
        uxx, uyy, uxy = uniform_filter(X * X, size=7), uniform_filter(Y * Y, size=7), uniform_filter(X * Y, size=7)
        vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
        S = ((2 * ux * uy + c1) * (2 * vxy + c2)) / ((ux ** 2 + uy ** 2 + c1) * (vx + vy + c2))
        ssims.append(S[3:-3, 3:-3].mean())
    return psnr, np.mean(ssims)


def _check_restoration(restored, gts, psnr, ssim):
    for i, (r, g) in enumerate(zip(restored, gts)):
        rp, rs = _ref_restoration(r, g)
        if np.isinf(rp):
            assert np.isinf(psnr[i]) and psnr[i] > 0, i
        else:
            assert abs(psnr[i] - rp) <= 1e-12 * abs(rp), (i, psnr[i], rp)
        assert abs(ssim[i] - rs) <= 1e-12, (i, ssim[i], rs)


def test_restoration_scores_match_the_restatement():
    from painter_b200.task_metrics import restoration_scores
    rng = np.random.RandomState(5)
    sizes = [(7, 7), (9, 13), (64, 48), (400, 600), (31, 700)]
    gts = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in sizes]
    restored = [g / 255. + rng.randn(*g.shape) * 0.1 for g in gts]      # values below 0 and above 1: clipped
    restored.append(gts[2] / 255.)                                     # identical: PSNR = inf
    gts.append(gts[2])
    psnr, ssim = restoration_scores(restored, gts)
    _check_restoration(restored, gts, psnr, ssim)
    assert np.isinf(psnr[-1]) and psnr[-1] > 0
    assert ssim[-1] == pytest.approx(1.0, abs=1e-12)
    p2, s2 = restoration_scores([torch.from_numpy(r).cuda() for r in restored], gts)
    np.testing.assert_array_equal(psnr, p2)
    np.testing.assert_array_equal(ssim, s2)


def test_restoration_scores_of_run_batch_outputs(painter):
    from painter_b200 import painter_inference as pi
    from painter_b200.task_metrics import restoration_scores
    rng = np.random.RandomState(7)
    sizes = [(600, 400), (64, 48), (13, 9)]
    canv = [(rng.randn(896, 448, 3), rng.randn(896, 448, 3)) for _ in sizes]
    outs = pi.run_batch([c[0] for c in canv], [c[1] for c in canv], sizes, painter, torch.device("cuda"), "restore")
    gts = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for w, h in sizes]
    psnr, ssim = restoration_scores(outs, gts)
    _check_restoration(outs, gts, psnr, ssim)
    p2, s2 = restoration_scores(outs, gts)
    np.testing.assert_array_equal(psnr, p2)
    np.testing.assert_array_equal(ssim, s2)
