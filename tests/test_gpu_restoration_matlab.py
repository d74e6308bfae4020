"""GPU checks of the derain and SIDD scores (painter_b200.task_metrics derain_scores, sidd_scores, ycbcr_y) against the
CPU restatement of the MATLAB scripts in oracle/matlab_ref.py:

- ycbcr_y equals the restatement on every one of the 2^24 colours (the 194 exact ties among them);
- derain_scores equals it on a ragged batch (PSNR to 1e-13 relative, +Inf for an identical pair; SSIM to 1e-12), and
  end to end from run_batch(task="restore") outputs against the PNG files written and read back as
  painter_inference_derain.py writes them;
- sidd_scores equals it to 1e-12 on 256 x 256 blocks and odd sizes down to 1 x 1;
- host and device inputs, and two runs, give bit-identical results."""
import numpy as np
import pytest
import torch

from oracle import matlab_ref as mr
from oracle import painter_oracle as po

from _common import build_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def painter():
    model, _ = build_model(po.PainterConfig(), 1)
    model.eval()
    yield model
    model.__dict__.pop("_pk_graphed", None)
    torch.cuda.empty_cache()


def test_ycbcr_y_on_every_colour():
    from painter_b200.task_metrics import ycbcr_y
    chunk = 1 << 20
    for c0 in range(0, 1 << 24, chunk):
        idx = torch.arange(c0, c0 + chunk, device="cuda", dtype=torch.int32)
        rgb = torch.stack([(idx >> 16) & 255, (idx >> 8) & 255, idx & 255], -1).to(torch.uint8).view(1024, 1024, 3)
        ours = ycbcr_y(rgb).cpu().numpy()
        want = mr.rgb2ycbcr_y(rgb.cpu().numpy())
        bad = np.flatnonzero(ours != want)
        assert bad.size == 0, (c0, bad[:5], ours.reshape(-1)[bad[:5]], want.reshape(-1)[bad[:5]])


def _check(ours_psnr, ours_ssim, want, ssim_tol):
    for i, (wp, ws) in enumerate(want):
        if np.isinf(wp):
            assert np.isinf(ours_psnr[i]) and ours_psnr[i] > 0, (i, ours_psnr[i])
        else:
            assert abs(ours_psnr[i] - wp) <= 1e-13 * abs(wp), (i, ours_psnr[i], wp)
        assert abs(ours_ssim[i] - ws) <= ssim_tol, (i, ours_ssim[i], ws)


def _bit_identical(fn, restored, gts, psnr, ssim):
    for inputs in (restored, [torch.from_numpy(r).cuda() for r in restored]):
        p2, s2 = fn(inputs, gts)
        np.testing.assert_array_equal(p2, psnr)
        np.testing.assert_array_equal(s2, ssim)


def test_derain_scores_match_the_restatement():
    from painter_b200.task_metrics import derain_scores
    rng = np.random.RandomState(11)
    sizes = [(11, 11), (12, 40), (321, 481), (481, 321), (1024, 777), (37, 53)]
    gts = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in sizes]
    restored = [g / 255. + rng.randn(*g.shape) * 0.08 for g in gts]       # values below 0 and above 1: clipped
    restored.append((gts[3] + 0.5) / 255.)                               # writes exactly gts[3]: PSNR = +Inf
    gts.append(gts[3])
    psnr, ssim = derain_scores(restored, gts)
    want = [mr.derain_scores(r, g) for r, g in zip(restored, gts)]
    _check(psnr, ssim, want, 1e-12)
    assert np.isinf(psnr[-1]) and psnr[-1] > 0 and ssim[-1] == pytest.approx(1.0, abs=1e-12)
    print("derain psnr", psnr, "ssim", ssim)
    _bit_identical(derain_scores, restored, gts, psnr, ssim)


def test_sidd_scores_match_the_restatement():
    from painter_b200.task_metrics import sidd_scores
    rng = np.random.RandomState(12)
    sizes = [(256, 256)] * 3 + [(1, 1), (5, 300), (37, 23), (17, 250), (300, 5)]
    gts = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in sizes]
    restored = [g / 255. + rng.randn(*g.shape) * 0.03 for g in gts]
    restored.append(gts[0].astype(np.float32) / np.float32(255))         # x == y after the float32 rounding
    gts.append(gts[0])
    restored = [np.asarray(r, dtype=np.float64) for r in restored]
    psnr, ssim = sidd_scores(restored, gts)
    want = [mr.sidd_scores(r, g) for r, g in zip(restored, gts)]
    _check(psnr, ssim, want, 1e-12)
    assert np.isinf(psnr[-1]) and ssim[-1] == pytest.approx(1.0, abs=1e-12)
    print("sidd psnr", psnr, "ssim", ssim)
    _bit_identical(sidd_scores, restored, gts, psnr, ssim)


def test_derain_png_round_trip_from_run_batch(painter, tmp_path):
    from PIL import Image
    from painter_b200 import painter_inference as pi
    from painter_b200.task_metrics import derain_scores, sidd_scores
    rng = np.random.RandomState(13)
    sizes = [(481, 321), (321, 481), (40, 12), (777, 1024)]                # (width, height), as run_batch takes them
    canv = [(rng.randn(896, 448, 3), rng.randn(896, 448, 3)) for _ in sizes]
    outs = pi.run_batch([c[0] for c in canv], [c[1] for c in canv], sizes, painter, torch.device("cuda"), "restore")
    gts = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for w, h in sizes]
    psnr, ssim = derain_scores(outs, gts)
    want = []
    for i, (o, g) in enumerate(zip(outs, gts)):
        # painter_inference_derain.py: rgb_restored = clip(output, 0, 1); Image.fromarray((rgb_restored * 255)
        # .astype(np.uint8)).save(...)
        path = str(tmp_path / f"{i}.png")
        Image.fromarray((np.clip(o, 0, 1) * 255).astype(np.uint8)).save(path)
        want.append(mr.derain_scores_u8(np.array(Image.open(path)), g))
    _check(psnr, ssim, want, 1e-12)
    _bit_identical(derain_scores, outs, gts, psnr, ssim)
    # SIDD from the same outputs: the float32 array the script saves
    sp, ss = sidd_scores(outs, gts)
    _check(sp, ss, [mr.sidd_scores(o, g) for o, g in zip(outs, gts)], 1e-12)
    _bit_identical(sidd_scores, outs, gts, sp, ss)
