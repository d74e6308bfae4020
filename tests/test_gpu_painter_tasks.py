"""GPU parity of the Painter task-inference mirrors (painter_b200.painter_inference) against the UNMODIFIED
`run_one_image` of every remaining Painter eval script: COCO panoptic semseg / instance, COCO pose, NYUv2 depth and the
SIDD / LoL / derain restoration scripts.

Protocol (as test_gpu_inference.py): both sides drive the SAME painter_b200 module at the full 896 x 448 geometry with
seeded random weights, the reference under torch.no_grad(), so the forward is identical and every difference is in
the wrapper.  The device kernels for de-normalisation, bilinear / nearest / bicubic resize, channel mean and integer
conversion must reproduce the reference's float64 torch-CPU arithmetic bit for bit: the PNG files decode to the same
arrays (and the depth PNG has the same mode), the restoration arrays are equal float64 arrays."""
import numpy as np
import pytest
import torch

from oracle import painter_oracle as po

from _common import build_model
from _painter_eval import painter_eval
from _refmods import have_reference

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_reference(), reason="reference tree not staged")]

# reference script (_painter_eval.EVAL_SCRIPTS key) -> (mirror, the script reads model.module.*)
TASKS = {
    "pano_semseg": ("run_one_image", True),
    "pano_inst": ("run_one_image_nearest", True),
    "pose": ("run_one_image_nearest", True),
    "depth": ("run_one_image_depth", False),
    "sidd": ("run_one_image_restore", False),
    "lol": ("run_one_image_restore", False),
    "derain": ("run_one_image_restore", False),
}
# (width, height) of the source image: identity, SIDD, LoL, NYUv2, 640 x 427, odd ratios, exact 2x upscale, and a
# size under 16 px on a side (bicubic taps clamped at both borders)
SIZES = [(448, 448), (256, 256), (600, 400), (640, 480), (640, 427), (301, 523), (896, 896), (13, 9)]


class Wrapped(torch.nn.Module):      # the pano / pose scripts call model(...) and model.module.* (a DDP wrapper)
    def __init__(self, m):
        super().__init__()
        self.module = m

    def forward(self, *a, **k):
        return self.module(*a, **k)


@pytest.fixture(scope="module")
def painter():
    model, _ = build_model(po.PainterConfig(), 1)
    model.eval()
    return model


def _inputs(seed):
    rng = np.random.RandomState(seed)
    return rng.randn(896, 448, 3), rng.randn(896, 448, 3)


def _run_both(task, model, size, tmp_path, seed):
    """(reference result, mirror result): PIL images read back from the two PNGs, or the two returned arrays."""
    from PIL import Image
    from painter_b200 import painter_inference as ours
    ref = painter_eval(task)
    name, wrapped = TASKS[task]
    m = Wrapped(model) if wrapped else model
    dev = torch.device("cuda")
    img, tgt = _inputs(seed)
    o_ref, o_our = str(tmp_path / f"ref_{task}.png"), str(tmp_path / f"our_{task}.png")
    with torch.no_grad():
        a = ref.run_one_image(img, tgt, size, m, o_ref, dev)
    b = getattr(ours, name)(img, tgt, size, m, o_our, dev)
    if name == "run_one_image_restore":
        return a, b
    return Image.open(o_ref), Image.open(o_our)


def _assert_same(task, size, a, b):
    w, h = size
    if TASKS[task][0] == "run_one_image_restore":
        assert isinstance(b, np.ndarray) and a.dtype == b.dtype == np.float64
        assert a.shape == b.shape == (h, w, 3)
        assert np.array_equal(a, b), (task, size, np.abs(a - b).max())
        return
    if task == "depth":
        assert a.mode == b.mode, (a.mode, b.mode)
    x, y = np.array(a), np.array(b)
    assert x.dtype == y.dtype and x.shape == y.shape == ((h, w) if task == "depth" else (h, w, 3))
    assert np.array_equal(x, y), (task, size, np.abs(x.astype(np.int64) - y.astype(np.int64)).max(),
                                  int((x != y).sum()))


@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
@pytest.mark.parametrize("task", list(TASKS))
def test_mirror_matches_reference_script(painter, task, size, tmp_path):
    a, b = _run_both(task, painter, size, tmp_path, seed=10 * list(TASKS).index(task) + SIZES.index(size))
    _assert_same(task, size, a, b)


@pytest.mark.parametrize("task", ["depth", "sidd"])
def test_auto_precision_runs_the_fp32_accurate_forward_without_autograd_state(painter, task, tmp_path):
    """precision = "auto": the mirror equals the reference function called under no_grad (the fp32-accurate
    forward), not the bf16 arithmetic the eval script itself would select, and leaves no gradient arena or .grad."""
    assert painter.__dict__.get("_pk_arena") is None
    painter.precision = "auto"
    try:
        size = (640, 480)
        a, b = _run_both(task, painter, size, tmp_path, seed=7)
        _assert_same(task, size, a, b)
    finally:
        painter.precision = "bf16"
    assert painter.__dict__.get("_pk_arena") is None
    assert all(p.grad is None for p in painter.parameters())
