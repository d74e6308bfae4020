"""GPU-side mirror of the Painter task-inference `run_one_image` functions (SURVEY §8 f.2): same arguments, same file
on disk (or the same returned array), with the nhwc->nchw conversion, the forward (CUDA-graph replay), unpatchify +
bottom half + de-normalisation and the resize to the source size on the GPU; only the finished image crosses back to
the host.

    run_one_image          Painter/eval/ade20k_semantic/painter_inference_segm.py:67-93,
                           coco_panoptic/painter_inference_pano_semseg.py          clip(x*255), bilinear, uint8 PNG
    run_one_image_nearest  coco_panoptic/painter_inference_pano_inst.py,
                           mmpose_custom/painter_inference_pose.py                 clip(x*255), nearest, uint8 PNG
    run_one_image_depth    nyuv2_depth/painter_inference_depth.py                  clip(x*10000), bilinear, channel
                                                                                   mean, int32 PNG
    run_one_image_restore  sidd/painter_inference_sidd.py, lol/painter_inference_lol.py,
                           derain/painter_inference_derain.py                      x, bicubic, returns float64 array

The eval scripts call the model without torch.no_grad(), so a module in precision "auto" runs its bf16 training
arithmetic there; these mirrors run under no_grad, which selects the fp32-accurate forward (and keeps no autograd
state), as the ADE20k mirror always has.

Each mirror is run_batch of its one image at forward batch 1: what run_batch returns or writes for an image is what
the mirror returns or writes for it alone.  Canvases other than float32 / float64 are refused with a ValueError.
"""
import ctypes

import numpy as np
import torch

from . import seggpt_engine as _se
from ._lib import check, lib
from .seggpt_engine import _graphed, _stream

# pk_denorm_bottom_batched finish codes
CLIP255, CLIP10000, PLAIN = 0, 1, 2


@torch.no_grad()
def run_one_image(img, tgt, size, model, out_path, device):
    """ADE20k semantic / COCO panoptic semseg.  img, tgt: numpy [2*S, S, 3] ImageNet-normalised canvases; size =
    (width, height) of the source image; model: the painter_b200 Painter module or a DistributedDataParallel wrapper
    of it (the script passes `model.module` users).  Writes the uint8 PNG to out_path and returns it on the device."""
    return _run([img], [tgt], [size], model, device, "segm", [out_path], pad=False)[0]


@torch.no_grad()
def run_one_image_nearest(img, tgt, size, model, out_path, device):
    """COCO panoptic instance / COCO pose: as run_one_image, with a nearest resize.  Writes the uint8 PNG."""
    return _run([img], [tgt], [size], model, device, "nearest", [out_path], pad=False)[0]


@torch.no_grad()
def run_one_image_depth(img, tgt, size, model, out_path, device):
    """NYUv2 depth: clip(x * 10000, 0, 10000), bilinear, mean over the channels, int32.  Writes the int32 PNG (depth
    in units of 1e-4)."""
    return _run([img], [tgt], [size], model, device, "depth", [out_path], pad=False)[0]


@torch.no_grad()
def run_one_image_restore(img, tgt, size, model, out_path, device):
    """SIDD denoising / LoL enhancement / deraining: the de-normalised prediction, bicubic-resized, unclipped.
    Returns the float64 numpy array [height, width, 3] (the caller clips it and scores it); out_path is unused, as in
    the reference."""
    return _run([img], [tgt], [size], model, device, "restore", None, pad=False)[0]


# run_batch task -> (the run_one_image* it batches, pk_denorm_bottom_batched finish, pk_finish_ragged op)
TASKS = {
    "segm": ("run_one_image", CLIP255, _se.FIN_BILINEAR_U8),
    "nearest": ("run_one_image_nearest", CLIP255, _se.FIN_NEAREST_U8),
    "depth": ("run_one_image_depth", CLIP10000, _se.FIN_DEPTH),
    "restore": ("run_one_image_restore", PLAIN, _se.FIN_BICUBIC_F64),
}


def _cl_form(task, OH, OW):
    """pk_finish_ragged's cl_form for one output size: whether torch-CPU's F.interpolate of the 3-channel image takes
    its channels-last kernel, whose nearest source index and bilinear tap order differ from its generic kernel's.  It
    does for OH + OW <= 128 and, for the depth task's bilinear resize, on one thread."""
    if task == "nearest":
        return int(OH + OW <= 128)
    if task == "depth":
        return int(torch.get_num_threads() == 1 or OH + OW <= 128)
    return 0


@torch.no_grad()
def run_batch(imgs, tgts, sizes, model, device, task, out_paths=None):
    """B images of one eval task in one forward: imgs, tgts are B numpy [2*S, S, 3] ImageNet-normalised canvases (as
    the eval scripts build them), sizes B (width, height) source sizes, task one of TASKS.  Returns, and for the PNG
    tasks writes to out_paths (if given), per image exactly what the matching run_one_image* returns or writes: device
    uint8 / int32 images, or float64 numpy arrays for "restore".  model: the module or a `.module` wrapper.

    One upload (canvases + descriptor table), one graphed forward, one de-normalise launch, one ragged resize launch,
    one download.  A batch smaller than one already captured for this canvas shape is padded to it by repeating the
    last canvas (the padding is dropped), so a dataset's tail batch replays the same CUDA graph."""
    return _run(imgs, tgts, sizes, model, device, task, out_paths, pad=True)


def _run(imgs, tgts, sizes, model, device, task, out_paths, pad):
    """run_batch, with a forward of exactly len(imgs) canvases unless pad."""
    if task not in TASKS:
        raise ValueError(f"run_batch: task must be one of {sorted(TASKS)}, got {task!r}")
    B = len(imgs)
    if B < 1 or len(tgts) != B or len(sizes) != B or (out_paths is not None and len(out_paths) != B):
        raise ValueError(f"run_batch: {B} canvases, {len(tgts)} targets, {len(sizes)} sizes")
    # one canvas stays a view: upload copies it into its pinned buffer, and a stack would copy it first
    x, t = (np.asarray(c[0])[None] if B == 1 else np.stack([np.asarray(a) for a in c]) for c in (imgs, tgts))
    if x.dtype not in (np.float32, np.float64) or t.dtype != x.dtype or x.shape != t.shape or x.shape[-1] != 3:
        raise ValueError(f"run_batch: canvases {x.shape} {x.dtype} / targets {t.shape} {t.dtype}")
    _, finish, op = TASKS[task]
    device = torch.device(device)
    net = model.module if hasattr(model, "module") else model
    out_hw = [(int(sz[1]), int(sz[0])) for sz in sizes]
    tab, offs, total, max_pix = _se.ragged_table(op, range(B), out_hw, [_cl_form(task, *hw) for hw in out_hw])
    xd, td, tab_d = _se.upload([x, t, tab], device)
    _, H, W, _ = x.shape
    p = net.patch_size
    h, w = H // p, W // p
    g = _graphed(net)
    Bc = g.captured_batch((B, 3, H, W), B) if pad else B
    _se.precheck_memory(net, Bc, H, W)
    xin = torch.empty((Bc, 3, H, W), dtype=torch.float32, device=device)
    tin = torch.empty((Bc, 3, H, W), dtype=torch.float32, device=device)
    for src, dst in ((xd, xin), (td, tin)):
        check(lib().pk_nhwc_to_nchw_f32(ctypes.c_void_p(src.data_ptr()), int(src.dtype == torch.float64),
                                        ctypes.c_void_p(dst.data_ptr()), B, H, W, _stream()), "pk_nhwc_to_nchw_f32")
        dst[B:] = dst[B - 1]
    c = net.__dict__.get("_pk_batch_consts")
    if c is None or c[0] != (Bc, H, W, device):
        n = h * w
        mask = torch.zeros(1, n, device=device)
        mask[:, n // 2:] = 1
        c = ((Bc, H, W, device), mask, torch.ones((Bc, 3, H, W), device=device))
        net.__dict__["_pk_batch_consts"] = c
    _, y, _ = g(xin, tin, c[1], c[2])
    seg, _ = _se.denorm_bottom_batched(y, B, h, w, p, finish)
    dst = _se.finish_ragged(op, seg, tab_d, B, max_pix, total)
    host = dst.cpu().numpy()
    per = 1 if task == "depth" else 3
    shapes = [(oh, ow) if task == "depth" else (oh, ow, 3) for oh, ow in out_hw]
    if task == "restore":
        return [host[o:o + oh * ow * per].reshape(s) for o, (oh, ow), s in zip(offs, out_hw, shapes)]
    out = []
    for b, (o, (oh, ow), s) in enumerate(zip(offs, out_hw, shapes)):
        out.append(dst[o:o + oh * ow * per].view(s))
        if out_paths is not None:
            from PIL import Image
            Image.fromarray(host[o:o + oh * ow * per].reshape(s)).save(out_paths[b])
    return out
