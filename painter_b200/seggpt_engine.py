"""GPU-side mirror of SegGPT/SegGPT_inference/seggpt_engine.py (SURVEY §8 f.2): the same three entry points

    run_one_image(img, tgt, model, device)                                   seggpt_engine.py:26-53
    inference_image(model, device, img_path, img2_paths, tgt2_paths, out_path)       :56-103
    inference_video(model, device, vid_path, num_frames, img2_paths, tgt2_paths, out_path)  :106-181

with identical arguments and results, but with everything between the decoded uint8 pixels and the finished uint8
frame on the GPU: stitch + ImageNet normalisation + nhwc->nchw (pk_stitch_normalize), the forward (one CUDA-graph
replay, painter_b200/graphs.py), unpatchify + bottom half + de-normalisation + clip (pk_denorm_bottom_batched),
nearest resize to the source size + alpha blend (pk_finish_ragged).  Image / video decoding, PIL resizing to 448x448
and file output stay on the host (file I/O is out of scope, SURVEY §2 row 5); the video path keeps its rolling
prompt cache (previous frames and their binarised predictions, seggpt_engine.py:13-23,128-171) resident in HBM, so a
frame costs one 0.6 MB upload however many cached prompts vote on it.
"""
import ctypes

import numpy as np
import torch

from . import ops
from ._lib import check, lib
from .graphs import GraphedForward

imagenet_mean = np.array([0.485, 0.456, 0.406])
imagenet_std = np.array([0.229, 0.224, 0.225])

_DT = {torch.uint8: 0, torch.float32: 1, torch.float64: 2}


class Cache(list):
    """seggpt_engine.py:13-23: bounded FIFO of prompt frames."""

    def __init__(self, max_size=0):
        super().__init__()
        self.max_size = max_size

    def append(self, x):
        if self.max_size <= 0:
            return
        super().append(x)
        if len(self) > self.max_size:
            self.pop(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _graphed(model):
    g = model.__dict__.get("_pk_graphed")
    if g is None:
        g = GraphedForward(model)
        model.__dict__["_pk_graphed"] = g
    return g


def stitch_normalize(tops, bottoms, S):
    """tops / bottoms: lists of P device tensors [S, S, 3] (uint8, or fp32 / fp64 in [0, 1]) -> fp32 [P, 3, 2S, S]."""
    P = len(tops)
    assert P == len(bottoms) and P >= 1
    dev = tops[0].device
    for t in list(tops) + list(bottoms):
        assert t.is_cuda and t.is_contiguous() and tuple(t.shape) == (S, S, 3) and t.dtype in _DT, (t.shape, t.dtype)
    arr = ctypes.c_void_p * P
    ia = ctypes.c_int * P
    out = torch.empty((P, 3, 2 * S, S), dtype=torch.float32, device=dev)
    check(lib().pk_stitch_normalize(arr(*[t.data_ptr() for t in tops]), ia(*[_DT[t.dtype] for t in tops]),
                                    arr(*[t.data_ptr() for t in bottoms]), ia(*[_DT[t.dtype] for t in bottoms]),
                                    ctypes.c_void_p(out.data_ptr()), P, S, _stream()), "pk_stitch_normalize")
    return out


def denorm_bottom_batched(patch, B, h, w, p, finish=0, src_stride=1, want_bin=False):
    """patchified prediction [*, h*w, p*p*3] fp32 -> fp64 [B, h*p/2, w*p, 3]: the bottom half of samples 0, src_stride,
    2 src_stride, .. de-normalised, then x255 clipped (finish 0), x10000 clipped (1) or left as is (2); optional fp32
    {0,1} mask [B, h*p/2, w*p] (finish 0 only).  Sample b is what a B = 1 call on sample b * src_stride alone gives."""
    assert patch.dtype == torch.float32 and patch.is_contiguous() and patch.shape[0] >= (B - 1) * src_stride + 1
    out = torch.empty((B, h * p // 2, w * p, 3), dtype=torch.float64, device=patch.device)
    b = torch.empty((B, h * p // 2, w * p), dtype=torch.float32, device=patch.device) if want_bin else None
    check(lib().pk_denorm_bottom_batched(ctypes.c_void_p(patch.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                         ctypes.c_void_p(b.data_ptr()) if b is not None else None, B, src_stride, h,
                                         w, p, finish, _stream()), "pk_denorm_bottom_batched")
    return out, b


# pk_finish_ragged ops (include/painter_b200.h PK_FIN_*) and their output dtype / elements per pixel
FIN_BILINEAR_U8, FIN_NEAREST_U8, FIN_DEPTH, FIN_BICUBIC_F64, FIN_NEAREST_BLEND = range(5)
_FIN_OUT = {FIN_BILINEAR_U8: (torch.uint8, 3), FIN_NEAREST_U8: (torch.uint8, 3), FIN_DEPTH: (torch.int32, 1),
            FIN_BICUBIC_F64: (torch.float64, 3), FIN_NEAREST_BLEND: (torch.uint8, 3)}
RAG_FIELDS = 6


def ragged_table(op, srcs, sizes, cl_forms=None):
    """Descriptor table of one pk_finish_ragged launch: image i is finished from source sample srcs[i] to
    sizes[i] = (OH, OW) with torch-CPU's form cl_forms[i].  Returns (int32 [n, RAG_FIELDS] rows [src, OH, OW, cl_form,
    offset lo, hi], element offset of every image in the packed output, total elements, largest OH * OW)."""
    n = len(srcs)
    if n < 1 or n > 65535 or len(sizes) != n or (cl_forms is not None and len(cl_forms) != n):
        raise ValueError(f"ragged_table: {n} images (1 .. 65535), {len(sizes)} sizes")
    per = _FIN_OUT[op][1]
    tab = np.zeros((n, RAG_FIELDS), dtype=np.int64)
    offs, off, max_pix = [], 0, 0
    for i, (s, (oh, ow)) in enumerate(zip(srcs, sizes)):
        oh, ow, s = int(oh), int(ow), int(s)
        if s < 0 or oh < 1 or ow < 1 or oh * ow * per >= 2 ** 31:
            raise ValueError(f"ragged_table: image {i}: source sample {s}, size {oh} x {ow}")
        tab[i, :4] = (s, oh, ow, int(cl_forms[i]) if cl_forms is not None else 0)
        tab[i, 4], tab[i, 5] = off & 0xFFFFFFFF, off >> 32
        offs.append(off)
        off += oh * ow * per
        max_pix = max(max_pix, oh * ow)
    return tab.astype(np.uint32).view(np.int32), offs, off, max_pix


def finish_ragged(op, src, table_dev, n, max_pix, total, image=None):
    """One launch finishing n images from src fp64 [B, SH, SW, 3] into a packed output of `total` elements
    (table_dev: ragged_table's rows on the device; image: the packed uint8 source images of the blend)."""
    assert src.dtype == torch.float64 and src.is_contiguous() and src.dim() == 4 and table_dev.dtype == torch.int32
    assert table_dev.is_contiguous() and table_dev.numel() == n * RAG_FIELDS
    dst = torch.empty((total,), dtype=_FIN_OUT[op][0], device=src.device)
    check(lib().pk_finish_ragged(op, ctypes.c_void_p(src.data_ptr()), src.shape[1], src.shape[2],
                                 ctypes.c_void_p(table_dev.data_ptr()), n, max_pix,
                                 ctypes.c_void_p(image.data_ptr()) if image is not None else None,
                                 ctypes.c_void_p(dst.data_ptr()), _stream()), "pk_finish_ragged")
    return dst


_staging = {}


def upload(arrays, device):
    """Copy host arrays to the device in ONE transfer from a reused pinned buffer.  Returns one device tensor per
    array (same dtype and shape, 16-byte aligned views of one device buffer)."""
    device = torch.device(device)
    arrays = [np.ascontiguousarray(a) for a in arrays]
    offs, n = [], 0
    for a in arrays:
        offs.append(n)
        n += (a.nbytes + 15) // 16 * 16
    ent = _staging.get(device)
    if ent is None or ent[0].numel() < n:
        ent = (torch.empty((max(n, 1),), dtype=torch.uint8, pin_memory=True), torch.cuda.Event())
        _staging[device] = ent
    host, done = ent
    done.synchronize()          # the previous transfer out of the pinned buffer has finished
    for a, o in zip(arrays, offs):      # torch copies on its intra-op threads, a numpy assignment on one
        host[o:o + a.nbytes].copy_(torch.from_numpy(a.reshape(-1).view(np.uint8)))
    dev = torch.empty((max(n, 1),), dtype=torch.uint8, device=device)
    dev.copy_(host[:max(n, 1)], non_blocking=True)
    done.record()
    return [dev[o:o + a.nbytes].view(torch.from_numpy(a[:0].reshape(-1)).dtype).view(a.shape)
            for a, o in zip(arrays, offs)]


def _half_mask(model, device):
    n = model.patch_embed.num_patches
    m = torch.zeros(1, n, device=device)
    m[:, n // 2:] = 1
    return m


def _forward(model, x, tgt, device, prompts_per_query=None):
    """The call of seggpt_engine.py:36-47 on device tensors x, tgt [P, 3, 896, 448] fp32; returns patchify(pred).
    prompts_per_query: the batch is [Q][P] members of Q queries, each ensembled over its own P prompts."""
    P = x.shape[0]
    key = ("seg_consts", P, str(device), model.seg_type)
    c = model.__dict__.get("_pk_seg_consts")
    if c is None or c[0] != key:
        seg_type = torch.ones([P, 1], device=device) if model.seg_type == 'instance' else \
            torch.zeros([P, 1], device=device)
        c = (key, _half_mask(model, device), torch.ones((P, 3, x.shape[2], x.shape[3]), device=device), seg_type)
        model.__dict__["_pk_seg_consts"] = c
    _, mask, valid, seg_type = c
    group = P if prompts_per_query is None else prompts_per_query
    feat_ensemble = 0 if group > 1 else -1
    _, y, _ = _graphed(model)(x, tgt, mask, valid, seg_type, feat_ensemble,
                              prompts_per_query if feat_ensemble == 0 else None)
    return y


@torch.no_grad()
def run_one_image(img, tgt, model, device):
    """img, tgt: numpy [P, 896, 448, 3] (already ImageNet-normalised, float64 as the reference callers build them).
    Returns what the reference returns: a CPU float64 tensor [448, 448, 3], the de-normalised bottom half in [0, 255]."""
    device = torch.device(device)
    x = torch.as_tensor(img)
    t = torch.as_tensor(tgt)
    P, H, W, _ = x.shape
    xd, td = x.to(device, non_blocking=True), t.to(device, non_blocking=True)
    xin = torch.empty((P, 3, H, W), dtype=torch.float32, device=device)
    tin = torch.empty((P, 3, H, W), dtype=torch.float32, device=device)
    for src, dst in ((xd, xin), (td, tin)):
        assert src.dtype in (torch.float32, torch.float64)
        check(lib().pk_nhwc_to_nchw_f32(ctypes.c_void_p(src.data_ptr()), int(src.dtype == torch.float64),
                                        ctypes.c_void_p(dst.data_ptr()), P, H, W, _stream()), "pk_nhwc_to_nchw_f32")
    y = _forward(model, xin, tin, device)
    p = model.patch_size
    out, _ = denorm_bottom_batched(y, 1, H // p, W // p, p)
    return out[0].cpu()


def _load_prompt(img2_path, tgt2_path, res, hres, device):
    from PIL import Image
    img2 = Image.open(img2_path).convert("RGB").resize((res, hres))
    tgt2 = Image.open(tgt2_path).convert("RGB").resize((res, hres), Image.NEAREST)
    return (torch.from_numpy(np.array(img2)).to(device), torch.from_numpy(np.array(tgt2)).to(device))


@torch.no_grad()
def segment(model, device, image_u8, prompts, want_bin=False):
    """image_u8: device uint8 [448, 448, 3] (the query, resized); prompts: list of (prompt image, prompt target)
    device tensors [448, 448, 3] (uint8, or float in [0,1] for cached video frames).  Returns (fp64 [448, 448, 3] in
    [0, 255], optional binarised mask) - seggpt_engine.py:65-93 without the host arithmetic."""
    out, binm = _segment(model, device, [image_u8], prompts, want_bin, pad=False)
    return out[0], None if binm is None else binm[0]


@torch.no_grad()
def segment_batch(model, device, images_u8, prompts, want_bin=False):
    """segment() of Q queries that share one prompt set, in one forward of Q x P members ([Q][P], each query ensembled
    over its own P prompts).  images_u8: device uint8 [Q, 448, 448, 3] (or a list of Q such images); prompts as in
    segment().  Returns (fp64 [Q, 448, 448, 3], optional mask [Q, 448, 448]); entry q equals segment(..., images_u8[q],
    prompts, want_bin) bit for bit.  A batch smaller than one already captured is padded to it by repeating the last
    query (its whole prompt group), so a folder runs on one CUDA graph; the padding is dropped."""
    Q, P = len(images_u8), len(prompts)
    if Q < 1 or P < 1:
        raise ValueError(f"segment_batch: {Q} queries, {P} prompts")
    return _segment(model, device, images_u8, prompts, want_bin, pad=True)


@torch.no_grad()
def _segment(model, device, images_u8, prompts, want_bin, pad):
    """segment_batch, with a forward of exactly len(images_u8) queries unless pad."""
    device = torch.device(device)
    Q, P = len(images_u8), len(prompts)
    S = images_u8[0].shape[0]
    p = model.patch_size
    Qc = _graphed(model).captured_batch((Q * P, 3, 2 * S, S), Q * P, P if P > 1 else None) // P if pad else Q
    qs = [images_u8[q] for q in range(Q)] + [images_u8[Q - 1]] * (Qc - Q)
    precheck_memory(model, Qc * P, 2 * S, S)
    x = stitch_normalize([pr[0] for _ in qs for pr in prompts], [q for q in qs for _ in prompts], S)
    t = stitch_normalize([pr[1] for _ in qs for pr in prompts], [pr[1] for _ in qs for pr in prompts], S)
    torch.manual_seed(2)      # seggpt_engine.py:91 (no random op follows in eval mode; kept for RNG-state parity)
    y = _forward(model, x, t, device, P)
    # query q is member q * P's bottom half (seggpt_engine.py:48 takes member 0 of its batch)
    return denorm_bottom_batched(y, Q, 2 * S // p, S // p, p, 0, src_stride=P, want_bin=want_bin)


def precheck_memory(model, B, H, W):
    """Refuse, before any allocation, an fp32-accurate forward of B canvases that cannot fit in the device memory
    left (accurate.workspace_bytes); the bf16 forward needs far less and is not checked."""
    from . import accurate
    if not accurate.selected(model):
        return
    need = accurate.workspace_bytes(model, B, H, W)
    free, _ = torch.cuda.mem_get_info()
    if need > free:     # each of these builds the allocator's whole statistics dict: read them only when they matter
        free += torch.cuda.memory_reserved() - torch.cuda.memory_allocated()
    if need > free:
        per = accurate.workspace_bytes(model, 1, H, W)
        raise RuntimeError(f"painter_b200: an fp32-accurate forward of {B} canvases of {H} x {W} needs about "
                           f"{need / 2**30:.1f} GiB and {free / 2**30:.1f} GiB is free; use a batch of at most "
                           f"{max(1, int(free // per))} canvases, or model.precision = 'bf16'")


def _blend(model, device, images, prompts, pad):
    """The queries' segmentations blended onto them at their own sizes (seggpt_engine.py:65-102): images are Q decoded
    RGB PIL images.  One upload (the resized queries, the source images and the blend's descriptor table), one
    forward (padded as in segment_batch if pad), one ragged blend launch.  Returns (packed uint8 device output, element
    offset of every image in it)."""
    srcs = [np.array(im) for im in images]
    small = np.stack([np.array(im.resize((448, 448))) for im in images])
    tab, offs, total, max_pix = ragged_table(FIN_NEAREST_BLEND, range(len(srcs)), [a.shape[:2] for a in srcs])
    flat = np.concatenate([a.reshape(-1) for a in srcs])
    small_d, flat_d, tab_d = upload([small, flat, tab], device)
    out, _ = _segment(model, device, small_d, prompts, want_bin=False, pad=pad)
    return finish_ragged(FIN_NEAREST_BLEND, out, tab_d, len(srcs), max_pix, total, image=flat_d), offs


def inference_images(model, device, img_paths, img2_paths, tgt2_paths, out_paths, batch_size=8):
    """inference_image() over a folder of queries sharing one prompt set, batch_size queries per forward: writes the
    same PNG files as one inference_image call per query.  Per batch: one upload, one forward, one ragged blend launch,
    one download."""
    from PIL import Image
    device = torch.device(device)
    if len(img_paths) != len(out_paths) or batch_size < 1:
        raise ValueError("inference_images: one output path per query image, batch_size >= 1")
    prompts = [_load_prompt(a, b, 448, 448, device) for a, b in zip(img2_paths, tgt2_paths)]
    for b0 in range(0, len(img_paths), batch_size):
        images = [Image.open(pth).convert("RGB") for pth in img_paths[b0:b0 + batch_size]]
        blended, offs = _blend(model, device, images, prompts, pad=True)
        host = blended.cpu().numpy()
        for q, (im, o) in enumerate(zip(images, offs)):
            h, w = im.height, im.width
            Image.fromarray(host[o:o + h * w * 3].reshape(h, w, 3)).save(out_paths[b0 + q])


def inference_image(model, device, img_path, img2_paths, tgt2_paths, out_path):
    from PIL import Image
    device = torch.device(device)
    image = Image.open(img_path).convert("RGB")
    prompts = [_load_prompt(a, b, 448, 448, device) for a, b in zip(img2_paths, tgt2_paths)]
    blended, _ = _blend(model, device, [image], prompts, pad=False)
    blended = blended.view(image.height, image.width, 3)
    Image.fromarray(blended.cpu().numpy()).save(out_path)
    return blended


def inference_video(model, device, vid_path, num_frames, img2_paths, tgt2_paths, out_path):
    import cv2
    from PIL import Image
    device = torch.device(device)
    res, hres = 448, 448
    cap = cv2.VideoCapture(vid_path)
    fps = cap.get(cv2.CAP_PROP_FPS)
    width = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH))
    height = int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
    fourcc = cv2.VideoWriter_fourcc(*'mp4v')
    video_writer = cv2.VideoWriter(out_path, fourcc, fps, (width, height), True)
    if img2_paths is None:
        _, frame = cap.read()
        img2 = Image.fromarray(frame[:, :, ::-1]).convert('RGB')
    else:
        img2 = Image.open(img2_paths[0]).convert("RGB")
    img2 = torch.from_numpy(np.array(img2.resize((res, hres)))).to(device)
    tgt2 = Image.open(tgt2_paths[0]).convert("RGB").resize((res, hres), Image.NEAREST)
    tgt2 = torch.from_numpy(np.array(tgt2)).to(device)
    frames_cache, target_cache = Cache(num_frames), Cache(num_frames)
    tab_d = None
    n = 0
    while True:
        ret, frame = cap.read()
        if not ret:
            break
        image = Image.fromarray(frame[:, :, ::-1]).convert('RGB')
        input_image = torch.from_numpy(np.array(image)).to(device)
        if tab_d is None:       # one blend table for the whole video
            hw = input_image.shape[:2]
            tab, _, total, max_pix = ragged_table(FIN_NEAREST_BLEND, [0], [hw])
            tab_d = torch.from_numpy(tab).to(device)
        elif input_image.shape[:2] != hw:
            raise ValueError(f"inference_video: frame {n} is {tuple(input_image.shape[:2])}, frame 0 {tuple(hw)}")
        image_r = torch.from_numpy(np.array(image.resize((res, hres)))).to(device)
        prompts = list(zip([img2] + frames_cache, [tgt2] + target_cache))
        out, binm = segment(model, device, image_r, prompts, want_bin=num_frames > 0)
        frames_cache.append(image_r)
        if num_frames > 0:
            target_cache.append(binm.unsqueeze(-1).expand(-1, -1, 3).contiguous())
        blended = finish_ragged(FIN_NEAREST_BLEND, out.unsqueeze(0), tab_d, 1, max_pix, total, image=input_image)
        video_writer.write(np.ascontiguousarray(blended.view(input_image.shape).cpu().numpy()[:, :, ::-1]))
        n += 1
    video_writer.release()
    return n
