"""Per-sample work of the training data path on the GPU (SURVEY §8 f.4): what `PairDataset.__getitem__`
(Painter/data/pairdataset.py:106-190) does after the images are decoded and augmented, without the host.

  DeviceMaskingGenerator   util/masking_generator.py:15-93 + the half-mask draw of pairdataset.py:149,183-186
  valid_maps               pairdataset.py:154-181 (per-task `valid` weighting of the loss)
  combine_pairs            pairdataset.py:100-104,136-146 (second pair stitched under the first)

The recipe's augmentations (DevicePairDataset, pair_collate, DevicePairAugment, DevicePairPrefetcher below) run on the
device bit-identically to PIL / torch-CPU; decoding and the random draws stay on the host."""
import ctypes
import json
import math
import os
import random

import numpy as np
import torch

from ._lib import check, lib

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class DeviceMaskingGenerator:
    """Same constructor as the reference MaskingGenerator; `gen(B, seed)` returns int32 [B, h, w] on the device."""

    def __init__(self, input_size, num_masking_patches, min_num_patches=4, max_num_patches=None, min_aspect=0.3,
                 max_aspect=None, half_mask_ratio=0.0, device="cuda"):
        if not isinstance(input_size, tuple):
            input_size = (input_size,) * 2
        self.height, self.width = input_size
        self.num_patches = self.height * self.width
        self.num_masking_patches = num_masking_patches
        self.min_num_patches = min_num_patches
        self.max_num_patches = num_masking_patches if max_num_patches is None else max_num_patches
        max_aspect = max_aspect or 1 / min_aspect
        self.log_aspect_ratio = (math.log(min_aspect), math.log(max_aspect))
        self.half_mask_ratio = half_mask_ratio
        self.device = torch.device(device)
        self._calls = 0

    def get_shape(self):
        return self.height, self.width

    def __call__(self, B=1, seed=None):
        if seed is None:
            seed = 0x5EED0000 + self._calls
        self._calls += 1
        out = torch.empty((B, self.height, self.width), dtype=torch.int32, device=self.device)
        check(lib().pk_block_masks(ctypes.c_void_p(out.data_ptr()), B, self.height, self.width,
                                   self.num_masking_patches, self.min_num_patches, self.max_num_patches,
                                   ctypes.c_float(self.log_aspect_ratio[0]), ctypes.c_float(self.log_aspect_ratio[1]),
                                   ctypes.c_float(self.half_mask_ratio), ctypes.c_ulonglong(seed), _stream()),
              "pk_block_masks")
        return out


def _rule_and_threshold(pair_type):
    """pairdataset.py:157-181 -> (rule code, threshold before normalisation)."""
    if "nyuv2_image2depth" in pair_type:
        return 1, 1e-3 * 0.1
    if "ade20k_image2semantic" in pair_type or "coco_image2panoptic_sem_seg" in pair_type:
        return 1, 1e-5
    if "image2pose" in pair_type:
        return 2, 1e-5
    if "image2panoptic_inst" in pair_type:
        return 3, 1e-5
    return 0, 0.0


def valid_maps(targets, pair_types):
    """targets: fp32 [B, 3, H, W] on the device (normalised); pair_types: list of B type strings -> valid [B,3,H,W]."""
    assert targets.is_cuda and targets.dtype == torch.float32 and targets.is_contiguous()
    B, _, H, W = targets.shape
    rules, thr = [], []
    mean = torch.tensor(IMAGENET_MEAN)
    std = torch.tensor(IMAGENET_STD)
    for t in pair_types:
        r, th = _rule_and_threshold(t)
        rules.append(r)
        thr.append((torch.ones(3) * th - mean) / std)      # the reference's fp32 torch arithmetic, bit for bit
    rule_d = torch.tensor(rules, dtype=torch.int32).to(targets.device)
    thr_d = torch.stack(thr).to(targets.device).contiguous()
    fg = torch.zeros(B, dtype=torch.int32, device=targets.device)
    valid = torch.empty_like(targets)
    check(lib().pk_valid_maps(ctypes.c_void_p(targets.data_ptr()), ctypes.c_void_p(rule_d.data_ptr()),
                              ctypes.c_void_p(thr_d.data_ptr()), ctypes.c_void_p(fg.data_ptr()),
                              ctypes.c_void_p(valid.data_ptr()), B, H, W, _stream()), "pk_valid_maps")
    return valid


def combine_pairs(first, second):
    """pairdataset.py:100-104: the second pair goes under the first ([.., 3, H, W] x 2 -> [.., 3, 2H, W])."""
    return torch.cat([first, second], dim=-2)


# ---------------------------------------------------------------------------------------------------------------------
# The recipe's paired augmentations (main_train.py:232-262, applied by pairdataset.py:106-190) with the pixel arithmetic
# on the device.  DevicePairDataset decodes and makes every random draw in the DataLoader worker (same calls, same
# generators, same order as PairDataset with the stock transforms); pair_collate packs a batch's uint8 images and
# descriptors into one flat buffer; DevicePairAugment turns it into (samples, targets, masks, valid) with one H2D copy
# and csrc/augment.cu's kernels, bit-identical to what PairDataset + default_collate produce from the same seeds.

_JIT = None


def _color_jitter():
    global _JIT
    if _JIT is None:
        from torchvision.transforms import ColorJitter
        _JIT = ColorJitter(0.4, 0.4, 0.2, 0.1)       # main_train.py:236; only its ranges and get_params are used
    return _JIT


def _shape_only(c, h, w):
    """A [c, h, w] tensor without storage: RandomResizedCrop.get_params reads nothing but the shape."""
    return torch.empty(1).expand(c, h, w)


class DevicePairDataset(torch.utils.data.Dataset):
    """PairDataset with the stock transforms, minus the pixel work.

    root, json_path_list, use_two_pairs and half_mask_ratio mean what they mean to PairDataset; input_size is
    main_train.py's (2S, S) and min_random_scale its --min_random_scale.  train=True is transform_train /
    transform_train2 / transform_train3 + transform_train_seccrop, train=False is transform_val alone.
    masked_position_generator is called per sample as PairDataset does (the reference MaskingGenerator keeps batches
    comparable); a DeviceMaskingGenerator is instead run per batch by DevicePairAugment.  `weights`, `pairs` and
    `pair_type_dict` are PairDataset's, so the reference samplers work unchanged.

    __getitem__ returns (images, record): uint8 [H, W, 3] arrays (image, target, then the second pair's) and the draws.
    """

    TYPE_WEIGHTS = (0.1, 0.2, 0.15, 0.25, 0.2, 0.15, 0.05, 0.05)    # pairdataset.py: per json file

    def __init__(self, root, json_path_list, input_size=(896, 448), min_random_scale=0.3, half_mask_ratio=0.0,
                 use_two_pairs=True, masked_position_generator=None, train=True, transforms=None):
        if transforms is not None:
            raise NotImplementedError("DevicePairDataset runs the stock recipe only (RandomErasing, GaussianBlur and "
                                      "other transforms have no device implementation)")
        if not isinstance(input_size, (tuple, list)):
            input_size = (input_size, input_size)
        if input_size[0] != 2 * input_size[1]:
            raise NotImplementedError("input_size must be (2S, S): two S x S pairs stitched")
        if train and not use_two_pairs:
            raise NotImplementedError("the second crop of the stock recipe needs the two-pair canvas")
        self.root = root
        self.input_size = tuple(input_size)
        self.size = input_size[1]
        self.min_random_scale = min_random_scale
        self.half_mask_ratio = half_mask_ratio
        self.use_two_pairs = use_two_pairs
        self.train = train
        self.masked_position_generator = masked_position_generator
        self.pairs, self.weights = [], []
        for idx, jp in enumerate(json_path_list):
            with open(jp) as f:
                cur = json.load(f)
            self.pairs.extend(cur)
            self.weights.extend([self.TYPE_WEIGHTS[idx] * 1. / len(cur)] * len(cur))
        self.pair_type_dict = {}
        if use_two_pairs:
            for idx, pair in enumerate(self.pairs):
                if "type" in pair:
                    self.pair_type_dict.setdefault(pair["type"], []).append(idx)

    def __len__(self):
        return len(self.pairs)

    def _load_image(self, path):
        """pairdataset.py _load_image: PIL decode, NYUv2 depth rescaled to 0..255, RGB."""
        from PIL import Image
        img = Image.open(os.path.join(self.root, path))
        if "sync_depth" in path:
            img = Image.fromarray(np.array(img) / 10000. * 255)
        return np.asarray(img.convert("RGB"))

    def _draw_pair(self, img, augment):
        """The draws of one pair's transform, in Compose order."""
        from torchvision.transforms import RandomResizedCrop
        h, w = img.shape[:2]
        scale = (self.min_random_scale, 1.0) if augment else (0.9999, 1.0)
        box = RandomResizedCrop.get_params(_shape_only(3, h, w), scale, (3. / 4., 4. / 3.))
        jitter, flip = None, False
        if augment:
            if not 0.8 < torch.rand(1):                               # RandomApply(p=0.8)
                cj = _color_jitter()
                fn_idx, b, c, s, hf = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
                jitter = ([int(k) for k in fn_idx], float(b), float(c), float(s), int(hf * 255) % 256)
            flip = bool(torch.rand(1) < 0.5)                          # RandomHorizontalFlip
        return {"box": tuple(int(v) for v in box), "jitter": jitter, "flip": flip}

    def __getitem__(self, index):
        from torchvision.transforms import RandomResizedCrop
        pair = self.pairs[index]
        ptype = pair["type"]
        if "depth" in ptype or "pose" in ptype:
            modes = (0, 0)
        elif "image2" in ptype:
            modes = (0, 1)
        elif "2image" in ptype:
            modes = (1, 0)
        else:
            modes = (0, 0)
        # transform_train augments; transform_train2 / 3 (instances, pose) and transform_val only crop
        augment = self.train and not ("inst" in ptype or "pose" in ptype)
        images = [self._load_image(pair["image_path"]), self._load_image(pair["target_path"])]
        pairs = [self._draw_pair(images[0], augment)]
        if self.use_two_pairs:
            pair2 = self.pairs[random.choice(self.pair_type_dict[ptype])]
            assert pair2["type"] == ptype
            images += [self._load_image(pair2["image_path"]), self._load_image(pair2["target_path"])]
            pairs.append(self._draw_pair(images[2], augment))
        half = bool(torch.rand(1)[0] < self.half_mask_ratio)
        sec = None
        if self.train and not ("inst" in ptype or "pose" in ptype or half):
            sec = tuple(int(v) for v in RandomResizedCrop.get_params(_shape_only(3, *self.input_size),
                                                                     (self.min_random_scale, 1.0), (0.3, 0.7)))
        mask = None
        if half:
            mask = np.zeros(self.masked_position_generator.get_shape(), dtype=np.int32)
            mask[mask.shape[0] // 2:, :] = 1
        elif not isinstance(self.masked_position_generator, DeviceMaskingGenerator):
            mask = np.asarray(self.masked_position_generator(), dtype=np.int32)
        record = {"type": ptype, "size": self.size, "modes": modes, "pairs": pairs, "half": half, "sec": sec, "mask": mask,
                  "mask_shape": tuple(self.masked_position_generator.get_shape())}
        return images, record



def _ceil_taps(src, size):
    """Pillow's coefficient count for a bicubic resize of `src` pixels to `size` (precompute_coeffs' ksize)."""
    return int(math.ceil(2.0 * max(float(src) / size, 1.0))) * 2 + 1


class PackedPairBatch:
    """One batch of DevicePairDataset items in a single flat uint8 buffer: an int32 descriptor table (crop, jitter and
    second-crop rows, valid-map rules and thresholds, masks) followed by every decoded image back to back."""

    def __init__(self, buf, meta):
        self.buf = buf
        self.meta = meta

    def pin_memory(self):
        return PackedPairBatch(self.buf.pin_memory(), self.meta)


def pair_collate(batch):
    """DataLoader collate_fn for DevicePairDataset: [(images, record)] -> PackedPairBatch."""
    B = len(batch)
    P = len(batch[0][0]) // 2
    rec0 = batch[0][1]
    S = None
    crop, jit, sec, rules, thr, masks, types, halves = [], [], [], [], [], [], [], []
    images, img_off, tmp_off, KP, max_rows = [], 0, 0, 5, 1
    mean, std = torch.tensor(IMAGENET_MEAN), torch.tensor(IMAGENET_STD)
    for b, (imgs, rec) in enumerate(batch):
        assert len(imgs) == 2 * P
        S = rec["size"]
        for p in range(P):
            d = rec["pairs"][p]
            top, left, h, w = d["box"]
            for t in range(2):
                a = imgs[2 * p + t]
                H, W = a.shape[:2]
                assert a.dtype == np.uint8 and a.shape[2] == 3 and 0 <= top and top + h <= H and 0 <= left \
                    and left + w <= W and h > 0 and w > 0
                mode = rec["modes"][t]
                rows = max(h, w) * S * 3 if mode == 0 else 0          # the first pass's intermediate
                if mode == 0:
                    KP = max(KP, _ceil_taps(h, S), _ceil_taps(w, S))
                    max_rows = max(max_rows, h, w)
                crop.append([img_off & 0xFFFFFFFF, img_off >> 32, H, W, top, left, h, w, mode, int(d["flip"]),
                             tmp_off & 0xFFFFFFFF, tmp_off >> 32])
                images.append(np.ascontiguousarray(a).reshape(-1))
                img_off += a.size
                tmp_off += rows
                slot = (b * P + p) * 2 + t
                if t == 0 and d["jitter"] is not None:
                    order, fb, fc, fs, hue = d["jitter"]
                    bits = np.array([fb, fc, fs], dtype=np.float32).view(np.int32).tolist()
                    jit.append([slot, *order, *bits, hue])
        for t in range(2):
            if rec["sec"] is not None:
                sec.append([*rec["sec"], rec["modes"][t]])
            else:
                sec.append([0, 0, P * S, S, 1])                    # full box, nearest: an exact copy
        r, th = _rule_and_threshold(rec["type"])
        rules.append(r)
        thr.append(((torch.ones(3) * th - mean) / std).numpy())    # PairDataset's fp32 torch arithmetic
        masks.append(rec["mask"])
        types.append(rec["type"])
        halves.append(rec["half"])
    have_masks = all(m is not None for m in masks)
    parts = [np.asarray(crop, np.int32).reshape(-1), np.asarray(jit, np.int32).reshape(-1),
             np.asarray(sec, np.int32).reshape(-1), np.asarray(rules, np.int32),
             np.stack(thr).astype(np.float32).view(np.int32).reshape(-1)]
    if have_masks:
        parts.append(np.stack(masks).astype(np.int32).reshape(-1))
    offs, n = [], 0
    for a in parts:
        offs.append(n)
        n += a.size
    table_bytes = (n * 4 + 255) // 256 * 256
    buf = torch.empty(table_bytes + img_off, dtype=torch.uint8)
    flat = buf.numpy()
    tab = flat[:n * 4].view(np.int32)
    for o, a in zip(offs, parts):
        tab[o:o + a.size] = a
    pos = table_bytes
    for a in images:
        flat[pos:pos + a.size] = a
        pos += a.size
    meta = {"B": B, "P": P, "S": S, "J": len(crop), "NJ": len(jit), "KP": KP, "max_rows": max_rows,
            "tmp_bytes": max(tmp_off, 1), "table_bytes": table_bytes, "offs": offs, "have_masks": have_masks,
            "mask_shape": rec0["mask_shape"], "half": halves, "types": types,
            "second_crop": any(r["sec"] is not None for _, r in batch)}
    return PackedPairBatch(buf, meta)


class DevicePairAugment:
    """PackedPairBatch -> (samples, targets, masks, valid) on the device: one H2D copy of the packed buffer, then
    resized crop, color jitter, normalise + stitch, second crop and valid maps (csrc/augment.cu, datapath.cu).

    The outputs are this object's persistent buffers, overwritten by the next call; DevicePairPrefetcher alternates two
    instances.  mask_generator (a DeviceMaskingGenerator) draws the masks of batches packed without them."""

    def __init__(self, device="cuda", mask_generator=None):
        self.device = torch.device(device)
        self.mask_generator = mask_generator
        self._bufs = {}

    def _buf(self, name, shape, dtype, exact=True):
        t = self._bufs.get(name)
        n = math.prod(shape)
        if t is None or t.dtype != dtype or (t.shape != torch.Size(shape) if exact else t.numel() < n):
            t = torch.empty(shape if exact else (n,), dtype=dtype, device=self.device)
            self._bufs[name] = t
        return t if exact else t[:n].view(shape)

    def __call__(self, packed):
        m = packed.meta
        B, P, S, J = m["B"], m["P"], m["S"], m["J"]
        L = lib()
        st = _stream()
        buf = self._buf("packed", (packed.buf.numel(),), torch.uint8, exact=False)
        buf.copy_(packed.buf, non_blocking=True)
        tab = buf[:m["table_bytes"]].view(torch.int32)
        o_crop, o_jit, o_sec, o_rule, o_thr = m["offs"][:5]
        ptr = lambda o: ctypes.c_void_p(tab.data_ptr() + 4 * o)          # noqa: E731
        KP = m["KP"]
        coef = self._buf("coef", (J, 2, S, KP), torch.int32, exact=False)
        bounds = self._buf("bounds", (J, 2, S, 2), torch.int32, exact=False)
        tmp = self._buf("tmp", (m["tmp_bytes"],), torch.uint8, exact=False)
        slots = self._buf("slots", (J, S, S, 3), torch.uint8)
        check(L.pk_aug_resized_crop(ctypes.c_void_p(buf.data_ptr() + m["table_bytes"]), ptr(o_crop), J, S, KP,
                                    m["max_rows"], ctypes.c_void_p(coef.data_ptr()), ctypes.c_void_p(bounds.data_ptr()),
                                    ctypes.c_void_p(tmp.data_ptr()), ctypes.c_void_p(slots.data_ptr()), st),
              "pk_aug_resized_crop")
        check(L.pk_aug_color_jitter(ctypes.c_void_p(slots.data_ptr()), ptr(o_jit), m["NJ"], ctypes.c_longlong(S * S),
                                    st), "pk_aug_color_jitter")
        OH, OW = P * S, S
        second = m["second_crop"]
        img = self._buf("canvas_img" if second else "img", (B, 3, OH, OW), torch.float32)
        tgt = self._buf("canvas_tgt" if second else "tgt", (B, 3, OH, OW), torch.float32)
        check(L.pk_aug_normalize(ctypes.c_void_p(slots.data_ptr()), B, P, S, ctypes.c_void_p(img.data_ptr()),
                                 ctypes.c_void_p(tgt.data_ptr()), st), "pk_aug_normalize")
        if second:
            img_o = self._buf("img", (B, 3, OH, OW), torch.float32)
            tgt_o = self._buf("tgt", (B, 3, OH, OW), torch.float32)
            wts = self._buf("sec_wts", (2 * B, 2, OH, 5), torch.float32)
            sb = self._buf("sec_bounds", (2 * B, 2, OH, 2), torch.int32)
            stmp = self._buf("sec_tmp", (2 * B, 3, OH, OW), torch.float32)
            check(L.pk_aug_second_crop(ctypes.c_void_p(img.data_ptr()), ctypes.c_void_p(tgt.data_ptr()), ptr(o_sec),
                                       B, OH, OW, ctypes.c_void_p(wts.data_ptr()), ctypes.c_void_p(sb.data_ptr()),
                                       ctypes.c_void_p(stmp.data_ptr()), ctypes.c_void_p(img_o.data_ptr()),
                                       ctypes.c_void_p(tgt_o.data_ptr()), st), "pk_aug_second_crop")
            img, tgt = img_o, tgt_o
        valid = self._buf("valid", (B, 3, OH, OW), torch.float32)
        fg = self._buf("fg", (B,), torch.int32)
        fg.zero_()
        check(L.pk_valid_maps(ctypes.c_void_p(tgt.data_ptr()), ptr(o_rule), ptr(o_thr), ctypes.c_void_p(fg.data_ptr()),
                              ctypes.c_void_p(valid.data_ptr()), B, OH, OW, st), "pk_valid_maps")
        mh, mw = m["mask_shape"]
        masks = self._buf("masks", (B, mh, mw), torch.int32)
        if m["have_masks"]:
            o = m["offs"][5]
            masks.copy_(tab[o:o + B * mh * mw].view(B, mh, mw))
        else:
            if self.mask_generator is None:
                raise ValueError("batch packed without masks: DevicePairAugment needs a mask_generator")
            drawn = self.mask_generator(B)
            if any(m["half"]):                   # the host drew the half-mask alternative for these samples
                half = torch.tensor(m["half"]).view(B, 1, 1).to(self.device, non_blocking=True)
                rows = (torch.arange(mh, device=self.device) >= mh // 2).view(1, mh, 1).to(torch.int32)
                drawn = torch.where(half, rows, drawn)
            masks.copy_(drawn)
        return img, tgt, masks, valid


class DevicePairPrefetcher:
    """Iterate over a DataLoader of PackedPairBatch; yield (samples, targets, masks, valid) on the device.

    Batch i+1 is copied and augmented on a side stream while step i runs, with DevicePrefetcher's buffer discipline:
    two DevicePairAugment instances (two sets of outputs) alternate, the work for a set is ordered after everything
    the consumer stream had enqueued when the previous batch was handed out, and the consumer waits on its event."""

    def __init__(self, batches, device="cuda", mask_generator=None):
        self.it = iter(batches)
        self.device = torch.device(device)
        self.side = torch.cuda.Stream(device=self.device)
        self.aug = [DevicePairAugment(self.device, mask_generator), DevicePairAugment(self.device, mask_generator)]
        self.k = 0
        self._next = None
        self._preload()

    def _preload(self):
        try:
            packed = next(self.it)
        except StopIteration:
            self._next = None
            return
        aug = self.aug[self.k]
        self.k ^= 1
        self.side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.side):
            out = aug(packed)
            ev = torch.cuda.Event()
            ev.record(self.side)
        self._next = (out, ev)

    def __iter__(self):
        return self

    def __next__(self):
        if self._next is None:
            raise StopIteration
        out, ev = self._next
        torch.cuda.current_stream(self.device).wait_event(ev)
        self._preload()
        return out
