"""Device augmentation kernels (csrc/augment.cu) bit for bit against PIL / torchvision / torch-CPU, and the whole
path (DevicePairDataset + pair_collate + DevicePairAugment) against the unmodified PairDataset with the stock recipe."""
import contextlib
import ctypes
import io
import random

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image, ImageEnhance
from torchvision.transforms import InterpolationMode as IM

from _augment_data import mask_generator, reference_dataset, write_dataset
from oracle import ref_loader

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_loader.available(), reason="reference tree not staged")]

BRI, CON, SAT, HUE = 0, 1, 2, 3


def _lib():
    from painter_b200._lib import check, lib
    return lib(), check


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _jitter(imgs_u8, rows):
    """imgs_u8: uint8 [n, H, W, 3] numpy; rows: per image (ops, (b, c, s), hue) -> uint8 numpy after the device ops."""
    L, check = _lib()
    d = torch.from_numpy(np.ascontiguousarray(imgs_u8)).cuda()
    tab = []
    for k, (ops, fac, hue) in enumerate(rows):
        ops = list(ops) + [-1] * (4 - len(ops))
        tab.append([k, *ops, *np.float32(fac).view(np.int32).tolist(), hue % 256])
    t = torch.tensor(tab, dtype=torch.int32).cuda()
    npix = imgs_u8.shape[1] * imgs_u8.shape[2]
    check(L.pk_aug_color_jitter(_p(d), _p(t), len(rows), ctypes.c_longlong(npix), _st()), "jitter")
    return d.cpu().numpy()


def _all_colours():
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(1, 4096, 4096, 3)


def test_luma_and_hsv_all_colours():
    rgb = _all_colours()
    im = Image.fromarray(rgb[0])
    # saturation with factor 0 is the L image replicated: blend(L, x, 0) = L
    got = _jitter(rgb, [([SAT], (1, 1, 0), 0)])[0]
    want = np.asarray(im.convert("L"))
    assert all(np.array_equal(got[..., c], want) for c in range(3))
    # RGB -> HSV -> (h + shift) -> RGB over every colour, for shifts that move every hue to every other class
    h, s, v = im.convert("HSV").split()
    for shift in (0, 1, 43, 128, 213, 255):
        hh = Image.fromarray(((np.asarray(h).astype(np.int64) + shift) % 256).astype(np.uint8), "L")
        want = np.asarray(Image.merge("HSV", (hh, s, v)).convert("RGB"))
        got = _jitter(rgb, [([HUE], (1, 1, 1), shift)])[0]
        assert np.array_equal(got, want), (shift, int((got != want).any(-1).sum()))


@pytest.mark.parametrize("factor", [0.0, 0.37, 0.6, 0.999, 1.0, 1.17, 1.4, 2.5])
def test_blend_all_pairs_through_contrast(factor):
    # image k: grey levels s = 0..255 then padding at k, so that the contrast mean int(mean(L) + 0.5) is k:
    # every (d, s) pair of Image.blend in one launch
    n = 256 * 256
    imgs = np.empty((256, 256, 256, 3), np.uint8)
    for k in range(256):
        flat = np.full((n, 3), k, np.uint8)
        flat[:256] = np.arange(256, dtype=np.uint8)[:, None]
        imgs[k] = flat.reshape(256, 256, 3)
    got = _jitter(imgs, [([CON], (1, factor, 1), 0)] * 256)
    for k in range(256):
        im = Image.fromarray(imgs[k])
        assert int(np.asarray(im.convert("L")).mean() + 0.5) == k
        want = np.asarray(ImageEnhance.Contrast(im).enhance(factor))
        assert np.array_equal(got[k], want), (k, factor)


def test_jitter_ops_and_random_orders():
    rng = np.random.RandomState(5)
    imgs = rng.randint(0, 256, (24, 96, 80, 3)).astype(np.uint8)
    imgs[:4] = (imgs[:4] // 64) * 64                                   # flat regions, grey pixels
    imgs[4:6, ..., 1] = imgs[4:6, ..., 0]
    rows, wants = [], []
    for k in range(24):
        g = torch.Generator().manual_seed(k)
        order = torch.randperm(4, generator=g).tolist()[: (k % 4) + 1] if k < 20 else [[BRI], [CON], [SAT], [HUE]][k - 20]
        b, c, s = (float(torch.empty(1).uniform_(lo, hi, generator=g)) for lo, hi in ((0.6, 1.4), (0.6, 1.4), (0.8, 1.2)))
        hf = float(torch.empty(1).uniform_(-0.1, 0.1, generator=g))
        im = Image.fromarray(imgs[k])
        for op in order:
            im = [lambda x: F.adjust_brightness(x, b), lambda x: F.adjust_contrast(x, c),
                  lambda x: F.adjust_saturation(x, s), lambda x: F.adjust_hue(x, hf)][op](im)
        rows.append((order, (b, c, s), int(hf * 255)))
        wants.append(np.asarray(im))
    got = _jitter(imgs, rows)
    for k in range(24):
        assert np.array_equal(got[k], wants[k]), (k, rows[k])


def _crop_table(srcs, boxes, modes, flips, S):
    tab, blob, off, tmp, KP, rows = [], [], 0, 0, 5, 1
    for a, (i, j, h, w), m, f in zip(srcs, boxes, modes, flips):
        tab.append([off & 0xFFFFFFFF, off >> 32, a.shape[0], a.shape[1], i, j, h, w, m, f, tmp & 0xFFFFFFFF, tmp >> 32])
        blob.append(a.reshape(-1))
        off += a.size
        tmp += max(h, w) * S * 3
        KP = max(KP, 2 * int(np.ceil(2 * max(h / S, w / S, 1.0))) + 1)
        rows = max(rows, h, w)
    return np.concatenate(blob), tab, tmp, KP, rows


def _resized_crop_dev(srcs, boxes, modes, flips, S=448):
    L, check = _lib()
    blob, tab, tmp, KP, rows = _crop_table(srcs, boxes, modes, flips, S)
    J = len(srcs)
    src = torch.from_numpy(blob).cuda()
    t = torch.tensor(tab, dtype=torch.int32).cuda()
    coef = torch.empty(J, 2, S, KP, dtype=torch.int32, device="cuda")
    bounds = torch.empty(J, 2, S, 2, dtype=torch.int32, device="cuda")
    tmpb = torch.empty(max(tmp, 1), dtype=torch.uint8, device="cuda")
    dst = torch.empty(J, S, S, 3, dtype=torch.uint8, device="cuda")
    check(L.pk_aug_resized_crop(_p(src), _p(t), J, S, KP, rows, _p(coef), _p(bounds), _p(tmpb), _p(dst), _st()), "crop")
    return dst.cpu().numpy()


def test_resized_crop_matches_pil():
    rng = np.random.RandomState(11)
    srcs, boxes, modes, flips = [], [], [], []
    for k in range(240):
        H, W = int(rng.randint(1, 1200)), int(rng.randint(1, 1200))
        if k % 9 == 4:
            W = int(rng.randint(1, 12))                               # around the pass-order switch
        if k % 40 == 0:
            H, W = 448, 448
        a = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
        if k % 40 == 0:
            i, j, h, w = 0, 0, 448, 448                               # Pillow's copy shortcut
        elif k % 40 in (2, 3):
            # tall and narrow: Pillow takes the vertical pass first when h > S and h > 100 w
            H, W = [(1001, 10), (1000, 10), (449, 4), (449, 5), (440, 2), (1300, 3)][(k // 40) % 6]
            a = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
            i, j, h, w = 0, 0, H, W
        elif k % 40 == 1:
            h, w = int(rng.randint(1, H + 1)), 1                      # one pixel wide
            i, j = int(rng.randint(0, H - h + 1)), int(rng.randint(0, W))
        else:
            h, w = int(rng.randint(1, H + 1)), int(rng.randint(1, W + 1))
            i, j = int(rng.randint(0, H - h + 1)), int(rng.randint(0, W - w + 1))
        srcs.append(a)
        boxes.append((i, j, h, w))
        modes.append(k % 3 == 2 and k % 40 not in (2, 3))
        flips.append(k % 2)
    got = _resized_crop_dev(srcs, boxes, [int(m) for m in modes], flips)
    for k, (a, (i, j, h, w), m, f) in enumerate(zip(srcs, boxes, modes, flips)):
        im = F.resized_crop(Image.fromarray(a), i, j, h, w, [448, 448], IM.NEAREST if m else IM.BICUBIC)
        if f:
            im = F.hflip(im)
        want = np.asarray(im)
        assert np.array_equal(got[k], want), (k, a.shape, (i, j, h, w), m, int((got[k] != want).sum()))


def test_second_crop_matches_torch_cpu():
    from torchvision.transforms import RandomResizedCrop
    L, check = _lib()
    torch.manual_seed(0)
    B, OH, OW = 12, 896, 448
    img = torch.randn(B, 3, OH, OW)
    tgt = torch.randn(B, 3, OH, OW)
    rows, want_i, want_t = [], [], []
    for b in range(B):
        box = RandomResizedCrop.get_params(img[b], (0.3, 1.0), (0.3, 0.7)) if b < B - 2 else (0, 0, OH, OW)
        m1, m2 = (b % 3 == 1), (b % 2 == 1)
        if b == B - 1:
            m1 = m2 = True                                             # the pass-through form: full box, nearest
        rows += [[*box, int(m1)], [*box, int(m2)]]
        want_i.append(F.resized_crop(img[b], *box, [OH, OW], IM.NEAREST if m1 else IM.BICUBIC, antialias=True))
        want_t.append(F.resized_crop(tgt[b], *box, [OH, OW], IM.NEAREST if m2 else IM.BICUBIC, antialias=True))
    di, dt = img.cuda(), tgt.cuda()
    oi, ot = torch.empty_like(di), torch.empty_like(dt)
    t = torch.tensor(rows, dtype=torch.int32).cuda()
    wts = torch.empty(2 * B, 2, OH, 5, device="cuda")
    bnd = torch.empty(2 * B, 2, OH, 2, dtype=torch.int32, device="cuda")
    tmp = torch.empty(2 * B, 3, OH, OW, device="cuda")
    check(L.pk_aug_second_crop(_p(di), _p(dt), _p(t), B, OH, OW, _p(wts), _p(bnd), _p(tmp), _p(oi), _p(ot), _st()),
          "second crop")
    for b in range(B):
        assert torch.equal(oi[b].cpu(), want_i[b]), (b, rows[2 * b])
        assert torch.equal(ot[b].cpu(), want_t[b]), (b, rows[2 * b + 1])
    assert torch.equal(oi[B - 1].cpu(), img[B - 1])


def _reference_batches(ref, idx, seed):
    torch.manual_seed(seed)
    random.seed(seed)
    np.random.seed(seed)
    items = [ref[i] for i in idx]
    return torch.utils.data.default_collate(items)


def _device_batch(ours, idx, seed, aug):
    from painter_b200.data_gpu import pair_collate
    torch.manual_seed(seed)
    random.seed(seed)
    np.random.seed(seed)
    return [t.cpu() for t in aug(pair_collate([ours[i] for i in idx]))]


@pytest.mark.parametrize("train", [True, False])
def test_end_to_end_bit_identical(tmp_path, train):
    from painter_b200.data_gpu import DevicePairAugment, DevicePairDataset
    lists = write_dataset(str(tmp_path), per_type=3)
    with contextlib.redirect_stdout(io.StringIO()):
        ref = reference_dataset(str(tmp_path), lists, train=train, half_mask_ratio=0.25, mask_generator=mask_generator())
    ours = DevicePairDataset(str(tmp_path), lists, input_size=(896, 448), min_random_scale=0.3, half_mask_ratio=0.25,
                             masked_position_generator=mask_generator(), train=train)
    aug = DevicePairAugment("cuda")
    n = len(ref)
    for step, seed in enumerate(range(3 if train else 1)):
        idx = [(k * 7 + step) % n for k in range(n)]
        for lo in range(0, n, 8):
            want = _reference_batches(ref, idx[lo:lo + 8], seed * 100 + lo)
            got = _device_batch(ours, idx[lo:lo + 8], seed * 100 + lo, aug)
            for name, w, g in zip(("samples", "targets", "masks", "valid"), want, got):
                assert w.dtype == g.dtype and w.shape == g.shape, name
                bad = (w != g).reshape(w.shape[0], -1).any(1)
                assert not bad.any(), (name, [ours.pairs[idx[lo + int(b)]]["type"] for b in bad.nonzero()])


def _worker_init(wid):
    s = torch.initial_seed() % 2 ** 32
    random.seed(s)
    np.random.seed(s)


def test_dataloader_two_workers(tmp_path):
    from painter_b200.data_gpu import DevicePairDataset, DevicePairPrefetcher, pair_collate
    lists = write_dataset(str(tmp_path), per_type=2)
    with contextlib.redirect_stdout(io.StringIO()):
        ref = reference_dataset(str(tmp_path), lists, train=True, half_mask_ratio=0.25, mask_generator=mask_generator())
    ours = DevicePairDataset(str(tmp_path), lists, half_mask_ratio=0.25, masked_position_generator=mask_generator())
    kw = dict(batch_size=4, num_workers=2, worker_init_fn=_worker_init, shuffle=False)
    want = torch.utils.data.DataLoader(ref, generator=torch.Generator().manual_seed(7), **kw)
    got = DevicePairPrefetcher(torch.utils.data.DataLoader(ours, generator=torch.Generator().manual_seed(7),
                                                           collate_fn=pair_collate, pin_memory=True, **kw))
    n = 0
    for w, g in zip(want, got):              # the prefetcher reuses two buffer sets: compare each batch on arrival
        for name, a, b in zip(("samples", "targets", "masks", "valid"), w, g):
            assert torch.equal(a, b.cpu()), (n, name)
        n += 1
    assert n == len(ref) // 4
