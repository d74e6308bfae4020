"""Batched task inference (painter_inference.run_batch, seggpt_engine.segment_batch / inference_images) against the
per-image mirrors, bit for bit.

The mirrors are pinned to the unmodified reference functions (test_gpu_inference.py, test_gpu_painter_tasks.py), so
equality with them carries that parity over.  Equality holds because no forward computation mixes samples in a way
that depends on the batch size (forward GEMMs never split K, attention is per (sample, head), LayerNorm per row, the
fp32-accurate decoder runs one image at a time, the prompt ensemble averages over one query's own members) and every
image of a finishing launch gets the same per-pixel code.  Everything runs at the full 896 x 448
geometry with seeded random weights, in the fp32-accurate mode ("auto" under no_grad, what the mirrors select) and in
bf16."""
import numpy as np
import pytest
import torch

from oracle import painter_oracle as po

from _common import build_model

pytestmark = pytest.mark.gpu

PRECISIONS = ["auto", "bf16"]
# (width, height): up- and down-scaling, odd sizes, OH + OW = 110 and 129 (either side of torch-CPU's channels-last
# switch at 128), and a source under 16 px on a side
SIZES = [(640, 427), (301, 523), (60, 50), (71, 58), (13, 9)]
TASKS = {"segm": "run_one_image", "nearest": "run_one_image_nearest", "depth": "run_one_image_depth",
         "restore": "run_one_image_restore"}


def _drop_graphs(*models):
    for m in models:
        m.__dict__.pop("_pk_graphed", None)
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def painter():
    model, _ = build_model(po.PainterConfig(), 1)
    model.eval()
    yield model
    _drop_graphs(model)


@pytest.fixture(scope="module")
def seggpt():
    model, _ = build_model(po.PainterConfig(seggpt=True), 3)
    model.eval()
    model.seg_type = "instance"
    yield model
    _drop_graphs(model)


@pytest.fixture(autouse=True)
def _fresh_graphs(request):
    # captured graphs keep their memory pools: an fp32-accurate batch's pool is several GB
    yield
    for name in ("painter", "seggpt"):
        if name in request.fixturenames:
            _drop_graphs(request.getfixturevalue(name))


class Wrapped(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.module = m


def _canvases(n, seed):
    rng = np.random.RandomState(seed)
    return [rng.randn(896, 448, 3) for _ in range(n)], [rng.randn(896, 448, 3) for _ in range(n)]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("task", list(TASKS))
def test_run_batch_equals_per_image_mirror(painter, task, precision, tmp_path):
    from painter_b200 import painter_inference as pi
    painter.precision = precision
    try:
        imgs, tgts = _canvases(len(SIZES), seed=len(task))
        dev = torch.device("cuda")
        model = Wrapped(painter) if task == "nearest" else painter
        single = []
        for b, size in enumerate(SIZES):
            single.append(getattr(pi, TASKS[task])(imgs[b], tgts[b], size, model, str(tmp_path / f"one{b}.png"), dev))
        paths = [str(tmp_path / f"batch{b}.png") for b in range(len(SIZES))]
        batch = pi.run_batch(imgs, tgts, SIZES, model, dev, task, out_paths=paths)
    finally:
        painter.precision = "bf16"
    assert len(batch) == len(SIZES)
    for b, (a, o) in enumerate(zip(single, batch)):
        if task == "restore":
            assert isinstance(o, np.ndarray) and o.dtype == a.dtype == np.float64 and o.shape == a.shape
            assert np.array_equal(a, o), (b, np.abs(a - o).max())
        else:
            assert a.dtype == o.dtype and a.shape == o.shape and torch.equal(a, o), (b, SIZES[b])
            assert open(tmp_path / f"one{b}.png", "rb").read() == open(paths[b], "rb").read(), b


@pytest.mark.parametrize("precision", PRECISIONS)
def test_prediction_is_batch_invariant(painter, precision):
    """A sample's patchified prediction is the same at B = 1, 3 and 8, and as a member of a padded tail batch."""
    from painter_b200.seggpt_engine import _graphed
    painter.precision = precision
    try:
        g = _graphed(painter)
        x, t = torch.randn(2, 8, 3, 896, 448, device="cuda").unbind(0)
        n = painter.patch_embed.num_patches
        mask = torch.zeros(1, n, device="cuda")
        mask[:, n // 2:] = 1

        def pred(xx, tt):
            with torch.no_grad():
                return g(xx, tt, mask, torch.ones_like(tt))[1].clone()

        y8 = pred(x, t)
        y3 = pred(x[:3], t[:3])
        y1 = pred(x[2:3], t[2:3])
        pad = torch.cat([x[:3], x[2:3]]), torch.cat([t[:3], t[2:3]])
        y4 = pred(*pad)
    finally:
        painter.precision = "bf16"
    assert torch.equal(y8[:3], y3)
    assert torch.equal(y8[2], y1[0]) and torch.equal(y3[2], y1[0])
    assert torch.equal(y4[:3], y3) and torch.equal(y4[3], y3[2])


def _prompts(P, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, 256, (448, 448, 3), generator=g, dtype=torch.uint8).cuda(),
             torch.randint(0, 256, (448, 448, 3), generator=g, dtype=torch.uint8).cuda()) for _ in range(P)]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("Q,P", [(4, 3), (4, 1)])
def test_segment_batch_equals_segment(seggpt, Q, P, precision):
    from painter_b200 import seggpt_engine as se
    seggpt.precision = precision
    try:
        prompts = _prompts(P, seed=Q * 10 + P)
        queries = torch.randint(0, 256, (Q, 448, 448, 3), dtype=torch.uint8, device="cuda")
        one = [se.segment(seggpt, "cuda", queries[q], prompts, want_bin=True) for q in range(Q)]
        one = [(o.clone(), b.clone()) for o, b in one]
        out, binm = se.segment_batch(seggpt, "cuda", queries, prompts, want_bin=True)
    finally:
        seggpt.precision = "bf16"
    assert out.shape == (Q, 448, 448, 3) and binm.shape == (Q, 448, 448)
    for q in range(Q):
        assert torch.equal(out[q], one[q][0]), (q, (out[q] - one[q][0]).abs().max())
        assert torch.equal(binm[q], one[q][1]), q


def test_segment_batch_more_than_16_members(seggpt):
    """Q x P = 18 members: the stitching launches in chunks, nothing is refused or truncated."""
    from painter_b200 import seggpt_engine as se
    Q, P = 6, 3
    prompts = _prompts(P, seed=5)
    queries = torch.randint(0, 256, (Q, 448, 448, 3), dtype=torch.uint8, device="cuda")
    x = se.stitch_normalize([p[0] for _ in range(Q) for p in prompts], [q for q in queries for _ in prompts], 448)
    for m in (0, 16, 17):
        ref = se.stitch_normalize([prompts[m % P][0]], [queries[m // P]], 448)
        assert torch.equal(x[m], ref[0]), m
    one = [se.segment(seggpt, "cuda", queries[q], prompts)[0].clone() for q in range(Q)]
    out, _ = se.segment_batch(seggpt, "cuda", queries, prompts)
    for q in range(Q):
        assert torch.equal(out[q], one[q]), q


def test_inference_images_writes_the_same_files(seggpt, tmp_path):
    from PIL import Image
    from painter_b200 import seggpt_engine as se
    rng = np.random.RandomState(4)
    sizes = [(640, 480), (301, 523), (448, 448), (97, 60), (500, 333)]
    qs = []
    for k, (w, h) in enumerate(sizes):
        qs.append(str(tmp_path / f"q{k}.png"))
        Image.fromarray(rng.randint(0, 256, (h, w, 3), dtype=np.uint8)).save(qs[-1])
    p_img, p_tgt = [], []
    for k in range(2):
        p_img.append(str(tmp_path / f"p{k}.png"))
        p_tgt.append(str(tmp_path / f"t{k}.png"))
        Image.fromarray(rng.randint(0, 256, (400, 520, 3), dtype=np.uint8)).save(p_img[-1])
        Image.fromarray((rng.rand(400, 520, 1) > 0.5).astype(np.uint8).repeat(3, 2) * 255).save(p_tgt[-1])
    one = [str(tmp_path / f"one{k}.png") for k in range(len(sizes))]
    many = [str(tmp_path / f"many{k}.png") for k in range(len(sizes))]
    for q, o in zip(qs, one):
        se.inference_image(seggpt, "cuda", q, p_img, p_tgt, o)
    se.inference_images(seggpt, "cuda", qs, p_img, p_tgt, many, batch_size=2)
    for a, b in zip(one, many):
        assert open(a, "rb").read() == open(b, "rb").read(), b


def test_ragged_launch_equals_one_image_launches():
    """Each image of one n-image pk_finish_ragged launch equals, bit for bit, a one-row launch of that image alone
    (its source sample as the only one, output at offset 0): the rows' source samples, output offsets and per-row
    cl_form are addressed right.  Likewise each sample of a strided pk_denorm_bottom_batched launch, mask included."""
    from painter_b200 import painter_inference as pi
    from painter_b200 import seggpt_engine as se
    torch.manual_seed(0)
    B, S = 3, 448
    src = (torch.rand(B, S, S, 3, dtype=torch.float64, device="cuda") * 255.0).contiguous()
    depth_src = (torch.rand(B, S, S, 3, dtype=torch.float64, device="cuda") * 10000.0).contiguous()
    sizes = [(427, 640), (523, 301), (50, 60), (58, 71), (9, 13), (448, 448), (896, 896)]    # (OH, OW)
    srcs = [k % B for k in range(len(sizes))]
    images = [torch.randint(0, 256, (oh, ow, 3), dtype=torch.uint8, device="cuda") for oh, ow in sizes]
    ops = {    # op -> (source, torch-CPU's cl_form for an output size)
        se.FIN_BILINEAR_U8: (src, lambda oh, ow: 0),
        se.FIN_NEAREST_U8: (src, lambda oh, ow: int(oh + ow <= 128)),
        se.FIN_DEPTH: (depth_src, lambda oh, ow: int(torch.get_num_threads() == 1 or oh + ow <= 128)),
        se.FIN_BICUBIC_F64: (src, lambda oh, ow: 0),
        se.FIN_NEAREST_BLEND: (src, lambda oh, ow: 0),
    }
    for op, (base, cl) in ops.items():
        blend = op == se.FIN_NEAREST_BLEND
        tab, offs, total, max_pix = se.ragged_table(op, srcs, sizes, [cl(oh, ow) for oh, ow in sizes])
        img = torch.cat([i.reshape(-1) for i in images]) if blend else None
        out = se.finish_ragged(op, base, torch.from_numpy(tab).cuda(), len(sizes), max_pix, total, image=img)
        for k, (oh, ow) in enumerate(sizes):
            tab1, _, total1, max_pix1 = se.ragged_table(op, [0], [(oh, ow)], [cl(oh, ow)])
            ref = se.finish_ragged(op, base[srcs[k]:srcs[k] + 1], torch.from_numpy(tab1).cuda(), 1, max_pix1, total1,
                                   image=images[k] if blend else None)
            assert torch.equal(out[offs[k]:offs[k] + total1], ref), (op, k, oh, ow)
    # strided batched de-normalisation (with the binarised mask) vs a one-sample launch on each sample
    p, h, w = 16, 56, 28
    patch = torch.randn(5, h * w, p * p * 3, device="cuda")
    for finish in (pi.CLIP255, pi.CLIP10000, pi.PLAIN):
        want_bin = finish == pi.CLIP255
        out, binm = se.denorm_bottom_batched(patch, 3, h, w, p, finish, src_stride=2, want_bin=want_bin)
        for b in range(3):
            ref, rbin = se.denorm_bottom_batched(patch[2 * b:2 * b + 1].contiguous(), 1, h, w, p, finish,
                                                 want_bin=want_bin)
            assert torch.equal(out[b], ref[0]), (finish, b)
            if want_bin:
                assert torch.equal(binm[b], rbin[0]), b


def test_tail_batch_replays_one_graph(painter, tmp_path):
    """11 images at batch 4: the tail of 3 is padded to 4, so one graph serves the whole set."""
    from painter_b200 import painter_inference as pi
    from painter_b200.seggpt_engine import _graphed
    imgs, tgts = _canvases(11, seed=11)
    sizes = [(300 + 7 * k, 200 + 5 * k) for k in range(11)]
    dev = torch.device("cuda")
    got = []
    for b0 in range(0, 11, 4):
        got += pi.run_batch(imgs[b0:b0 + 4], tgts[b0:b0 + 4], sizes[b0:b0 + 4], painter, dev, "segm")
    shapes = [k[0] for k in _graphed(painter).entries]
    assert shapes == [(4, 3, 896, 448)], shapes
    for k in range(11):
        ref = pi.run_one_image(imgs[k], tgts[k], sizes[k], painter, str(tmp_path / f"{k}.png"), dev)
        assert torch.equal(got[k], ref), k


def test_public_forward_still_ensembles_the_whole_batch(seggpt):
    """model(..., merge_between_batch=0) on 4 members averages over all 4 (the reference's meaning); the grouped
    forward of Q = 2 queries x P = 2 prompts differs from it and equals two separate P = 2 forwards."""
    torch.manual_seed(1)
    x, t = torch.randn(2, 4, 3, 896, 448, device="cuda").unbind(0)
    n = seggpt.patch_embed.num_patches
    mask = torch.zeros(4, n, dtype=torch.bool, device="cuda")
    mask[:, n // 2:] = True
    valid = torch.ones_like(t)
    st = torch.ones(4, 1, device="cuda")
    with torch.no_grad():
        _, plain, _ = seggpt(x, t, mask, valid, st, 0)
        _, whole = seggpt._run(x, t, mask, valid, st, 0, prompts_per_query=4)
        _, grouped = seggpt._run(x, t, mask, valid, st, 0, prompts_per_query=2)
        _, first, _ = seggpt(x[:2], t[:2], mask[:2], valid[:2], st[:2], 0)
        _, second, _ = seggpt(x[2:], t[2:], mask[2:], valid[2:], st[2:], 0)
    assert torch.equal(plain, whole)
    assert not torch.equal(plain, grouped)
    assert torch.equal(grouped[:2], first) and torch.equal(grouped[2:], second)
