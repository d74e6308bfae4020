"""World-size-2 gloo (CPU) checks of the data-parallel host logic: per-rank data seeds, max-over-ranks timing,
gradient averaging == DDP == mean of the per-rank gradients (computed with the tiny oracle model)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import painter_oracle as po
    from oracle.synth import synth_inputs, synth_state_dict
    from painter_b200 import dist_utils as du
    cfg = po.PainterConfig(img_size=(64, 32), embed_dim=64, num_heads=1, decoder_embed_dim=64)
    sd = {k: v.clone().requires_grad_(True) for k, v in synth_state_dict(cfg, 0).items()}
    seed = du.rank_seed(1234, rank)
    imgs, tgts, mask, valid = synth_inputs(cfg, 2, seed)
    loss, _, _ = po.forward(sd, cfg, imgs, tgts, mask, valid)
    loss.backward()
    local = {k: v.grad.clone() for k, v in sd.items()}
    du.average_gradients(list(sd.values()))
    # gather every rank's local gradient of one tensor and compare with the averaged one
    key = "blocks.3.attn.qkv.weight"
    gl = [torch.zeros_like(local[key]) for _ in range(world)]
    dist.all_gather(gl, local[key])
    want = sum(gl) / world
    err = (sd[key].grad - want).abs().max().item()
    tmax = du.max_over_ranks([float(rank + 1), 10.0 - rank])
    if rank == 0:
        torch.save(dict(err=err, tmax=tmax, seeds=[du.rank_seed(1234, r) for r in range(world)],
                        differ=bool((gl[0] - gl[1]).abs().max() > 0)), out)
    dist.barrier()
    dist.destroy_process_group()


def test_gloo_world2_gradient_average_and_timing(tmp_path):
    out = str(tmp_path / "res.pt")
    mp.spawn(_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    r = torch.load(out)
    assert r["err"] < 1e-7
    assert r["tmax"] == [2.0, 10.0]
    assert len(set(r["seeds"])) == 2 and r["differ"]      # ranks really process different batches


def _tiny_module(seggpt=False):
    from functools import partial
    from painter_b200 import models_painter, models_seggpt
    torch.manual_seed(0)
    cls = models_seggpt.SegGPT if seggpt else models_painter.Painter
    return cls(img_size=(64, 32), embed_dim=64, num_heads=1, decoder_embed_dim=64, use_rel_pos=True, depth=24,
               norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def _sync_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from painter_b200.arena import get_arena
    from painter_b200.dist_utils import GradSync
    m = _tiny_module()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(float(rank))               # ranks start different: GradSync must broadcast rank 0's weights
    sync = GradSync(m, bucket_mb=0.2)
    arena = get_arena(m)
    same = all(bool((p - q).abs().max() == 0) for p, q in zip(m.parameters(), _tiny_module().parameters()))
    # drive the arena protocol the way the backward stages do (the CUDA kernels are replaced by plain fills)
    results = []
    for micro in range(2):                    # second pass = gradient accumulation (p.grad already set)
        tok = object()
        assert arena.begin_backward(tok)
        grads = {}
        for name, a, b in arena.group_ranges:
            for p in arena.params:
                off, n, _ = arena.offsets[id(p)]
                if a <= off < b:
                    v = arena.view(p)
                    v.fill_(float(rank + 1) * (micro + 1) + off % 7)
                    grads[id(p)] = v
            arena.stage_done(name)
        arena.end_backward()
        for p in arena.params:                # what autograd's AccumulateGrad does with the returned views
            if p.grad is None:
                p.grad = grads[id(p)]
            else:
                p.grad += grads[id(p)]
        results.append([p.grad.clone() for p in arena.params])
    errs = []
    for micro, res in enumerate(results):
        for p, g in zip(arena.params, res):
            off = arena.offsets[id(p)][0]
            want = sum(((1 + 2) / 2.0) * (k + 1) + off % 7 for k in range(micro + 1))
            errs.append((g - want).abs().max().item())
    if rank == 0:
        torch.save(dict(err=max(errs), same=same, nb=len(sync.buckets), in_arena=arena.grads_in_arena(),
                        total=arena.total, covered=sync.buckets[-1][1], first=sync.buckets[0][0]), out)
    dist.barrier()
    dist.destroy_process_group()


def test_gloo_world2_gradsync_buckets_average_the_arena(tmp_path):
    """dist_utils.GradSync (own bucketed all-reduce, replaces the DDP reducer of main_train.py:340): parameters
    broadcast from rank 0, every arena bucket averaged over ranks, gradient accumulation through the scratch slab."""
    out = str(tmp_path / "res.pt")
    mp.spawn(_sync_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    r = torch.load(out)
    assert r["same"] and r["err"] < 1e-6 and r["nb"] > 2 and r["in_arena"]
    assert r["first"] == 0 and r["covered"] == r["total"]


def test_arena_layout_follows_backward_production_order():
    from painter_b200.arena import GradArena
    from painter_b200.dist_utils import GradSync
    m = _tiny_module()
    a = GradArena(m)
    names = [g[0] for g in a.group_ranges]
    assert names == ["decoder"] + [f"block{i}" for i in range(23, -1, -1)] + ["embed"]
    assert all(a.offsets[id(p)][0] % GradArena.ALIGN == 0 for p in m.parameters())
    assert a.total >= sum(p.numel() for p in m.parameters())
    spans = sorted((a.offsets[id(p)][0], a.offsets[id(p)][0] + p.numel()) for p in m.parameters())
    assert all(s1[1] <= s2[0] for s1, s2 in zip(spans, spans[1:]))          # no overlap
    b = GradSync.plan(a.group_ranges, 0.05)
    assert b[0][0] == 0 and b[-1][1] == a.total and all(x[1] == y[0] for x, y in zip(b, b[1:]))


BLOCK_PARAMS = ("norm1.weight", "norm1.bias", "attn.rel_pos_h", "attn.rel_pos_w", "attn.qkv.weight", "attn.qkv.bias",
                "attn.proj.weight", "attn.proj.bias", "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias",
                "mlp.fc2.weight", "mlp.fc2.bias")


@pytest.mark.parametrize("seggpt", [False, True])
def test_arena_slab_layout_is_pinned(seggpt):
    """Every parameter's offset and every group's range in the gradient slab, spelled out by parameter name: GradSync
    buckets and FusedAdamW chunks are cut along them."""
    from painter_b200.arena import GradArena
    m = _tiny_module(seggpt)
    groups = [("decoder", ["norm.weight", "norm.bias", "decoder_embed.weight", "decoder_embed.bias",
                           "decoder_pred.0.weight", "decoder_pred.0.bias", "decoder_pred.1.weight",
                           "decoder_pred.1.bias", "decoder_pred.3.weight", "decoder_pred.3.bias"])]
    groups += [(f"block{i}", [f"blocks.{i}.{n}" for n in BLOCK_PARAMS]) for i in range(23, -1, -1)]
    groups.append(("embed", ["patch_embed.proj.weight", "patch_embed.proj.bias", "mask_token", "segment_token_x",
                             "segment_token_y"] + (["type_token_cls", "type_token_ins"] if seggpt else []) +
                   ["pos_embed"]))
    prm = dict(m.named_parameters())
    assert sorted(prm) == sorted(n for _, names in groups for n in names)
    want_offsets, want_ranges, off = {}, [], 0
    for name, names in groups:
        start = off
        for n in names:
            want_offsets[n] = off
            off += -(-prm[n].numel() // 64) * 64
        want_ranges.append((name, start, off))
    a = GradArena(m)
    assert a.group_ranges == want_ranges
    assert {n: a.offsets[id(p)][0] for n, p in prm.items()} == want_offsets
    assert a.total == off == (5525248 if seggpt else 5525120)
