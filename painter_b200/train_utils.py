"""The optimizer recipe around the hot path (SURVEY §8 f.1), restated for painter_b200 modules:

  param_groups_lrd       Painter/util/lr_decay.py:15-76   layer-wise lr decay groups (BEiT rule), same group order
  adjust_learning_rate   Painter/util/lr_sched.py:9-21    half-cycle cosine after linear warm-up, per iteration
  FusedStep              Painter/util/misc.py:252-278      NativeScalerWithGradNormCount.__call__ (unscale -> clip ->
                                                           step) for FusedAdamW: the global gradient norm is one launch
                                                           over the flat arena, the clip coefficient stays on the device
                                                           and rides into the AdamW kernel - no host sync in the step
  GraphedTrainStep       Painter/engine_train.py:58-93     forward + backward + optimizer update of one iteration as
                                                           ONE CUDA graph replay
"""
import math

import torch

from .optim import FusedAdamW, global_grad_norm


def layer_id_for_vit(name, num_layers):
    """lr_decay.get_layer_id_for_vit (:64-76)."""
    if name in ("cls_token", "pos_embed"):
        return 0
    if name.startswith("patch_embed"):
        return 0
    if name.startswith("blocks"):
        return int(name.split(".")[1]) + 1
    return num_layers


def param_groups_lrd(model, weight_decay=0.05, no_weight_decay_list=(), layer_decay=0.75):
    """Groups {lr_scale, weight_decay, params} exactly as the reference builds them (same keys, same order)."""
    num_layers = len(model.blocks) + 1
    scales = [layer_decay ** (num_layers - i) for i in range(num_layers + 1)]
    groups = {}
    for n, p in model.named_parameters():
        if not p.requires_grad:
            continue
        if p.ndim == 1 or n in no_weight_decay_list:
            tag, wd = "no_decay", 0.0
        else:
            tag, wd = "decay", weight_decay
        lid = layer_id_for_vit(n, num_layers)
        key = "layer_%d_%s" % (lid, tag)
        if key not in groups:
            groups[key] = {"lr_scale": scales[lid], "weight_decay": wd, "params": []}
        groups[key]["params"].append(p)
    return list(groups.values())


def adjust_learning_rate(optimizer, epoch, lr, min_lr=0.0, warmup_epochs=0, epochs=1):
    """lr_sched.adjust_learning_rate with explicit arguments instead of the argparse namespace."""
    if epoch < warmup_epochs:
        cur = lr * epoch / warmup_epochs
    else:
        cur = min_lr + (lr - min_lr) * 0.5 * (1.0 + math.cos(math.pi * (epoch - warmup_epochs) /
                                                              (epochs - warmup_epochs)))
    for g in optimizer.param_groups:
        g["lr"] = cur * g["lr_scale"] if "lr_scale" in g else cur
    return cur


class FusedStep:
    """loss -> backward -> (clip) -> FusedAdamW.step, the sequence of misc.NativeScalerWithGradNormCount.__call__
    without a loss scale (the module computes in bf16 operands / fp32 accumulate whatever the autocast dtype, so
    gradients cannot overflow the way fp16 ones do).  Returns the gradient norm as a 0-dim DEVICE tensor."""

    def __init__(self, optimizer: FusedAdamW):
        self.opt = optimizer

    def __call__(self, loss, clip_grad=None, parameters=None, update_grad=True):
        loss.backward()
        if not update_grad:
            return None
        params = list(parameters) if parameters is not None else [p for g in self.opt.param_groups for p in g["params"]]
        norm = global_grad_norm(params)
        if clip_grad is not None:
            coef = (clip_grad / (norm + 1e-6)).reshape(1).float()      # clip_grad_norm_: min(1, max_norm / (norm + 1e-6))
            self.opt.step(grad_scale=coef, grad_scale_cap=1.0)
        else:
            self.opt.step()
        return norm


class GraphedTrainStep:
    """One training iteration (`engine_train.py:58-93`: autocast forward, `loss.backward()`, optimizer update) captured
    into a CUDA graph and replayed: ~800 kernel launches per step become one `cudaGraphLaunch`, the launch gaps between
    kernels close and, with programmatic dependent launch, each kernel's prologue overlaps its predecessor's tail.

        step = GraphedTrainStep(model, optimizer)          # optimizer: painter_b200.optim.FusedAdamW
        for samples, targets, bool_masked_pos, valid in loader:
            adjust_learning_rate(optimizer, ...)             # per-iteration schedules keep working (see below)
            loss = step(samples, targets, bool_masked_pos, valid)     # 0-dim device tensor (static buffer)

    A SegGPT module takes its per-sample seg types as a fifth input, `step(samples, targets, bool_masked_pos, valid,
    seg_type)` ([B, 1]: 0 semantic, 1 instance); they get a static buffer like the other inputs, so every replay
    reads the current batch's types.

    What makes the step capture-safe: gradients live in the module's flat arena (static addresses, zeroed by the
    optimizer kernel), the bf16 operand copies are refreshed by the optimizer kernel, DropPath draws come from the
    graph-registered CUDA generator, and everything that changes from one iteration to the next - learning rates,
    weight decays, Adam's step count - is data in device memory that `FusedAdamW.graph_prepare()` rewrites in place
    before the replay.  The first call with a new input shape runs `warmup` eager iterations on a side stream to
    populate caches and allocator pools; parameters, optimizer state and the CUDA RNG state are snapshotted before
    and restored after, so the first replay is the first real iteration.  Gradient clipping / loss scaling are not
    part of the captured step (use `FusedStep` for those recipes)."""

    def __init__(self, model, optimizer, warmup=2, autocast_dtype=torch.bfloat16):
        if not isinstance(optimizer, FusedAdamW):
            raise TypeError("GraphedTrainStep needs painter_b200.optim.FusedAdamW")
        self.model, self.opt, self.warmup, self.dtype = model, optimizer, warmup, autocast_dtype
        self.seggpt = getattr(model, "seggpt", False)
        self.entries = {}

    def _eager(self, si):
        kw = {"seg_type": si[4]} if self.seggpt else {}
        with torch.autocast("cuda", dtype=self.dtype):
            loss, _, _ = self.model(si[0], si[1], bool_masked_pos=si[2], valid=si[3], **kw)
        loss.backward()
        return loss

    def _capture(self, inputs):
        dev = next(self.model.parameters()).device
        si = [t.detach().to(dev, copy=True) for t in inputs]
        params = [p for g in self.opt.param_groups for p in g["params"]]
        # snapshot everything the warm-up iterations change
        with torch.no_grad():
            saved_p = [p.detach().clone() for p in params]
        saved_state = {id(p): {k: (v.clone() if torch.is_tensor(v) else v) for k, v in self.opt.state.get(p, {}).items()}
                       for p in params}
        rng = torch.cuda.get_rng_state(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(1, self.warmup)):
                self.opt.zero_grad(set_to_none=True)
                self._eager(si)
                self.opt.graph_prepare()
                self.opt.graph_launch()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.opt.zero_grad(set_to_none=True)       # the captured backward hands its arena views to autograd afresh
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            loss = self._eager(si)
            self.opt.graph_launch()
            out = loss.detach()
        # restore: the warm-up never happened
        with torch.no_grad():
            for p, q in zip(params, saved_p):
                p.copy_(q)
                ent = getattr(p, "_pk_bf16", None)
                if ent is not None and ent[1] == p.data_ptr():
                    # the bf16 operand copy (zero-padded for the rel-pos tables) follows the parameter, in place:
                    # the graph reads this very tensor
                    ent[2].view(-1)[:q.numel()].copy_(q.reshape(-1))
                    p._pk_bf16 = (p._version, p.data_ptr(), ent[2])
        for p in params:
            st, old = self.opt.state.get(p), saved_state[id(p)]
            if st is None:
                continue
            if not old:
                st["step"] = 0
                st["exp_avg"].zero_()
                st["exp_avg_sq"].zero_()
            else:
                for k, v in old.items():
                    if torch.is_tensor(v) and torch.is_tensor(st.get(k)):
                        st[k].copy_(v)
                    else:
                        st[k] = v
        torch.cuda.set_rng_state(rng, dev)
        self.opt.zero_grad(set_to_none=True)   # gradients are produced and consumed inside the graph (arena slots)
        torch.cuda.synchronize(dev)
        return si, g, out

    def __call__(self, imgs, tgts, bool_masked_pos, valid, seg_type=None):
        # inputs may live on the device or in (pinned) host memory: they are copied into the graph's static buffers
        if self.seggpt != (seg_type is not None):
            raise ValueError("GraphedTrainStep: seg_type is required for a SegGPT module and not accepted otherwise")
        inputs = (imgs, tgts, bool_masked_pos, valid) + ((seg_type,) if seg_type is not None else ())
        key = (tuple(imgs.shape), imgs.dtype, tuple(bool_masked_pos.shape), bool_masked_pos.dtype, tuple(valid.shape),
               None if seg_type is None else (tuple(seg_type.shape), seg_type.dtype))
        ent = self.entries.get(key)
        if ent is None:
            if len(self.entries) > 4:
                self.entries.clear()
            ent = self.entries[key] = self._capture(inputs)
        si, g, out = ent
        for buf, t in zip(si, inputs):
            buf.copy_(t, non_blocking=True)
        self.opt.graph_prepare()
        g.replay()
        return out
