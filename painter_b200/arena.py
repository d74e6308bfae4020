"""Flat fp32 gradient arena of a painter_b200 module.

Every parameter gradient of a training step is produced by exactly one backward stage (engine.py), so the stages
write them straight into ONE zero-initialised fp32 slab laid out in the order backward produces them
(decoder -> block 23 ... block 0 -> embedding), as the module's `grad_stages()` states it.  What that buys:

  * one memset per step instead of ~700 zero fills (stream-K weight-gradient GEMMs, LayerNorm / bias / rel-pos
    accumulators all need zero-initialised targets) - or none at all when `optim.FusedAdamW` clears each gradient as it
    consumes it;
  * `p.grad` is a VIEW of the slab (autograd steals the returned views), so the optimizer and the gradient norm run
    over one contiguous range and the data-parallel all-reduce (dist_utils.GradSync; replaces the DDP reducer of
    Painter/main_train.py:340) is issued per contiguous bucket as soon as the producing stages have been enqueued,
    with no copy into communication buffers.

Gradient accumulation (engine_train.py accum_iter > 1: backward called again while p.grad is set): the stages write
the micro-step's gradients into a second, scratch slab (zeroed first, all-reduced the same way) and autograd adds the
returned views into the live p.grad, exactly like a plain module.
"""
import weakref

import torch


class GradArena:
    ALIGN = 64  # floats: every view starts on a 256-byte boundary (vector stores, TMA-free epilogues, NCCL)

    def __init__(self, model):
        dev = next(model.parameters()).device
        self.device = dev
        groups = [(name, list(prm.values())) for name, prm in model.grad_stages().items()]   # production order
        self.offsets = {}
        self.group_ranges = []          # (name, start, end) in floats, production order
        off = 0
        seen = set()
        for name, params in groups:
            start = off
            for p in params:
                if id(p) in seen:
                    continue
                seen.add(id(p))
                self.offsets[id(p)] = (off, p.numel(), tuple(p.shape))
                off += (p.numel() + self.ALIGN - 1) // self.ALIGN * self.ALIGN
            self.group_ranges.append((name, start, off))
        missing = [n for n, p in model.named_parameters() if id(p) not in seen]
        if missing:
            raise RuntimeError(f"painter_b200.GradArena: parameters without a slot: {missing}")
        self.total = off
        self.slab = torch.zeros(off, dtype=torch.float32, device=dev)
        self.params = [p for _, ps in groups for p in ps]
        ref = weakref.ref(self)
        for p in self.params:
            p._pk_arena = ref          # lets optim.FusedAdamW find the arena from the parameters it steps
        self.scratch = None          # second slab for gradient-accumulation micro-steps
        self.cur = self.slab         # the slab the running backward writes into
        self.clean = True            # slab is all zeros
        self.active = False          # a backward is writing into `cur`
        self.sync = None             # dist_utils.GradSync, when data parallel
        self._step = None

    # ------------------------------------------------------------------ views
    def view(self, p):
        """Fresh view of p's gradient slot (a new tensor object every call, so autograd can steal it as p.grad)."""
        off, n, shape = self.offsets[id(p)]
        return self.cur[off:off + n].view(shape)

    def owns(self, p):
        return id(p) in self.offsets

    def grads_in_arena(self):
        lo, hi = self.slab.data_ptr(), self.slab.data_ptr() + self.total * 4
        return all(p.grad is not None and lo <= p.grad.data_ptr() < hi for p in self.params)

    # ------------------------------------------------------------------ step protocol
    def begin_backward(self, step_token):
        """Called by every backward stage; the first call of a step decides whether this backward may write into
        the slab (no gradient is live) and clears it if the previous step left values behind."""
        if self._step is step_token:
            return self.active
        self._step = step_token
        accumulating = any(p.grad is not None for p in self.params)
        self.active = True
        if accumulating:
            if self.scratch is None:
                self.scratch = torch.empty_like(self.slab)
            self.cur = self.scratch
            self.cur.zero_()
        else:
            self.cur = self.slab
            if not self.clean:
                self.slab.zero_()
            self.clean = False
        if self.sync is not None:
            self.sync.begin(self)
        return self.active

    def stage_done(self, group_name):
        """A backward stage has enqueued every kernel that writes its group of gradients."""
        if self.active and self.sync is not None:
            self.sync.stage_done(self, group_name)

    def end_backward(self):
        if self.active and self.sync is not None:
            self.sync.finish(self)

    def mark_clean(self):
        self.clean = True


def get_arena(model):
    """The module's arena (created on first use; rebuilt if the parameters moved to another device)."""
    a = getattr(model, "_pk_arena", None)
    dev = next(model.parameters()).device
    if a is None or a.device != dev or any(not a.owns(p) for p in model.parameters()):
        a = GradArena(model)
        model.__dict__["_pk_arena"] = a
    return a
