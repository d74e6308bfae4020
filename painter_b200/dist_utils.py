"""Host-side helpers of the multi-GPU (data-parallel) path, backend-agnostic so they can be exercised with gloo on
CPU.  The reference shards by batch only (DDP, Painter/main_train.py:340); each rank owns a replica, draws its own
samples (sampler seed offset by rank, main_train.py:228-270) and gradients are averaged by all-reduce."""
import os

import torch
import torch.distributed as dist


def world_info():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))


def rank_seed(base_seed: int, rank: int) -> int:
    """Distinct, reproducible data seed per rank (weak scaling: every rank processes its own batch)."""
    return base_seed + 1000003 * rank


def max_over_ranks(values, device=None):
    """Element-wise MAX over ranks of a list of python floats (timings are reported as the slowest rank's)."""
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        if t.is_cuda:
            t = t.float()
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.tolist()


class GradSync:
    """Data-parallel gradient averaging for a painter_b200 module: replaces the DistributedDataParallel reducer of
    Painter/main_train.py:340.

    The module's backward stages write every gradient into the flat arena (painter_b200/arena.py) in production
    order; as soon as the stages of a bucket (a contiguous arena range of >= bucket_mb) have been enqueued, ONE
    all-reduce(mean) of that range is issued asynchronously (NCCL runs it on its own stream after the producing
    kernels, over NVLink / NVSwitch), so communication overlaps the rest of backward with no copy into separate
    buckets and a handful of large collectives per step.  The last stage waits for all of them.  While collectives
    are in flight the persistent GEMM sizes its grid for `132 - sm_reserve` SMs, so that a NCCL kernel
    holding a few SMs never pushes statically scheduled tiles into a second wave.

    Semantics = DDP: parameters are broadcast from rank 0 at construction, gradients are averaged over ranks
    every backward (also with gradient accumulation, like engine_train.py which never uses no_sync())."""

    def __init__(self, model, process_group=None, bucket_mb=200, sm_reserve=0, broadcast=True, bg_ctas=0,
                 tail_mb=120):
        """bg_ctas > 0 (NCCL only): buckets whose all-reduce has the rest of backward to hide behind run on a second
        communicator limited to `bg_ctas` CTAs (NCCL's default of up to 32 CTAs takes that many SMs away from the
        persistent GEMM grids for the duration of every bucket); the last `tail_mb` MB of gradients - whose latency
        is exposed at the end of backward - keep the full-width default communicator."""
        from .arena import get_arena
        self.group = process_group
        self.world = dist.get_world_size(process_group)
        self.backend = dist.get_backend(process_group)
        self.sm_reserve = int(sm_reserve)
        self.bg_group = None
        if bg_ctas > 0 and self.backend == "nccl" and self.world > 1:
            opts = dist.ProcessGroupNCCL.Options()
            opts.config.max_ctas = int(bg_ctas)
            opts.config.min_ctas = 1
            self.bg_group = dist.new_group(backend="nccl", pg_options=opts)
        self.tail_floats = int(tail_mb * (1 << 20) / 4)
        arena = get_arena(model)
        arena.sync = self
        self.arena = arena
        self.buckets = self.plan(arena.group_ranges, bucket_mb)
        self._works = []
        self._next = 0
        self._old_budget = None
        if broadcast and self.world > 1:
            with torch.no_grad():
                for p in model.parameters():
                    dist.broadcast(p.data, 0, group=process_group)
                for b in model.buffers():
                    dist.broadcast(b.data, 0, group=process_group)

    @staticmethod
    def plan(group_ranges, bucket_mb):
        """[(start, end, last_group_name)]: consecutive stage groups merged until a bucket holds >= bucket_mb MB."""
        want = int(bucket_mb * (1 << 20) / 4)
        out, start, last = [], None, None
        for name, a, b in group_ranges:
            if start is None:
                start = a
            last = (name, b)
            if b - start >= want:
                out.append((start, b, name))
                start = None
        if start is not None:
            out.append((start, last[1], last[0]))
        return out

    # ---- protocol driven by GradArena
    def begin(self, arena):
        self._works = []
        self._next = 0
        if self.sm_reserve > 0 and arena.slab.is_cuda and self._old_budget is None:
            from . import ops
            total = torch.cuda.get_device_properties(arena.slab.device).multi_processor_count
            self._old_budget = ops.set_sm_budget(total - self.sm_reserve)

    def stage_done(self, arena, name):
        if self._next < len(self.buckets) and self.buckets[self._next][2] == name:
            a, b, _ = self.buckets[self._next]
            self._next += 1
            if self.world > 1 and not os.environ.get("PK_GRADSYNC_SKIP"):   # (diagnostic: everything but the wire)
                t = arena.cur[a:b]
                if self.backend == "nccl":
                    g = self.group
                    if self.bg_group is not None and b <= arena.total - self.tail_floats:
                        g = self.bg_group
                    w = dist.all_reduce(t, op=dist.ReduceOp.AVG, group=g, async_op=True)
                    self._works.append((w, None))
                else:
                    w = dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
                    self._works.append((w, t))

    def finish(self, arena):
        if self._next != len(self.buckets):
            raise RuntimeError("painter_b200.GradSync: backward ended before every gradient bucket was produced")
        for w, t in self._works:
            w.wait()
            if t is not None:
                t.div_(self.world)
        self._works = []
        if self._old_budget is not None:
            from . import ops
            ops.set_sm_budget(self._old_budget)
            self._old_budget = None


def average_gradients(params):
    """Reference semantics of DDP's reducer: grad <- mean over ranks (flat bucket, one all-reduce)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    flat /= dist.get_world_size()
    off = 0
    for g in grads:
        n = g.numel()
        g.copy_(flat[off:off + n].view_as(g))
        off += n
