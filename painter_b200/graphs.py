"""CUDA-graph replay of the inference forward.

SegGPT in-context inference with one prompt (BASELINE.json configs[2]) is a launch-latency regime: ~600 kernel
launches for ~2 ms of tensor-core work (M = 3136 / 1568 rows).  `GraphedForward` captures one no-grad forward of the
module into a CUDA graph per (input shapes, seg type layout, ensemble flag, prompt grouping, weight versions) and
replays it: the inputs are copied into static buffers, one `cudaGraphLaunch` runs every kernel back to back, the
outputs are the graph's static result tensors (valid until the next call with the same key).

Everything in the forward is capture-safe: kernels go to the capture stream, TMA descriptors travel as kernel
parameters, temporaries come from the graph's private memory pool, and there is no host synchronisation.
"""
import torch


class GraphedForward:
    def __init__(self, model, warmup=2):
        self.model = model
        self.warmup = warmup
        self.entries = {}

    def _weights_version(self):
        return sum(p._version for p in self.model.parameters())

    def captured_batch(self, imgs_shape, B, prompts_per_query=None):
        """The smallest batch >= B of a graph already captured for canvases of shape imgs_shape[1:] (and the same
        prompt grouping), else B: a batched caller pads a tail batch to it and replays that graph."""
        sizes = [k[0][0] for k in self.entries
                 if k[0][1:] == tuple(imgs_shape[1:]) and k[-1] == prompts_per_query and k[0][0] >= B]
        return min(sizes, default=B)

    def __call__(self, imgs, tgts, bool_masked_pos, valid, seg_type=None, merge_between_batch=-1,
                 prompts_per_query=None):
        """Same arguments / results as `model._run(...)` under no_grad: (loss, patchify(pred), mask).  The returned
        loss and prediction are the graph's static buffers (overwritten by the next replay of the same shape)."""
        m = self.model
        mask = bool_masked_pos.flatten(1).to(torch.bool)
        key = (tuple(imgs.shape), tuple(mask.shape), tuple(valid.shape), None if seg_type is None else
               tuple(seg_type.shape), int(merge_between_batch), getattr(m, "precision", "bf16"),
               self._weights_version(), imgs.device.index, prompts_per_query)
        ent = self.entries.get(key)
        if ent is None:
            if len(self.entries) > 8:
                self.entries.clear()
            ent = self._capture(imgs, tgts, mask, valid, seg_type, merge_between_batch, prompts_per_query)
            self.entries[key] = ent
        static_in, graph, out = ent
        static_in[0].copy_(imgs, non_blocking=True)
        static_in[1].copy_(tgts, non_blocking=True)
        static_in[2].copy_(mask, non_blocking=True)
        static_in[3].copy_(valid, non_blocking=True)
        if seg_type is not None:
            static_in[4].copy_(seg_type, non_blocking=True)
        graph.replay()
        return out[0], out[1], mask

    def _capture(self, imgs, tgts, mask, valid, seg_type, merge, prompts_per_query):
        m = self.model
        dev = imgs.device
        si = [imgs.detach().float().clone(), tgts.detach().float().clone(), mask.clone(),
              valid.detach().float().clone(), None if seg_type is None else seg_type.detach().float().clone()]

        def run():
            with torch.no_grad():
                if seg_type is None:
                    return m._run(si[0], si[1], si[2], si[3])
                return m._run(si[0], si[1], si[2], si[3], si[4], merge, prompts_per_query)

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                run()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        # the warm-up's temporaries go back to the device before the graph's private pool allocates its own: a large
        # fp32-accurate batch would otherwise hold both
        torch.cuda.empty_cache()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = run()
        return si, g, out
