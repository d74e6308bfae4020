"""Warm kernel timeline of the training step (torch.profiler / CUPTI): per-kernel totals inside real steps and the
idle time between kernels on the compute stream.  Unlike the ncu launch list (cold caches, serialised replays) these
are the durations the step actually sees.
Usage (on the GPU machine): python scripts/step_timeline.py [steps] > step_timeline.txt"""
import collections
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from painter_b200 import models_painter  # noqa: E402
from painter_b200.optim import FusedAdamW  # noqa: E402
from painter_b200.train_utils import adjust_learning_rate, param_groups_lrd  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
dev = torch.device("cuda", 0)
torch.manual_seed(0)
model = models_painter.painter_vit_large_patch16_input896x448_win_dec64_8glb_sl1().to(dev)
with torch.no_grad():
    for n, p in model.named_parameters():
        if "rel_pos" in n:
            p.normal_(std=0.02)
model.train()
groups = param_groups_lrd(model, 0.05, no_weight_decay_list=model.no_weight_decay(), layer_decay=0.8)
opt = FusedAdamW(groups, lr=1e-4, betas=(0.9, 0.999))
adjust_learning_rate(opt, 1.0, 1e-4, 0.0, 1, 15)
batch = [t.to(dev) for t in bench._batch(8, 0)]


def step():
    imgs, tgts, mask, valid = batch
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss, _, _ = model(imgs, tgts, bool_masked_pos=mask, valid=valid)
    loss.backward()
    opt.step()
    opt.zero_grad(set_to_none=True)


for _ in range(4):
    step()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(steps):
    step()
e1.record()
torch.cuda.synchronize()
print(f"# unprofiled: {e0.elapsed_time(e1) / steps:.3f} ms per step")

with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(steps):
        step()
    torch.cuda.synchronize()

evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range is not None]
ks = sorted(((e.time_range.start, e.time_range.end, e.name) for e in evs), key=lambda t: t[0])
if not ks:
    print("no CUDA events captured")
    sys.exit(1)
span = ks[-1][1] - ks[0][0]
busy, gaps, cur_end = 0.0, [], ks[0][0]
gap_after = collections.defaultdict(lambda: [0, 0.0])
prev = None
for s, e, n in ks:
    if s > cur_end:
        gaps.append(s - cur_end)
        if prev is not None:
            g = gap_after[prev.split("(")[0][:60]]
            g[0] += 1
            g[1] += s - cur_end
    busy += max(0.0, e - max(s, cur_end))
    cur_end = max(cur_end, e)
    prev = n
print(f"# profiled: {steps} steps, {len(ks)} kernels/memops, span {span / 1e3 / steps:.3f} ms per step, "
      f"busy {busy / 1e3 / steps:.3f} ms per step, idle {sum(gaps) / 1e3 / steps:.3f} ms per step in "
      f"{len(gaps) / steps:.0f} gaps (mean {sum(gaps) / max(1, len(gaps)):.2f} us)")
agg = collections.defaultdict(lambda: [0, 0.0])
for s, e, n in ks:
    a = agg[n.split("(")[0][:70]]
    a[0] += 1
    a[1] += e - s
print("# per kernel (warm, inside the step): total ms/step, launches/step, mean us")
for n, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"{t / 1e3 / steps:9.3f} ms  n={c / steps:6.1f}  avg {t / c:9.1f} us  {n}")
print("# idle time by preceding kernel: total us/step, count/step")
for n, (c, t) in sorted(gap_after.items(), key=lambda kv: -kv[1][1])[:25]:
    print(f"{t / steps:9.1f} us  n={c / steps:6.1f}  {n}")
