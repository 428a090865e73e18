"""Per-kernel device time of the bench forward (QM8 LanczosNet, B = 1024) from torch.profiler:
eager launches, so every kernel of the step shows up under its own name (profiling aid).

    python tools/prof_forward_kernels.py [steps] [trace.json]
"""
import os
import sys
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import bench  # noqa: E402

dev = torch.device('cuda:0')
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
mod, _ = bench.build_model()
mod = mod.to(dev).eval()
mod.use_cuda_graph = False
bt = bench.make_batches(1, bench.BATCH, 1000)[0]
t = {k: torch.from_numpy(bt[k]).to(dev) for k in ('node_feat', 'L', 'D', 'V', 'node_mask')}


def step():
  return mod(t['node_feat'], t['L'], t['D'], t['V'], mask=t['node_mask'])


with torch.no_grad():
  for _ in range(5):
    step()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
      step()
    torch.cuda.synchronize()

tot, cnt = defaultdict(float), defaultdict(int)
for e in prof.events():
  if e.device_type == torch.autograd.DeviceType.CUDA:
    tot[e.name] += e.device_time
    cnt[e.name] += 1
print('%10s %6s  %s' % ('us/step', 'calls', 'kernel'))
for name in sorted(tot, key=tot.get, reverse=True):
  print('%10.1f %6d  %s' % (tot[name] / steps, cnt[name] // steps, name[:110]))
print('%10.1f         sum of kernel time per step' % (sum(tot.values()) / steps))
if len(sys.argv) > 2:
  prof.export_chrome_trace(sys.argv[2])
