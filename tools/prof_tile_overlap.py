"""Device intervals of the bench forward's kernels (QM8 LanczosNet, B = 1024) from torch.profiler, for
one eager forward and one CUDA-graph replay: shows the tile placement (tile_assign_kernel) running
beside the filter-MLP chain, and the gap between the chain's end and the convolution stack's start
(profiling aid).

    python tools/prof_tile_overlap.py [out.json]
"""
import json
import os
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import bench  # noqa: E402

KERNELS = (('prepare', 'graph_prepare_kernel'), ('rowmap', 'ritz_rowmap_kernel'),
           ('tile_assign', 'tile_assign_kernel'), ('chain', 'ChainPolicy'), ('stack', 'SpectralPolicy'))

dev = torch.device('cuda:0')
mod, _ = bench.build_model()
mod = mod.to(dev).eval()
bt = bench.make_batches(1, bench.BATCH, 1000)[0]
t = {k: torch.from_numpy(bt[k]).to(dev) for k in ('node_feat', 'L', 'D', 'V', 'node_mask')}


def step():
  return mod(t['node_feat'], t['L'], t['D'], t['V'], mask=t['node_mask'])


def intervals(graph):
  mod.use_cuda_graph = graph
  for _ in range(5):                  # warm caches; with graphs, captures the zero-copy graph
    step()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
  spans = {}
  for e in prof.events():
    if e.device_type != torch.autograd.DeviceType.CUDA:
      continue
    for key, pat in KERNELS:
      if pat in e.name and key not in spans:
        spans[key] = [e.time_range.start, e.time_range.end]
  t0 = min(s for s, _ in spans.values())
  spans = {k: [round(s - t0, 1), round(e - t0, 1)] for k, (s, e) in spans.items()}   # us from the first kernel
  res = {'intervals_us': spans}
  if 'tile_assign' in spans and 'chain' in spans:
    ta, ch = spans['tile_assign'], spans['chain']
    res['tile_assign_inside_chain_us'] = round(max(0.0, min(ta[1], ch[1]) - max(ta[0], ch[0])), 1)
  if 'chain' in spans and 'stack' in spans:
    res['chain_end_to_stack_start_us'] = round(spans['stack'][0] - spans['chain'][1], 1)
  return res


with torch.no_grad():
  out = {'gpu': torch.cuda.get_device_name(dev), 'eager': intervals(False), 'graph_replay': intervals(True)}
print(json.dumps(out, indent=1))
if len(sys.argv) > 1:
  with open(sys.argv[1], 'w') as f:
    json.dump(out, f, indent=1)
