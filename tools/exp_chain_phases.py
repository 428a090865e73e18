"""Filter-MLP chain kernel alone on the bench workload (QM8 LanczosNet, B = 1024), replayed from its own
CUDA graph, as built and with the skeleton's debug switches (LNB_DBG: 2 skips the MMAs, 4 the W loads,
8 produce(), 6 MMAs and W loads): what is left with the tensor side switched off is the CUDA-core and
hand-over work of the items (profiling aid; results are wrong with any switch set)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import bench  # noqa: E402
from lanczosnetwork_b200 import ops  # noqa: E402
from lanczosnetwork_b200.spectral_conv import ritz_filter_coefficients  # noqa: E402

dev = torch.device('cuda:0')
mod, _ = bench.build_model()
mod = mod.to(dev).eval()
bt = bench.make_batches(1, bench.BATCH, 1000)[0]
t = {k: torch.from_numpy(bt[k]).to(dev) for k in ('L', 'D', 'V')}
L, V, D = t['L'].float().contiguous(), t['V'].float().contiguous(), t['D'].float().contiguous()


def graph_time(fn, reps=50):
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(3):
      fn()
  torch.cuda.current_stream().wait_stream(s)
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    fn()
  for _ in range(3):
    g.replay()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(reps):
    g.replay()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / reps * 1e3


with torch.no_grad():
  prep = ops.graph_prepare(L, V)
  table = ops.ritz_power_table(D, mod.long_diffusion_dist)
  mlp = mod._filter_mlp_params()
  for flag in (0, 2, 4, 8, 6):
    os.environ['LNB_DBG'] = str(flag)          # read when the kernel is launched (captured)
    us = graph_time(lambda: ritz_filter_coefficients(D, mod.long_diffusion_dist, mlp, mod._wcache, prep,
                                                     table=table))
    print('LNB_DBG=%d  filter MLP chain %.1f us' % (flag, us))
  os.environ.pop('LNB_DBG')
