"""Measurements of the BASELINE.json model configs other than the bench.py headline (profiling aid;
numbers are printed; the Lanczos configs are in tools/time_lanczos.py).  Run on an H100:
python tools/bench_configs.py"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from helpers import deterministic_state_dict  # noqa: E402
from lanczosnetwork_b200 import configs, data  # noqa: E402
from lanczosnetwork_b200.model import AdaLanczosNet, LanczosNetGeneral  # noqa: E402

dev = torch.device('cuda:0')


def timeit(fn, iters=10, warm=3):
  for _ in range(warm):
    fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / iters


def ada_forward(out):
  cfg = configs.qm8_ada_lanczos_net()
  mod = AdaLanczosNet(cfg)
  mod.load_state_dict(deterministic_state_dict(mod, 2024))
  mod = mod.to(dev).eval()
  for B in (64, 256):
    batch = data.synthetic_qm8_batch(B, seed=3)
    nf = torch.from_numpy(batch['node_feat']).to(dev)
    L = torch.from_numpy(batch['L']).to(dev)
    mask = torch.from_numpy(batch['node_mask']).to(dev)
    with torch.no_grad():
      t = timeit(lambda: mod(nf, L, mask=mask), iters=5, warm=2)
    rec = {'config': 'QM8 AdaLanczosNet forward', 'batch': B, 'ms': t, 'molecules_per_s': B / (t * 1e-3)}
    out.append(('ada', rec))
    print(json.dumps(rec), flush=True)


def general_forward(out):
  graphs = data.synthetic_regression_graphs(num_graphs=16, seed=123)
  b = data.collate(graphs, 20)
  mod = LanczosNetGeneral(configs.graph_lanczos_net())
  mod.load_state_dict(deterministic_state_dict(mod, 4321))
  mod = mod.to(dev).eval()
  args = [torch.from_numpy(b[k]).to(dev) for k in ('node_feat', 'L', 'D', 'V')]
  mask = torch.from_numpy(b['node_mask']).to(dev)
  with torch.no_grad():
    t = timeit(lambda: mod(*args, mask=mask))
  rec = {'config': 'synthetic graph regression LanczosNetGeneral B=16 N<=100', 'ms': t,
         'graphs_per_s': 16 / (t * 1e-3)}
  out.append(('general', rec))
  print(json.dumps(rec), flush=True)


if __name__ == '__main__':
  res = []
  which = sys.argv[1:] or ['general', 'ada']
  if 'general' in which:
    general_forward(res)
  if 'ada' in which:
    ada_forward(res)
