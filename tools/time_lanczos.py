"""Timings of the fused Lanczos+QL+Ritz kernel at the BASELINE.json sizes (profiling aid)."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import bench  # noqa: E402
from lanczosnetwork_b200 import data, ops  # noqa: E402

dev = torch.device('cuda:0')
peaks = bench.load_peaks()
which = [a for a in sys.argv[1:] if a != 'phases-only'] or ['qm8', '64', '256', '1024']
PHASES_ONLY = 'phases-only' in sys.argv


def report(name, t, G, N, K, st):
  by = bench.lanczos_alg_bytes(N, K, True)
  print(json.dumps({'name': name, 'ms': t, 'graphs_per_s': G / (t * 1e-3),
                    'alg_GBs': G * by / (t * 1e-3) / 1e9,
                    'frac_hbm': G * by / (t * 1e-3) / 1e9 / peaks['hbm_gbs'],
                    'streamed': int((st & 2).sum().item() // 2), 'ql_fail': int((st & 1).sum().item())}), flush=True)


if 'qm8' in which:
  b = data.synthetic_qm8_batch(1024, seed=1)
  A = torch.from_numpy(b['L'][..., 0].copy()).to(dev)
  mask = torch.from_numpy(b['node_mask']).to(dev)
  q1 = torch.randn(1024, 26, generator=torch.Generator().manual_seed(1)).to(dev)
  o = ops.lanczos_ritz(A, mask, q1, 20)
  for kw in ([] if PHASES_ONLY else [{}, {'want_ritz': False}, {'want_T': False, 'want_Q': False}]):
    t = bench.time_events(lambda: ops.lanczos_ritz(A, mask, q1, 20, **kw), 20, 5)
    report('qm8 %s' % kw, t, 1024, 26, 20, o['status'])
for N, G in ((64, 10000), (256, 10000), (1024, 10000)):
  if str(N) not in which:
    continue
  rng = np.random.RandomState(1234 + N)
  base = np.stack([bench.gnp_operator(rng, N, min(0.5, 8.0 / N)) for _ in range(8)])
  Ad = torch.from_numpy(base).to(dev).repeat((G + 7) // 8, 1, 1)[:G].contiguous()
  q1 = torch.randn(G, N, generator=torch.Generator().manual_seed(1234)).to(dev)
  o = ops.lanczos_ritz(Ad, None, q1, 40)
  for kw in ([] if PHASES_ONLY else [{}, {'want_ritz': False}, {'want_T': False, 'want_Q': False}]):
    t = bench.time_events(lambda: ops.lanczos_ritz(Ad, None, q1, 40, **kw), 3, 1)
    report('N=%d %s' % (N, kw), t, G, N, 40, o['status'])
  del Ad
  torch.cuda.empty_cache()

# per-phase clock64 totals (cycles per graph, thread 0 of each group)
import ctypes
from lanczosnetwork_b200 import _lib
lib = _lib.load()
names = ['compress', 'start', 'lanczos', 'post+TQ', 'QL', 'V=QZ', 'write V']


def phases(tag, fn):
  prof = torch.zeros(64, dtype=torch.int64, device=dev)
  _lib.check(lib.lnb_debug_set_prof(ctypes.c_void_p(prof.data_ptr())), 'set_prof')
  fn()
  torch.cuda.synchronize()
  lib.lnb_debug_set_prof(None)
  p = prof.cpu().double()
  n = max(p[8].item(), 1)
  print(tag, ' '.join('%s=%d' % (nm, p[i].item() / n) for i, nm in enumerate(names)), 'graphs=%d' % n, flush=True)


if 'qm8' in which:
  q1 = torch.randn(1024, 26, generator=torch.Generator().manual_seed(1)).to(dev)
  phases('phases qm8', lambda: ops.lanczos_ritz(A, mask, q1, 20))
for N, G in ((64, 10000), (256, 10000), (1024, 2000)):
  if str(N) not in which:
    continue
  rng = np.random.RandomState(1234 + N)
  base = np.stack([bench.gnp_operator(rng, N, min(0.5, 8.0 / N)) for _ in range(8)])
  Ad = torch.from_numpy(base).to(dev).repeat((G + 7) // 8, 1, 1)[:G].contiguous()
  q1 = torch.randn(G, N, generator=torch.Generator().manual_seed(1234)).to(dev)
  phases('phases N=%d' % N, lambda: ops.lanczos_ritz(Ad, None, q1, 40))
  del Ad
