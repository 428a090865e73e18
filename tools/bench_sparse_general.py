"""LanczosNetGeneral from bond-list records: the padded forward against SparseLanczosNetGeneral.forward_sparse
with and without eigenpairs in the records, and one training step, eager and captured.

    python tools/bench_sparse_general.py [--B 64 1024] [--iters 20] [--repeats 3]

Per batch size (config graph_lanczos_net: 7 layers of 128, K = 20, input width 10; seeded weights,
data.synthetic_regression_graphs: G(n, 0.5), n in [20, 100], N = batch max), one JSON line.  Every time is
measured ``--repeats`` times, the rows alternating within each repeat, and reported as median, min and max:
  * forward_padded_ms: ``forward`` from a pinned host batch (node_feat, L, D, V, mask), replayed from its
    CUDA graph, copies included;
  * forward_sparse_eigs_ms / forward_sparse_noeigs_ms: ``forward_sparse`` from pinned records with the host's
    eigenpairs (D, V_rows), or with only K (one lnb_graph_eigs_sparse launch in the graph);
  * step_eager_ms: one eager training step (forward, loss, backward, Adam) from device inputs;
    step_graphed_padded_ms / step_graphed_sparse_eigs_ms / step_graphed_sparse_noeigs_ms: one
    train.GraphedStep replay from pinned host memory: the padded batch, or the records with / without
    eigenpairs.
Once per batch size, on the host: host_eigh_ms, numpy's fp64 eigh of every graph's L4 (what the records
without eigenpairs leave to the device).
Once per batch size: the bytes each forward copies host to device, and the device time per forward of each
kernel group (torch.profiler, a separate run): prepare, eigensolver, filter-MLP chain, layer 0 (the unfused
first layer) and the convolution stack.  The GPU's name and power limit go into every line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lanczosnetwork_b200 import configs, data, train  # noqa: E402
from lanczosnetwork_b200.model import LanczosNetGeneral, SparseLanczosNetGeneral  # noqa: E402
from bench_sparse_dropins import event_ms, gpu_info  # noqa: E402

K = 20
# kernel groups of one forward, by substring of the kernel name (first match wins)
GROUPS = [('prepare', ('batch_prepare_sparse_kernel', 'graph_prepare_kernel', 'tile_assign')),
          ('eigensolver', ('graph_eigs',)),
          ('filter_chain', ('ChainPolicy', 'ritz_power_table', 'ritz_rowmap')),
          ('stack', ('SpectralPolicy',)),
          ('layer0', ('batched_gemm', 'RowLoadPolicy', 'graph_messages', 'operator_chain', 'split_tf32'))]


def nbytes(*ts):
  return int(sum(t.numel() * t.element_size() for t in ts if torch.is_tensor(t)))


def pinned(x):
  return torch.from_numpy(np.ascontiguousarray(x)).pin_memory()


def kernel_groups(fn, iters):
  """Device microseconds per call of each kernel group, and of every kernel, over ``iters`` calls."""
  from torch.profiler import ProfilerActivity, profile
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(iters):
      fn()
    torch.cuda.synchronize()
  groups = {g: 0.0 for g, _ in GROUPS}
  groups['other'] = 0.0
  kernels = {}
  for e in prof.key_averages():
    if e.device_time_total <= 0 or e.key.startswith('Memcpy') or e.key.startswith('Memset'):
      continue
    us = e.device_time_total / iters
    kernels[e.key[:80]] = round(us, 2)
    g = next((g for g, subs in GROUPS if any(s in e.key for s in subs)), 'other')
    groups[g] += us
  return {k: round(v, 2) for k, v in groups.items()}, kernels


def row(B, iters, repeats, dev):
  samples = data.synthetic_regression_graphs(B, seed=B + 11)
  c = data.collate(samples, K)
  padded = [pinned(c[k]) for k in ('node_feat', 'L', 'D', 'V', 'node_mask')]
  label = pinned(c['label'])
  dpadded, dlabel = [t.to(dev) for t in padded], label.to(dev)
  rec_eigs = {k: (pinned(v) if isinstance(v, np.ndarray) else v)
              for k, v in data.sparse_collate(samples, K).items() if k != 'label'}
  rec = {k: (pinned(v) if isinstance(v, np.ndarray) else v)
         for k, v in data.sparse_collate(samples, K, eigs=False).items() if k != 'label'}
  cfg = configs.graph_lanczos_net()
  torch.manual_seed(0)
  weights = LanczosNetGeneral(cfg).state_dict()

  def fresh():
    mod = SparseLanczosNetGeneral(cfg)
    mod.load_state_dict(weights)
    return mod.to(dev)

  inf = fresh().eval()
  out = {'gpu': gpu_info(), 'B': B, 'N': int(c['L'].shape[1]), 'bonds': int(rec['edge_ptr'][-1])}
  fwd = {'forward_padded_ms': lambda: inf(*padded[:4], mask=padded[4]),
         'forward_sparse_eigs_ms': lambda: inf.forward_sparse(rec_eigs),
         'forward_sparse_noeigs_ms': lambda: inf.forward_sparse(rec)}
  with torch.no_grad():
    want = fwd['forward_padded_ms']()
    out['forward_sparse_eigs_equal'] = bool(torch.equal(fwd['forward_sparse_eigs_ms'](), want))
    out['forward_sparse_noeigs_max_abs_diff'] = float((fwd['forward_sparse_noeigs_ms']() - want).abs().max())

  eager = fresh().train()
  opt_e = torch.optim.Adam(eager.parameters(), lr=1e-4)

  def eager_step():
    opt_e.zero_grad()
    eager(*dpadded[:4], label=dlabel, mask=dpadded[4])[1].backward()
    opt_e.step()

  mod_p = fresh()
  st_p = train.GraphedStep(mod_p, torch.optim.Adam(mod_p.parameters(), lr=1e-4), tuple(padded[:4]),
                           {'label': label, 'mask': padded[4]})
  steps = {'step_eager_ms': eager_step,
           'step_graphed_padded_ms': lambda: st_p(*padded[:4], label=label, mask=padded[4])}
  for name, r in (('step_graphed_sparse_eigs_ms', rec_eigs), ('step_graphed_sparse_noeigs_ms', rec)):
    mod_s = fresh()
    st_s = train.GraphedStep(mod_s, torch.optim.Adam(mod_s.parameters(), lr=1e-4), (r,), {'label': label},
                             sparse=True)
    steps[name] = lambda st_s=st_s, r=r: st_s(r, label=label)
  timers = [(k, f, iters, False) for k, f in fwd.items()] + [(k, f, max(iters // 4, 3), True)
                                                              for k, f in steps.items()]
  vals = {name: [] for name, _, _, _ in timers}
  for _ in range(repeats):                         # the rows alternate within every repeat
    for name, fn, n, grad in timers:
      with torch.set_grad_enabled(grad):
        vals[name].append(event_ms(fn, n))
  for name, v in vals.items():
    out[name] = {'median': round(float(np.median(v)), 4), 'min': round(float(min(v)), 4),
                 'max': round(float(max(v)), 4)}
  out['repeats'] = repeats
  t0 = time.perf_counter()
  for s in samples:
    np.linalg.eigh(s['L_simple_4'])
  out['host_eigh_ms'] = round((time.perf_counter() - t0) * 1e3, 2)
  out['h2d_bytes'] = {'forward_padded': nbytes(*padded),
                      'forward_sparse_eigs': nbytes(*rec_eigs.values()),
                      'forward_sparse_noeigs': nbytes(*rec.values())}
  # per-kernel times in a separate, eager run (LNB_NO_GRAPH semantics: the graph cache off)
  inf.use_cuda_graph = False
  prof = {}
  with torch.no_grad():
    for name, fn in fwd.items():
      prof[name.replace('_ms', '')] = kernel_groups(fn, 5)
  out['kernel_us_per_forward'] = {k: v[0] for k, v in prof.items()}
  out['kernels_us'] = {k: v[1] for k, v in prof.items()}
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, nargs='+', default=[64, 1024])
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--repeats', type=int, default=3)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_sparse_general: needs a CUDA device')
  dev = torch.device('cuda:0')
  for B in args.B:
    print(json.dumps(row(B, args.iters, args.repeats, dev)), flush=True)


if __name__ == '__main__':
  main()
