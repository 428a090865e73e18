"""The operator drop-ins from padded batches against forward_sparse from bond-list records.

    python tools/bench_sparse_dropins.py [--B 1024] [--iters 30] [--models GCN GPNN ...]

Per model (seeded weights, data.synthetic_qm8_samples at B, N = 26), one JSON line with:
  * resident_padded_ms / resident_sparse_ms: the forward from device-resident padded inputs
    (node_feat, L or GAT's bias, mask) and from device-resident sparse records (CUDA events; both
    replay the model's captured graph);
  * e2e_padded_ms / e2e_sparse_ms: from pinned host memory (padded tensors vs sparse records) to the
    score on the device, the copies included (CUDA events);
  * collate_padded_ms / collate_sparse_ms: the host collate alone (data.collate (+ data.gat_bias for GAT)
    vs data.sparse_collate, eigs=False), wall clock;
  * GPNN only: partition_sparse_ms (lnb_spectral_partition_sparse) against partition_dense_ms
    (lnb_spectral_partition + graph_prepare of the two operators), each as one captured graph.
  * SampledGraphSAGE (Mean, Max, LSTM, K = 40): the padded side is data.sage_collate (numpy's draws) +
    forward; the records carry a sample_key and the neighbours are drawn on the device.  bit_equal compares
    forward_sparse with forward on the padded batch of the device's samples.  sampler_kernel_ms: the
    sampler kernel (ELL rows of M, as Mean / Max inference runs it) and operators_prepare_kernel_ms: the
    padded path's lnb_sage_operators + graph_prepare kernels, both per call from torch.profiler.
The GPU's name and power limit go into every line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lanczosnetwork_b200 import configs, data, ops  # noqa: E402
from lanczosnetwork_b200 import model as models  # noqa: E402

MODELS = {
    'GCN': lambda: models.GCN(configs.qm8_gcn()),
    'GCNFP': lambda: models.GCNFP(configs.qm8_gcn()),
    'DCNN': lambda: models.DCNN(configs.qm8_dcnn()),
    'ChebyNet': lambda: models.ChebyNet(configs.qm8_cheby_net()),
    'GAT': lambda: models.GAT(configs.qm8_gat()),
    'GGNN': lambda: models.GGNN(configs.qm8_ggnn()),
    'MPNN': lambda: models.MPNN(configs.qm8_mpnn()),
    'GPNN': lambda: models.GPNN(configs.qm8_gpnn()),
    'SampledGraphSAGE-Mean': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean')),
    'SampledGraphSAGE-Max': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='Max')),
    'SampledGraphSAGE-LSTM': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='LSTM')),
}
SAGE_K = 40


def event_ms(fn, iters):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / iters


def graph_ms(fn, iters):
  """Mean ms per replay of fn captured as one CUDA graph."""
  fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    with torch.cuda.graph(g, stream=s):
      fn()
  torch.cuda.current_stream().wait_stream(s)
  return event_ms(g.replay, iters)


def wall_ms(fn, reps=3):
  best = None
  for _ in range(reps):
    t0 = time.perf_counter()
    fn()
    t = (time.perf_counter() - t0) * 1e3
    best = t if best is None else min(best, t)
  return best


def gpu_info():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except Exception:
    out = torch.cuda.get_device_name(0)
  return out


def profiled_kernel_ms(fn, iters, names):
  """Mean CUDA time per call of the kernels whose names contain one of ``names`` (torch.profiler)."""
  from torch.profiler import ProfilerActivity, profile
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(iters):
      fn()
    torch.cuda.synchronize()
  total = sum(e.device_time_total for e in prof.key_averages() if any(n in e.key for n in names))
  return total / 1e3 / iters


def sage_row(name, mod, samples, row, iters, dev):
  """The SampledGraphSAGE measurements: data.sage_collate + forward against the records."""
  c = data.sage_collate(samples, SAGE_K, np.random.RandomState(0))
  host_pad = [torch.from_numpy(c[k]).pin_memory() for k in ('node_feat', 'nn_idx', 'nonempty_mask', 'node_mask')]
  dev_pad = [t.to(dev) for t in host_pad]
  sp = data.sparse_collate(samples, 20, eigs=False)
  sp['sample_key'] = np.array([1234, 0], np.int64)
  host_sp = {k: (torch.from_numpy(v).pin_memory() if isinstance(v, np.ndarray) else v) for k, v in sp.items()}
  dev_sp = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in host_sp.items()}
  E1 = mod.num_edgetype + 1
  rec = [dev_sp[k] for k in ('sizes', 'node_ptr', 'node_feat', 'edge_ptr', 'edges', 'sample_key')]
  with torch.no_grad():
    node_ids, mask, ne, nn_idx, _, _ = ops.sage_sample_sparse(*rec, sp['N'], E1, SAGE_K)
    ref = mod(node_ids, nn_idx.long(), ne, mask=mask)
    row['bit_equal'] = bool(torch.equal(mod.forward_sparse(dev_sp), ref))
    row['resident_padded_ms'] = round(event_ms(lambda: mod(dev_pad[0], dev_pad[1], dev_pad[2], mask=dev_pad[3]),
                                               iters), 4)
    row['resident_sparse_ms'] = round(event_ms(lambda: mod.forward_sparse(dev_sp), iters), 4)
    row['e2e_padded_ms'] = round(event_ms(lambda: mod(host_pad[0], host_pad[1], host_pad[2], mask=host_pad[3]),
                                          iters), 4)
    row['e2e_sparse_ms'] = round(event_ms(lambda: mod.forward_sparse(host_sp), iters), 4)
    if name.endswith('Mean'):
      row['sampler_kernel_ms'] = round(profiled_kernel_ms(
          lambda: ops.sage_sample_sparse(*rec, sp['N'], E1, SAGE_K, want_nn_idx=False, want_ell=True), iters,
          ['sage_sample_kernel']), 4)
      row['sampler_ell_t_kernel_ms'] = round(profiled_kernel_ms(
          lambda: ops.sage_sample_sparse(*rec, sp['N'], E1, SAGE_K, want_nn_idx=False, want_ell=True,
                                         want_ell_t=True), iters, ['sage_sample_kernel']), 4)
      row['operators_prepare_kernel_ms'] = round(profiled_kernel_ms(
          lambda: ops.graph_prepare(ops.sage_operators(dev_pad[1], dev_pad[2]), defer_tiles=True), iters,
          ['sage_operator_kernel', 'graph_prepare_kernel']), 4)
  row['h2d_padded_bytes'] = int(sum(t.numel() * t.element_size() for t in host_pad))
  row['h2d_sparse_bytes'] = int(sum(v.numel() * v.element_size() for v in host_sp.values() if torch.is_tensor(v)))
  row['collate_padded_ms'] = round(wall_ms(lambda: data.sage_collate(samples, SAGE_K, np.random.RandomState(0))), 2)
  row['collate_sparse_ms'] = round(wall_ms(lambda: data.sparse_collate(samples, 20, eigs=False)), 2)


def padded_inputs(name, samples, K):
  c = data.collate(samples, K)
  L = data.gat_bias(c['L']) if name == 'GAT' else c['L']
  return c['node_feat'], L, c['node_mask']


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, default=1024)
  ap.add_argument('--iters', type=int, default=30)
  ap.add_argument('--models', nargs='+', default=list(MODELS))
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_sparse_dropins: needs a CUDA device')
  dev = torch.device('cuda:0')
  gpu = gpu_info()
  K = 20
  samples = data.synthetic_qm8_samples(args.B, seed=5)
  for name in args.models:
    torch.manual_seed(0)
    mod = MODELS[name]().to(dev).eval()
    if name.startswith('SampledGraphSAGE'):
      row = {'model': name, 'B': args.B, 'N': int(max(s['L_simple_4'].shape[0] for s in samples)), 'gpu': gpu}
      sage_row(name, mod, samples, row, args.iters, dev)
      print(json.dumps(row), flush=True)
      continue
    nf, L, mask = padded_inputs(name, samples, K)
    sp = data.sparse_collate(samples, K, eigs=False)
    host_pad = [torch.from_numpy(a).pin_memory() for a in (nf, L, mask)]
    dev_pad = [t.to(dev) for t in host_pad]
    host_sp = {k: (torch.from_numpy(v).pin_memory() if isinstance(v, np.ndarray) else v) for k, v in sp.items()}
    dev_sp = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in host_sp.items()}
    row = {'model': name, 'B': args.B, 'N': int(sp['N']), 'gpu': gpu}
    with torch.no_grad():
      ref = mod(dev_pad[0], dev_pad[1], mask=dev_pad[2])
      row['bit_equal'] = bool(torch.equal(mod.forward_sparse(dev_sp), ref))
      row['resident_padded_ms'] = round(event_ms(lambda: mod(dev_pad[0], dev_pad[1], mask=dev_pad[2]), args.iters), 4)
      row['resident_sparse_ms'] = round(event_ms(lambda: mod.forward_sparse(dev_sp), args.iters), 4)
      row['e2e_padded_ms'] = round(event_ms(lambda: mod(host_pad[0], host_pad[1], mask=host_pad[2]), args.iters), 4)
      row['e2e_sparse_ms'] = round(event_ms(lambda: mod.forward_sparse(host_sp), args.iters), 4)
    row['h2d_padded_bytes'] = int(sum(t.numel() * t.element_size() for t in host_pad))
    row['h2d_sparse_bytes'] = int(sum(v.numel() * v.element_size() for v in host_sp.values() if torch.is_tensor(v)))
    if name == 'GAT':
      row['collate_padded_ms'] = round(wall_ms(lambda: data.gat_bias(data.collate(samples, K)['L'])), 2)
    else:
      row['collate_padded_ms'] = round(wall_ms(lambda: data.collate(samples, K)), 2)
    row['collate_sparse_ms'] = round(wall_ms(lambda: data.sparse_collate(samples, K, eigs=False)), 2)
    if name == 'GPNN':
      P, N = mod.num_partition, int(sp['N'])
      Ld = dev_pad[1]
      zeros = torch.zeros((args.B, N, 4), device=dev)

      def dense():
        _, Lc, Lt, _ = ops.spectral_partition(Ld, P)
        ops.graph_prepare(torch.stack([Lc, Lt], 3), zeros)
      row['partition_dense_ms'] = round(graph_ms(dense, args.iters), 4)
      row['partition_sparse_ms'] = round(graph_ms(lambda: ops.spectral_partition_sparse(
          dev_sp['sizes'], dev_sp['edge_ptr'], dev_sp['edges'], N, P, mod.num_edgetype), args.iters), 4)
    print(json.dumps(row), flush=True)


if __name__ == '__main__':
  main()
