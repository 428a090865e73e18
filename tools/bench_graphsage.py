"""Inference throughput of the GraphSAGE drop-in on QM8-shaped batches (config/qm8_graphsage.yaml), one GPU.

    python tools/bench_graphsage.py [--agg Mean|Max] [--batches 4] [--steps 50] [--warmup 5] [--out result.json]

Workload: rotating synthetic QM8 batches (data.synthetic_qm8_samples + data.sage_collate, B = 1024,
N = 26, K = 40 neighbour samples), resident on the device.  Reports, in one JSON document:
  * ms per forward and molecules/s with CUDA-graph replay (CUDA events around the timed window);
  * per-kernel device times from torch.profiler, in a separate eager run: the operator construction
    (sage_operator_kernel), lnb_graph_prepare (graph_prepare_kernel + tile_assign_kernel) and the stack;
  * the stack's fp32-equivalent rate on the algorithmic GEMM FLOPs and the operator construction's
    bytes/s (both from shapes, over the profiled kernel times);
  * the eager fp32 oracle (oracle/sage_oracle.py, plain PyTorch gathers) on the same GPU;
  * the card's name and power limit, read in the same process.
Writes nothing into the tree unless --out points there."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from helpers import deterministic_state_dict  # noqa: E402
from lanczosnetwork_b200 import configs, data  # noqa: E402
from lanczosnetwork_b200.model import GraphSAGE  # noqa: E402
from oracle import sage_oracle  # noqa: E402


def card():
  out = {'name': torch.cuda.get_device_name(0)}
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    out['nvidia_smi'] = q
  except Exception as exc:      # the measurement stands; the record says the query failed
    out['nvidia_smi'] = 'query failed: %s' % exc
  return out


def shape_arithmetic(cfg, B, N):
  """Algorithmic FLOPs of the propagation layers' GEMMs (every row, padded ones included) and the bytes
  the operator construction moves (nn_idx + nonempty read, dense operators written).  From shapes, not
  measured."""
  m = cfg.model
  E1 = cfg.dataset.num_bond_type + 1
  dims = [m.input_dim] + list(m.hidden_dim)
  gemm_flops = [2.0 * B * N * dims[t] * E1 * dims[t + 1] for t in range(m.num_layer - 1)]
  op_bytes = 8.0 * B * N * m.num_sample_neighbors * E1 + 4.0 * B * N + 4.0 * B * N * N * E1
  return gemm_flops, op_bytes


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--agg', default='Mean', choices=['Mean', 'Max'])
  ap.add_argument('--batches', type=int, default=4)
  ap.add_argument('--batch-size', type=int, default=1024)
  ap.add_argument('--steps', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--oracle-steps', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_graphsage: needs a CUDA device')
  dev = torch.device('cuda:0')
  cfg = configs.qm8_graphsage(agg_func=args.agg)
  B = args.batch_size
  batches = []
  for i in range(args.batches):
    b = data.sage_collate(data.synthetic_qm8_samples(B, seed=1000 + i), cfg.model.num_sample_neighbors,
                          np.random.RandomState(i))
    batches.append({k: torch.from_numpy(b[k]).to(dev) for k in ('node_feat', 'nn_idx', 'nonempty_mask',
                                                                'node_mask')})
  N = int(batches[0]['node_feat'].shape[1])
  mod = GraphSAGE(cfg)
  params = deterministic_state_dict(mod, 1234)
  mod.load_state_dict(params)
  mod = mod.to(dev).eval()

  def step(i):
    b = batches[i % len(batches)]
    return mod(b['node_feat'], b['nn_idx'], b['nonempty_mask'], mask=b['node_mask'])

  res = {'workload': {'model': 'GraphSAGE', 'config': 'config/qm8_graphsage.yaml', 'agg_func': args.agg,
                      'B': B, 'N': N, 'K': cfg.model.num_sample_neighbors, 'rotating_batches': args.batches}}
  with torch.no_grad():
    # 1. CUDA-graph replay, timed with events
    for i in range(args.warmup + 2 * args.batches):
      step(i)
    torch.cuda.synchronize()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(args.steps):
      step(i)
    e.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(e) / args.steps
    res['graph_replay'] = {'ms_per_forward': ms, 'molecules_per_s': B / ms * 1e3, 'steps': args.steps,
                           'graph_stats': mod.graph_stats()}

    # 2. per-kernel device times, eager launches, separate run
    mod.use_cuda_graph = False
    for i in range(3):
      step(i)
    torch.cuda.synchronize()
    prof_steps = 10
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      for i in range(prof_steps):
        step(i)
      torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
      t = getattr(ev, 'device_time_total', None)
      if t is None:
        t = ev.cuda_time_total
      if t > 0 and ev.count > 0:
        kernels[ev.key] = {'us_per_forward': t / prof_steps, 'launches_per_forward': ev.count / prof_steps}
    res['kernels'] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]['us_per_forward']))
    mod.use_cuda_graph = True

    def total_us(pattern):
      return sum(v['us_per_forward'] for k, v in kernels.items() if pattern in k)

    gemm_flops, op_bytes = shape_arithmetic(cfg, B, N)
    stack_us, op_us = total_us('tc_gemm'), total_us('sage_operator')
    prep_us = total_us('graph_prepare') + total_us('tile_assign')
    res['shape_arithmetic_not_measured'] = {
        'gemm_gflop_per_forward': [f / 1e9 for f in gemm_flops],
        'gemm_gflop_total': sum(gemm_flops) / 1e9,
        'dense_operator_mb': 4.0 * B * N * N * (cfg.dataset.num_bond_type + 1) / 1e6,
        'operator_construction_hbm_mb': op_bytes / 1e6}
    res['rates'] = {
        'stack_kernel_us_per_forward': stack_us,
        'stack_fp32_equiv_tflops': sum(gemm_flops) / (stack_us * 1e-6) / 1e12 if stack_us else None,
        'operator_construction_us_per_forward': op_us,
        'operator_construction_tb_per_s': op_bytes / (op_us * 1e-6) / 1e12 if op_us else None,
        'graph_prepare_us_per_forward': prep_us}

    # 3. eager fp32 oracle (plain PyTorch) on the same GPU
    spec = sage_oracle.make_spec(cfg.model.num_layer, cfg.model.agg_func, cfg.dataset.num_bond_type)
    gparams = {k: v.to(dev) for k, v in params.items()}
    b0 = batches[0]
    oargs = (b0['node_feat'], b0['nn_idx'], b0['nonempty_mask'], b0['node_mask'])
    ref = sage_oracle.sage_forward(gparams, spec, *oargs, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.oracle_steps):
      sage_oracle.sage_forward(gparams, spec, *oargs, device=dev)
    torch.cuda.synchronize()
    oms = (time.perf_counter() - t0) * 1e3 / args.oracle_steps
    ours = mod(b0['node_feat'], b0['nn_idx'], b0['nonempty_mask'], mask=b0['node_mask'])
    res['eager_fp32_oracle'] = {'ms_per_forward': oms, 'molecules_per_s': B / oms * 1e3,
                                'max_abs_diff_vs_dropin': float((ours - ref).abs().max())}
    res['speedup_vs_eager_oracle'] = oms / ms
  res['card'] = card()
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, 'w') as fh:
      json.dump(res, fh, indent=1)


if __name__ == '__main__':
  main()
