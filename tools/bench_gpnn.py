"""Throughput of the GPNN drop-in on QM8-shaped batches (config/qm8_gpnn.yaml), one GPU.

    python tools/bench_gpnn.py [--batches 4] [--steps 20] [--warmup 3] [--out result.json]

Workload: rotating synthetic QM8 batches (data.synthetic_qm8_batch, B = 1024, N = 26) with partition
operators from seeded labels (data.random_partition_labels + data.partition_operators), resident on the
device.  Reports, in one JSON document:
  * ms per forward and molecules/s with CUDA-graph replay (CUDA events around the timed window);
  * per-kernel device times from torch.profiler, in a separate eager run;
  * lnb_gpnn_partition_update's fp32-equivalent rate on algorithmic FLOPs (the gi and gh products of both
    parts; the zero gate blocks it also multiplies are not counted), from the profiled kernel time;
  * the shape arithmetic of one step (not measured);
  * the eager fp32 oracle (oracle/gpnn_oracle.py, plain PyTorch) on the same GPU;
  * a training step at B = 64, eager and under train.GraphedStep;
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
from lanczosnetwork_b200.model import GPNN  # noqa: E402
from lanczosnetwork_b200.train import GraphedStep  # noqa: E402
from oracle import gpnn_oracle  # noqa: E402

KEYS = ('node_feat', 'L', 'L_cluster', 'L_cut', 'node_mask', 'label')


def card():
  out = {'name': torch.cuda.get_device_name(0)}
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    out['nvidia_smi'] = q
  except Exception as exc:      # the measurement stands; the record says the query failed
    out['nvidia_smi'] = 'query failed: %s' % exc
  return out


def batch(B, seed, dev):
  b = data.synthetic_qm8_batch(B, seed=seed)
  lab = data.random_partition_labels(np.random.RandomState(seed), B, b['L'].shape[1])
  b['L_cluster'], b['L_cut'] = data.partition_operators(b['L'][:, :, :, 0], lab)
  return {k: torch.from_numpy(b[k]).to(dev) for k in KEYS}


def step_gflop(B, N, H, E1):
  """Algorithmic GFLOP of one propagation step at the default 1 / 1 partition counts (shapes, not
  measured)."""
  R = B * N
  msg0 = 2.0 * R * (H * 128 + 128 * H)
  part = 2 * (2.0 * R * H * 3 * H + 2.0 * R * H * 3 * H)        # gi + gh of both parts
  part_exec = 2 * 2.0 * R * (2 * H) * (4 * H)                     # the [4H, 2H] gate GEMM of both parts
  state = 2.0 * R * (3 * H * 512 + 512 * H)
  msgs = 2.0 * R * E1 * (H * 128 + 128 * H)
  upd = 2.0 * R * E1 * H * 3 * H + 2.0 * R * H * 3 * H
  out = {'msg_func0': msg0, 'partition_update': part, 'partition_update_executed': part_exec,
         'state_func': state, 'message_layers': msgs, 'ggnn_update': upd}
  out = {k: v / 1e9 for k, v in out.items()}
  out['total'] = sum(v for k, v in out.items() if k != 'partition_update_executed')
  return out


def event_ms(fn, reps):
  fn()
  torch.cuda.synchronize()
  a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(reps):
    fn()
  e.record()
  torch.cuda.synchronize()
  return a.elapsed_time(e) / reps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batches', type=int, default=4)
  ap.add_argument('--batch-size', type=int, default=1024)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--oracle-steps', type=int, default=2)
  ap.add_argument('--train-batch', type=int, default=64)
  ap.add_argument('--train-steps', type=int, default=10)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_gpnn: needs a CUDA device')
  dev = torch.device('cuda:0')
  cfg = configs.qm8_gpnn()
  B = args.batch_size
  batches = [batch(B, 1000 + i, dev) for i in range(args.batches)]
  N, E1 = int(batches[0]['L'].shape[1]), int(batches[0]['L'].shape[3])
  H, P = cfg.model.hidden_dim, cfg.model.num_prop
  mod = GPNN(cfg)
  params = deterministic_state_dict(mod, 1234)
  mod.load_state_dict(params)
  mod = mod.to(dev).eval()

  def step(i):
    b = batches[i % len(batches)]
    return mod(b['node_feat'], b['L'], b['L_cluster'], b['L_cut'], mask=b['node_mask'])

  res = {'workload': {'model': 'GPNN', 'config': 'config/qm8_gpnn.yaml', 'B': B, 'N': N, 'hidden': H,
                      'num_prop': P, 'rotating_batches': args.batches}}
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
    for i in range(2):
      step(i)
    torch.cuda.synchronize()
    prof_steps = 4
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
    part_us = sum(v['us_per_forward'] for k, v in kernels.items() if 'GpnnPartitionPolicy' in k)
    flops = step_gflop(B, N, H, E1)
    res['shape_arithmetic_not_measured'] = {'gflop_per_step': flops}
    res['rates'] = {'partition_kernel_us_per_launch': part_us / P,
                    'partition_fp32_equiv_tflops':
                        P * flops['partition_update'] * 1e9 / (part_us * 1e-6) / 1e12 if part_us else None,
                    'forward_fp32_equiv_tflops': P * flops['total'] * 1e9 / (ms * 1e-3) / 1e12}

    # 3. eager fp32 oracle (plain PyTorch) on the same GPU
    spec = gpnn_oracle.make_spec(P, cfg.model.num_prop_cluster, cfg.model.num_prop_cut, cfg.model.aggregate_type,
                                 cfg.model.update_func, cfg.dataset.num_bond_type)
    gparams = {k: v.to(dev) for k, v in params.items()}
    b0 = batches[0]
    oargs = (b0['node_feat'], b0['L'], b0['L_cluster'], b0['L_cut'], b0['node_mask'])
    ref = gpnn_oracle.gpnn_forward(gparams, spec, *oargs, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.oracle_steps):
      gpnn_oracle.gpnn_forward(gparams, spec, *oargs, device=dev)
    torch.cuda.synchronize()
    oms = (time.perf_counter() - t0) * 1e3 / args.oracle_steps
    ours = mod(b0['node_feat'], b0['L'], b0['L_cluster'], b0['L_cut'], mask=b0['node_mask'])
    res['eager_fp32_oracle'] = {'ms_per_forward': oms, 'molecules_per_s': B / oms * 1e3,
                                'max_abs_diff_vs_dropin': float((ours - ref).abs().max())}
    res['speedup_vs_eager_oracle'] = oms / ms

  # 4. one training step at the reference's batch size: eager loop body and GraphedStep
  t = batch(args.train_batch, 7, dev)
  targs = (t['node_feat'], t['L'], t['L_cluster'], t['L_cut'])
  tm = GPNN(cfg)
  tm.load_state_dict(deterministic_state_dict(tm, 1234))
  tm = tm.to(dev).train()
  opt = torch.optim.Adam(tm.parameters(), lr=1e-4)

  def eager_step():
    opt.zero_grad()
    _, loss = tm(*targs, label=t['label'], mask=t['node_mask'])
    loss.backward()
    opt.step()

  eager_ms = event_ms(eager_step, args.train_steps)
  gstep = GraphedStep(tm, opt, targs, {'label': t['label'], 'mask': t['node_mask']})
  graphed_ms = event_ms(lambda: gstep(*targs, label=t['label'], mask=t['node_mask']), args.train_steps)
  res['train_step'] = {'B': args.train_batch, 'eager_ms': eager_ms, 'graphed_ms': graphed_ms}
  res['card'] = card()
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, 'w') as fh:
      json.dump(res, fh, indent=1)


if __name__ == '__main__':
  main()
