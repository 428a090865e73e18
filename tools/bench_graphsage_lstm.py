"""Inference throughput of LSTMGraphSAGE with ``agg_func: LSTM`` on QM8-shaped batches
(config/qm8_graphsage.yaml with the LSTM aggregator), one GPU, plus the training path's memory.

    python tools/bench_graphsage_lstm.py [--batch-size 1024] [--batches 2] [--steps 10] [--warmup 2] [--out r.json]

Workload: rotating synthetic QM8 batches (data.synthetic_qm8_samples + data.sage_collate, K = 40 neighbour
samples), resident on the device.  Reports, in one JSON document:
  * ms per forward and molecules/s with CUDA-graph replay (CUDA events around the timed window);
  * per-kernel device times from torch.profiler in a separate eager run, the lnb_sage_lstm_step launches
    (sage_lstm_step_kernel) per forward and per step;
  * the step kernel's fp32-equivalent rate: shape-derived FLOPs of the live sequences (nonempty = 1) over
    the profiled kernel time;
  * the same forward through the training formulation (train.sage_train) under no_grad, the in-repo
    baseline, and the largest score difference between the two paths;
  * peak device memory of one training step (forward + backward) at the reference's batch size (64);
  * the card's name and power limit, read in the same process.
Writes nothing into the tree unless --out points there."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from helpers import deterministic_state_dict  # noqa: E402
from lanczosnetwork_b200 import configs, data  # noqa: E402
from lanczosnetwork_b200.model import LSTMGraphSAGE  # noqa: E402
from lanczosnetwork_b200.train import sage_train  # noqa: E402


def card():
  out = {'name': torch.cuda.get_device_name(0)}
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    out['nvidia_smi'] = q
  except Exception as exc:      # the measurement stands; the record says the query failed
    out['nvidia_smi'] = 'query failed: %s' % exc
  return out


def lstm_flops(cfg, live_nodes, padded_nodes):
  """Cell-step GEMM FLOPs of one forward, from shapes: per layer, K steps of 2 * 4D * 2D per sequence (D
  for the x half only at t = 0), E1 sequences per node.  Returns (live sequences only, all sequences)."""
  m = cfg.model
  E1 = cfg.dataset.num_bond_type + 1
  K = m.num_sample_neighbors
  dims = [m.input_dim] + list(m.hidden_dim)
  per_seq = sum(2.0 * 4 * d * d * (2 * K - 1) for d in dims[:m.num_layer - 1])
  return per_seq * E1 * live_nodes, per_seq * E1 * padded_nodes


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch-size', type=int, default=1024)
  ap.add_argument('--batches', type=int, default=2)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=2)
  ap.add_argument('--train-batch', type=int, default=64)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_graphsage_lstm: needs a CUDA device')
  dev = torch.device('cuda:0')
  cfg = configs.qm8_graphsage(agg_func='LSTM')
  B = args.batch_size
  batches = []
  for i in range(args.batches):
    b = data.sage_collate(data.synthetic_qm8_samples(B, seed=1000 + i), cfg.model.num_sample_neighbors,
                          np.random.RandomState(i))
    batches.append({k: torch.from_numpy(b[k]).to(dev) for k in ('node_feat', 'nn_idx', 'nonempty_mask',
                                                                'node_mask')})
  N = int(batches[0]['node_feat'].shape[1])
  mod = LSTMGraphSAGE(cfg)
  mod.load_state_dict(deterministic_state_dict(mod, 1234))
  mod = mod.to(dev).eval()

  def step(i):
    b = batches[i % len(batches)]
    return mod(b['node_feat'], b['nn_idx'], b['nonempty_mask'], mask=b['node_mask'])

  live = float(batches[0]['nonempty_mask'].sum())
  res = {'workload': {'model': 'LSTMGraphSAGE', 'config': 'config/qm8_graphsage.yaml, agg_func LSTM', 'B': B,
                      'N': N, 'K': cfg.model.num_sample_neighbors, 'live_nodes': live,
                      'rotating_batches': args.batches}}
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

    # 2. per-kernel device times, eager launches, separate run (batch 0 only: its live-row count)
    mod.use_cuda_graph = False
    step(0)
    torch.cuda.synchronize()
    prof_steps = 3
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      for _ in range(prof_steps):
        step(0)
      torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
      t = getattr(ev, 'device_time_total', None)
      if t is None:
        t = ev.cuda_time_total
      if t > 0 and ev.count > 0:
        kernels[ev.key] = {'us_per_forward': t / prof_steps, 'launches_per_forward': ev.count / prof_steps}
    res['kernels'] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]['us_per_forward'])[:12])
    mod.use_cuda_graph = True
    lstm = [v for k, v in kernels.items() if 'sage_lstm_step_kernel' in k]
    lstm_us = sum(v['us_per_forward'] for v in lstm)
    lstm_launches = sum(v['launches_per_forward'] for v in lstm)
    f_live, f_all = lstm_flops(cfg, live, B * N)
    res['shape_arithmetic_not_measured'] = {'lstm_gflop_live_rows': f_live / 1e9, 'lstm_gflop_all_rows': f_all / 1e9}
    res['lstm_step'] = {
        'us_per_forward': lstm_us, 'launches_per_forward': lstm_launches,
        'us_per_step': lstm_us / lstm_launches if lstm_launches else None,
        'fp32_equiv_tflops_live_rows': f_live / (lstm_us * 1e-6) / 1e12 if lstm_us else None,
        'share_of_forward_device_time': lstm_us / sum(v['us_per_forward'] for v in kernels.values())}

    # 3. the training formulation under no_grad, same batch
    b0 = batches[0]
    ours = step(0)
    tr_args = (b0['node_feat'], None, b0['node_mask'])
    samples = (b0['nn_idx'], b0['nonempty_mask'])
    ref = sage_train(mod, *tr_args, samples=samples)
    torch.cuda.synchronize()
    a.record()
    for _ in range(2):
      sage_train(mod, *tr_args, samples=samples)
    e.record()
    torch.cuda.synchronize()
    tms = a.elapsed_time(e) / 2
    res['training_formulation_no_grad'] = {'ms_per_forward': tms, 'molecules_per_s': B / tms * 1e3,
                                           'max_abs_score_diff_vs_kernel_path': float((ours - ref).abs().max()),
                                           'score_scale': float(ref.abs().max())}
    res['speedup_vs_training_formulation'] = tms / ms

  # 4. peak memory of one training step at the reference's batch size
  bt = data.sage_collate(data.synthetic_qm8_samples(args.train_batch, seed=7), cfg.model.num_sample_neighbors,
                         np.random.RandomState(7))
  tb = {k: torch.from_numpy(bt[k]).to(dev) for k in ('node_feat', 'nn_idx', 'nonempty_mask', 'node_mask')}
  label = torch.randn(args.train_batch, 16, device=dev)
  mod.train()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats(dev)
  base = torch.cuda.memory_allocated(dev)
  a.record()
  _, loss = mod(tb['node_feat'], tb['nn_idx'], tb['nonempty_mask'], label=label, mask=tb['node_mask'])
  loss.backward()
  e.record()
  torch.cuda.synchronize()
  res['training_step'] = {'B': args.train_batch, 'N': int(tb['node_feat'].shape[1]),
                          'peak_mb_above_model': (torch.cuda.max_memory_allocated(dev) - base) / 1e6,
                          'ms_first_step': a.elapsed_time(e)}
  res['card'] = card()
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, 'w') as fh:
      json.dump(res, fh, indent=1)


if __name__ == '__main__':
  main()
