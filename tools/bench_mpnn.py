"""Throughput of the MPNN drop-in on QM8-shaped batches (config/qm8_mpnn.yaml), one GPU.

    python tools/bench_mpnn.py [--batches 4] [--steps 20] [--warmup 3] [--out result.json]

Workload: rotating synthetic QM8 batches (data.synthetic_qm8_batch, B = 1024, N = 26), resident on the
device.  Reports, in one JSON document:
  * ms per forward and molecules/s with CUDA-graph replay (CUDA events around the timed window);
  * per-kernel device times from torch.profiler, in a separate eager run;
  * lnb_mpnn_update's fp32-equivalent rate on algorithmic FLOPs: gi = 2 rows 3D (64 E1 + E1) over the
    folded S / degree columns and gh = 2 rows 3D D (the zero gate blocks and the degree block's padding
    it also multiplies are not counted), from the profiled kernel time;
  * the eager fp32 oracle (oracle/mpnn_oracle.py, plain PyTorch: the edge MLP on every bond, Set2Vec graph
    by graph as in the reference) on the same GPU;
  * a training step at B = 64, eager and under train.GraphedStep;
  * the card's name and power limit, read in the same process.
Writes nothing into the tree unless --out points there."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from helpers import deterministic_state_dict  # noqa: E402
from lanczosnetwork_b200 import configs, data, ops  # noqa: E402
from lanczosnetwork_b200.model import MPNN  # noqa: E402
from lanczosnetwork_b200.train import GraphedStep  # noqa: E402
from oracle import mpnn_oracle  # noqa: E402


def card():
  out = {'name': torch.cuda.get_device_name(0)}
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    out['nvidia_smi'] = q
  except Exception as exc:      # the measurement stands; the record says the query failed
    out['nvidia_smi'] = 'query failed: %s' % exc
  return out


def update_flops(B, N, D, E1):
  """Algorithmic FLOPs of one update launch: gi = [S | deg] F^T and gh = h W_hh^T (shapes, not measured)."""
  return 2.0 * B * N * (3 * D) * (ops.MPNN_EDGE_HIDDEN * E1 + E1), 2.0 * B * N * D * (3 * D)


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
  ap.add_argument('--oracle-steps', type=int, default=1)
  ap.add_argument('--train-batch', type=int, default=64)
  ap.add_argument('--train-steps', type=int, default=10)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_mpnn: needs a CUDA device')
  dev = torch.device('cuda:0')
  cfg = configs.qm8_mpnn()
  B = args.batch_size
  batches = []
  for i in range(args.batches):
    b = data.synthetic_qm8_batch(B, seed=1000 + i)
    batches.append({k: torch.from_numpy(b[k]).to(dev) for k in ('node_feat', 'L', 'node_mask')})
  N, E1 = int(batches[0]['L'].shape[1]), int(batches[0]['L'].shape[3])
  D, P = cfg.model.hidden_dim, cfg.model.num_prop
  mod = MPNN(cfg)
  params = deterministic_state_dict(mod, 1234)
  mod.load_state_dict(params)
  mod = mod.to(dev).eval()

  def step(i):
    b = batches[i % len(batches)]
    return mod(b['node_feat'], b['L'], mask=b['node_mask'])

  res = {'workload': {'model': 'MPNN', 'config': 'config/qm8_mpnn.yaml', 'B': B, 'N': N, 'hidden': D,
                      'num_prop': P, 'num_step_set2vec': cfg.model.num_step_set2vec,
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
    upd_us = sum(v['us_per_forward'] for k, v in kernels.items() if 'MpnnUpdatePolicy' in k)
    gi, gh = update_flops(B, N, D, E1)
    res['shape_arithmetic_not_measured'] = {'update_gi_gflop_per_step': gi / 1e9,
                                            'update_gh_gflop_per_step': gh / 1e9}
    res['rates'] = {'update_kernel_us_per_forward': upd_us,
                    'update_fp32_equiv_tflops': P * (gi + gh) / (upd_us * 1e-6) / 1e12 if upd_us else None}

    # 3. eager fp32 oracle (plain PyTorch) on the same GPU
    spec = mpnn_oracle.make_spec(P, cfg.model.aggregate_type, cfg.model.msg_func, cfg.dataset.num_bond_type,
                                 cfg.model.num_step_set2vec)
    gparams = {k: v.to(dev) for k, v in params.items()}
    b0 = batches[0]
    ref = mpnn_oracle.mpnn_forward(gparams, spec, b0['node_feat'], b0['L'], b0['node_mask'], device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.oracle_steps):
      mpnn_oracle.mpnn_forward(gparams, spec, b0['node_feat'], b0['L'], b0['node_mask'], device=dev)
    torch.cuda.synchronize()
    oms = (time.perf_counter() - t0) * 1e3 / args.oracle_steps
    ours = mod(b0['node_feat'], b0['L'], mask=b0['node_mask'])
    res['eager_fp32_oracle'] = {'ms_per_forward': oms, 'molecules_per_s': B / oms * 1e3,
                                'max_abs_diff_vs_dropin': float((ours - ref).abs().max())}
    res['speedup_vs_eager_oracle'] = oms / ms

  # 4. one training step at the reference's batch size: eager loop body and GraphedStep
  tb = data.synthetic_qm8_batch(args.train_batch, seed=7)
  t = {k: torch.from_numpy(tb[k]).to(dev) for k in ('node_feat', 'L', 'node_mask', 'label')}
  tm = MPNN(cfg)
  tm.load_state_dict(deterministic_state_dict(tm, 1234))
  tm = tm.to(dev).train()
  opt = torch.optim.Adam(tm.parameters(), lr=1e-4)

  def eager_step():
    opt.zero_grad()
    _, loss = tm(t['node_feat'], t['L'], label=t['label'], mask=t['node_mask'])
    loss.backward()
    opt.step()

  eager_ms = event_ms(eager_step, args.train_steps)
  gstep = GraphedStep(tm, opt, (t['node_feat'], t['L']), {'label': t['label'], 'mask': t['node_mask']})
  graphed_ms = event_ms(lambda: gstep(t['node_feat'], t['L'], label=t['label'], mask=t['node_mask']),
                        args.train_steps)
  res['train_step'] = {'B': args.train_batch, 'eager_ms': eager_ms, 'graphed_ms': graphed_ms}
  res['card'] = card()
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, 'w') as fh:
      json.dump(res, fh, indent=1)


if __name__ == '__main__':
  main()
