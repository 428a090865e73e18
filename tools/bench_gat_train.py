"""Training-step time of TrainableGAT on QM8-shaped batches (config/qm8_gat.yaml: 7 layers, 8 heads,
F = 16, dropout 0.0), one GPU.

    python tools/bench_gat_train.py [--batch-sizes 64,1024] [--steps 20] [--warmup 3] [--out result.json]

Workload per batch size: one synthetic QM8 batch (data.synthetic_qm8_batch, N = 26, attention bias from
data.gat_bias), resident on the device; a step is zero_grad, forward + MSE loss, backward and an SGD
update.  Reports, in one JSON document, per batch size:
  * the eager training step of TrainableGAT (CUDA events around the timed window);
  * the same step replayed through train.GraphedStep;
  * the eager fp32 oracle's autograd step (tests/gat_train_oracle.py, the differentiable form of
    oracle/gat_oracle.py: plain PyTorch, the reference's per-head formulation) on the same GPU;
  * per-kernel device times of one eager step from torch.profiler, and gat_attention_backward_kernel
    against gat_attention_kernel per layer;
and the card's name and power limit, read in the same process.  Writes nothing into the tree unless --out
points there."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench_gat import card  # noqa: E402
from helpers import deterministic_state_dict  # noqa: E402
from lanczosnetwork_b200 import configs, data  # noqa: E402
from lanczosnetwork_b200.model import TrainableGAT  # noqa: E402
from lanczosnetwork_b200.train import GraphedStep  # noqa: E402
from oracle import gat_oracle  # noqa: E402
import gat_train_oracle  # noqa: E402


def timed(fn, steps, warmup):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(steps):
    fn()
  e.record()
  torch.cuda.synchronize()
  return a.elapsed_time(e) / steps


def bench(cfg, B, args, dev):
  b = data.synthetic_qm8_batch(B, seed=1000)
  nf = torch.from_numpy(b['node_feat']).to(dev)
  L = torch.from_numpy(data.gat_bias(b['L'])).to(dev)
  mask = torch.from_numpy(b['node_mask']).to(dev)
  label = torch.from_numpy(b['label']).to(dev)
  N = int(L.shape[1])
  mod = TrainableGAT(cfg)
  params = deterministic_state_dict(mod, 1234)
  mod.load_state_dict(params)
  mod = mod.to(dev).train()
  opt = torch.optim.SGD(mod.parameters(), lr=1e-4)

  def eager_step():
    opt.zero_grad(set_to_none=True)
    _, loss = mod(nf, L, label=label, mask=mask)
    loss.backward()
    opt.step()

  res = {'B': B, 'N': N}
  res['eager_step_ms'] = timed(eager_step, args.steps, args.warmup)
  step = GraphedStep(mod, opt, (nf, L), {'label': label, 'mask': mask})
  res['graphed_step_ms'] = timed(lambda: step(nf, L, label=label, mask=mask), args.steps, args.warmup)

  spec = gat_oracle.make_spec(cfg.model.num_layer, cfg.model.num_heads, cfg.dataset.num_bond_type)
  p32 = {k: v.to(dev).float().requires_grad_(True) for k, v in params.items()}
  opt_o = torch.optim.SGD(list(p32.values()), lr=1e-4)

  def oracle_step():
    opt_o.zero_grad(set_to_none=True)
    s = gat_train_oracle.gat_forward(p32, spec, nf, L, mask, device=dev)
    torch.nn.functional.mse_loss(s, label).backward()
    opt_o.step()

  n_or = max(1, args.steps // 4)
  oracle_step()
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(n_or):
    oracle_step()
  torch.cuda.synchronize()
  res['fp32_oracle_autograd_step_ms'] = (time.perf_counter() - t0) * 1e3 / n_or
  res['oracle_over_graphed'] = res['fp32_oracle_autograd_step_ms'] / res['graphed_step_ms']

  from torch.profiler import ProfilerActivity, profile
  prof_steps = 5
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(prof_steps):
      eager_step()
    torch.cuda.synchronize()
  kernels = {}
  for ev in prof.key_averages():
    t = getattr(ev, 'device_time_total', None)
    if t is None:
      t = ev.cuda_time_total
    if t > 0 and ev.count > 0:
      kernels[ev.key] = {'us_per_step': t / prof_steps, 'launches_per_step': ev.count / prof_steps}
  res['kernels'] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]['us_per_step'])[:12])

  def per_layer(name):
    hits = [v for k, v in kernels.items() if name in k and (name != 'gat_attention_kernel' or 'backward' not in k)]
    us = sum(v['us_per_step'] for v in hits)
    n = sum(v['launches_per_step'] for v in hits)
    return us / n if n else None

  res['attention_us_per_layer'] = {'forward': per_layer('gat_attention_kernel'),
                                   'backward': per_layer('gat_attention_backward_kernel')}
  del step
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch-sizes', default='64,1024')
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_gat_train: needs a CUDA device')
  dev = torch.device('cuda:0')
  cfg = configs.qm8_gat()
  res = {'workload': {'model': 'TrainableGAT', 'config': 'config/qm8_gat.yaml', 'optimizer': 'SGD'},
         'runs': [bench(cfg, int(B), args, dev) for B in args.batch_sizes.split(',')]}
  res['card'] = card()
  print(json.dumps(res))
  if args.out:
    with open(args.out, 'w') as fh:
      json.dump(res, fh, indent=1)


if __name__ == '__main__':
  main()
