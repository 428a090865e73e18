"""Training-step time of KeyedGAT with dropout against TrainableGAT without, on QM8-shaped batches
(config/qm8_gat.yaml: 7 layers, 8 heads, F = 16), one GPU.

    python tools/bench_gat_dropout.py [--batch-sizes 64,1024] [--p 0.1] [--steps 20] [--warmup 3] [--out f.json]

Per batch size (one synthetic QM8 batch, N = 26, resident on the device; a step is zero_grad, forward + MSE
loss, backward and an SGD update), in one JSON document:
  * the train.GraphedStep replay of TrainableGAT at dropout 0 and of KeyedGAT at dropout p (its own key,
    advanced on the device every replay);
  * the eager fp32 oracle's autograd step with torch's F.dropout at the reference's three sites (plain
    PyTorch, the reference's per-head formulation) on the same GPU;
  * per-kernel device times of one eager KeyedGAT step from torch.profiler;
and the card's name, power limit and clocks, read in the same process.  Writes nothing into the tree unless
--out points there."""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench_gat import card  # noqa: E402
from bench_gat_train import timed  # noqa: E402
from helpers import deterministic_state_dict  # noqa: E402
from lanczosnetwork_b200 import configs, data  # noqa: E402
from lanczosnetwork_b200.model import KeyedGAT, TrainableGAT  # noqa: E402
from lanczosnetwork_b200.train import GraphedStep  # noqa: E402
from oracle import gat_oracle  # noqa: E402
from gat_train_oracle import _linear  # noqa: E402


def oracle_forward_torch_dropout(params, spec, node_feat, L, mask, p):
  """gat_train_oracle.gat_forward with the reference's F.dropout at its three sites (model/gat.py:149-163)."""
  B, N = node_feat.shape
  E, nl = spec['num_edgetype'], spec['num_layer']
  state = params['embedding.weight'][node_feat]
  for t in range(nl):
    h = []
    for jj in range(E + 1):
      for ii in range(spec['num_heads'][t]):
        k = '%d.%d.%d' % (t, jj, ii)
        x = F.dropout(state, p, training=True)
        Wh = _linear(params, 'filter.' + k, x.reshape(B * N, -1)).reshape(B, N, -1)
        s1, s2 = _linear(params, 'att_net_1.' + k, Wh), _linear(params, 'att_net_2.' + k, Wh)
        att = F.softmax(F.leaky_relu(s1 + s2.transpose(1, 2), negative_slope=0.2) + L[:, :, :, jj], dim=1)
        out = torch.bmm(F.dropout(att, p, training=True), F.dropout(Wh, p, training=True))
        out = out + params['bias_%d_%d_%d' % (ii, E, t)].view(1, 1, -1)
        h.append(out if t == nl - 1 else F.elu(out))
    state = torch.mean(torch.stack(h, dim=0), dim=0) if t == nl - 1 else torch.cat(h, dim=2)
  flat = state.reshape(B * N, -1)
  y = (torch.sigmoid(_linear(params, 'att_func.0', flat)) * _linear(params, 'output_func.0', flat)).reshape(B, N, -1)
  m = mask.bool()
  return torch.stack([y[b, m[b], :].mean(dim=0) for b in range(B)])


def graphed_ms(cls, cfg, batch, args):
  nf, L, mask, label = batch
  mod = cls(cfg)
  mod.load_state_dict(deterministic_state_dict(mod, 1234))
  mod = mod.to(nf.device).train()
  opt = torch.optim.SGD(mod.parameters(), lr=1e-4)
  step = GraphedStep(mod, opt, (nf, L), {'label': label, 'mask': mask})
  ms = timed(lambda: step(nf, L, label=label, mask=mask), args.steps, args.warmup)
  return ms, mod, opt


def bench(B, args, dev):
  b = data.synthetic_qm8_batch(B, seed=1000)
  nf = torch.from_numpy(b['node_feat']).to(dev)
  L = torch.from_numpy(data.gat_bias(b['L'])).to(dev)
  mask = torch.from_numpy(b['node_mask']).to(dev)
  label = torch.from_numpy(b['label']).to(dev)
  batch = (nf, L, mask, label)
  res = {'B': B, 'N': int(L.shape[1]), 'p': args.p}
  res['trainable_gat_p0_graphed_step_ms'], _, _ = graphed_ms(TrainableGAT, configs.qm8_gat(), batch, args)
  cfg = configs.qm8_gat(dropout=args.p)
  res['keyed_gat_graphed_step_ms'], mod, opt = graphed_ms(KeyedGAT, cfg, batch, args)
  res['keyed_over_p0'] = res['keyed_gat_graphed_step_ms'] / res['trainable_gat_p0_graphed_step_ms']

  spec = gat_oracle.make_spec(cfg.model.num_layer, cfg.model.num_heads, cfg.dataset.num_bond_type)
  p32 = {k: v.detach().clone().requires_grad_(True) for k, v in mod.state_dict().items()}
  opt_o = torch.optim.SGD(list(p32.values()), lr=1e-4)

  def oracle_step():
    opt_o.zero_grad(set_to_none=True)
    F.mse_loss(oracle_forward_torch_dropout(p32, spec, nf, L, mask, args.p), label).backward()
    opt_o.step()

  n_or = max(1, args.steps // 4)
  oracle_step()
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(n_or):
    oracle_step()
  torch.cuda.synchronize()
  res['fp32_oracle_torch_dropout_step_ms'] = (time.perf_counter() - t0) * 1e3 / n_or
  res['oracle_over_keyed_graphed'] = res['fp32_oracle_torch_dropout_step_ms'] / res['keyed_gat_graphed_step_ms']

  def eager_step():
    opt.zero_grad(set_to_none=True)
    _, loss = mod(nf, L, label=label, mask=mask)
    loss.backward()
    opt.step()

  from torch.profiler import ProfilerActivity, profile
  eager_step()
  torch.cuda.synchronize()
  prof_steps = 3
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
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch-sizes', default='64,1024')
  ap.add_argument('--p', type=float, default=0.1)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_gat_dropout: needs a CUDA device')
  dev = torch.device('cuda:0')
  res = {'workload': {'models': ['TrainableGAT dropout 0', 'KeyedGAT dropout %g' % args.p],
                      'config': 'config/qm8_gat.yaml', 'optimizer': 'SGD'},
         'runs': [bench(int(B), args, dev) for B in args.batch_sizes.split(',')]}
  res['card'] = card()
  print(json.dumps(res))
  if args.out:
    with open(args.out, 'w') as fh:
      json.dump(res, fh, indent=1)


if __name__ == '__main__':
  main()
