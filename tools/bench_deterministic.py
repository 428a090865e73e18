"""What reproducible training costs: the fp32-atomic segment sum (lnb_unsorted_segment_sum_forward) against
its exact, order-independent twin (lnb_unsorted_segment_sum_exact), and captured training steps with
torch.use_deterministic_algorithms off and on.
    python tools/bench_deterministic.py [--iters 200] [--steps 50] [--out r.json]
Reports, in one JSON document:
  * ms per ops.segment_sum_forward call (output and workspace allocation included) at the three shapes the
    training path sums, at B = 64 and 1024 molecules of N = 26 padded nodes:
      - embedding: the atom-embedding gradient, B N rows of 64 into the 70 atom ids;
      - neighbour_max: GraphSAGE Max's first-layer adjoint, B N E1 D scalars (E1 = 7, D = 64) into B N D;
      - lstm_gather: one LSTM-aggregator step's P[ids] adjoint, B N E1 rows of 4 D = 512 into B N rows;
  * ms per train.GraphedStep replay (Adam) at B = 64 for LanczosNet (the train_qm8 workload), GGNN and
    LSTMGraphSAGE, the step captured with the flag off and with it on;
  * the card's name and power limit, read in the same process.
CUDA events around each timed window.  Writes nothing into the tree unless --out points there."""
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
from lanczosnetwork_b200 import configs, data, ops, train  # noqa: E402
from lanczosnetwork_b200.model import GGNN, LanczosNet, LSTMGraphSAGE  # noqa: E402

N, E1 = 26, 7


def card():
  out = {'name': torch.cuda.get_device_name(0)}
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    out['nvidia_smi'] = q
  except Exception as exc:      # the measurement stands; the record says the query failed
    out['nvidia_smi'] = 'query failed: %s' % exc
  return out


def timed_ms(fn, iters, warmup=5):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / iters


def segment_shapes(B, dev, rng):
  """(data [1, rows, width], ids [1, rows], segments) of each training-path sum at B molecules."""
  D = 64
  nf = torch.from_numpy(data.collate(data.synthetic_qm8_samples(B, seed=B), 4, num_nodes=N)['node_feat'])
  emb = (torch.randn(1, B * N, D), nf.reshape(1, -1), 70)
  arg = torch.from_numpy(rng.randint(-1, N, (B, N, E1, D)))          # argmax node per (node, channel, feature)
  b = torch.arange(B).view(B, 1, 1, 1)
  f = torch.arange(D).view(1, 1, 1, D)
  seg = torch.where(arg >= 0, (b * N + arg) * D + f, -1)
  nmax = (torch.randn(1, B * N * E1 * D, 1), seg.reshape(1, -1), B * N * D)
  rows = torch.from_numpy(rng.randint(0, N, (B, N, E1))) + N * torch.arange(B).view(B, 1, 1)
  lstm = (torch.randn(1, B * N * E1, 4 * 128), rows.reshape(1, -1), B * N)
  return {k: (x.to(dev), i.to(dev), S) for k, (x, i, S) in
          (('embedding', emb), ('neighbour_max', nmax), ('lstm_gather', lstm))}


def graphed_step(name, deterministic, dev, B=64):
  samples = data.synthetic_qm8_samples(B, seed=5)
  if name == 'LSTMGraphSAGE':
    cfg = configs.qm8_graphsage(agg_func='LSTM')
    mod = LSTMGraphSAGE(cfg)
    c = data.sage_collate(samples, cfg.model.num_sample_neighbors, np.random.RandomState(0))
    args = tuple(torch.from_numpy(c[k]).to(dev) for k in ('node_feat', 'nn_idx', 'nonempty_mask'))
  else:
    mod = LanczosNet(configs.qm8_lanczos_net()) if name == 'LanczosNet' else GGNN(configs.qm8_ggnn())
    c = data.collate(samples, 20, num_nodes=N)
    args = (torch.from_numpy(c['node_feat']).to(dev), torch.from_numpy(c['L']).to(dev))
    if name == 'LanczosNet':
      args += (torch.from_numpy(c['D']).to(dev), torch.from_numpy(c['V']).to(dev))
  kw = {'label': torch.from_numpy(c['label']).to(dev), 'mask': torch.from_numpy(c['node_mask']).to(dev)}
  mod.load_state_dict(deterministic_state_dict(mod, 1234))
  mod = mod.to(dev)
  prev = torch.are_deterministic_algorithms_enabled()
  torch.use_deterministic_algorithms(deterministic)
  try:
    step = train.GraphedStep(mod, torch.optim.Adam(mod.parameters(), lr=1e-3), args, kw)
  finally:
    torch.use_deterministic_algorithms(prev)
  return lambda: step(*args, **kw)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=200)
  ap.add_argument('--steps', type=int, default=50)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_deterministic: needs a CUDA device')
  dev = torch.device('cuda:0')
  out = {'card': card(), 'segment_sum_ms': {}, 'graphed_step_ms': {}}
  rng = np.random.RandomState(0)
  for B in (64, 1024):
    for name, (x, ids, S) in segment_shapes(B, dev, rng).items():
      row = {'rows': int(x.shape[1]), 'width': int(x.shape[2]), 'segments': S}
      for exact in (False, True):
        row['exact' if exact else 'atomic'] = round(timed_ms(
            lambda: ops.segment_sum_forward(x, ids, S, exact=exact), args.iters), 4)
      row['exact_over_atomic'] = round(row['exact'] / row['atomic'], 2)
      out['segment_sum_ms']['%s_B%d' % (name, B)] = row
  for name in ('LanczosNet', 'GGNN', 'LSTMGraphSAGE'):
    steps = {flag: graphed_step(name, flag, dev) for flag in (False, True)}
    row = {}
    for rep in range(2):          # alternate the two captures so drift hits both
      for flag, fn in steps.items():
        key = 'deterministic' if flag else 'default'
        row[key] = min(row.get(key, 1e9), round(timed_ms(fn, args.steps, warmup=3), 4))
    row['ratio'] = round(row['deterministic'] / row['default'], 3)
    out['graphed_step_ms'][name + '_B64'] = row
  text = json.dumps(out, indent=1)
  print(text)
  if args.out:
    with open(args.out, 'w') as fh:
      fh.write(text + '\n')


if __name__ == '__main__':
  main()
