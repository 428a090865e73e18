"""Training steps of the operator drop-ins from padded batches against forward_sparse_train from bond-list
records.

    python tools/bench_sparse_train.py [--B 64 1024] [--iters 20] [--models GCN GPNN ...]

Per model and batch size (seeded weights, data.synthetic_qm8_samples, N = 26, Adam), one JSON line with:
  * graphed_padded_ms / graphed_sparse_ms: one train.GraphedStep replay (forward, loss, backward, Adam)
    from pinned host memory, the copies into the captured buffers included: the padded batch of
    data.collate(..., num_nodes=N) against the records (GraphedStep(..., sparse=True)); CUDA events;
  * eager_padded_ms / eager_sparse_ms: the same step without capture, from device-resident inputs;
  * collate_padded_ms / collate_sparse_ms: the host collate alone (data.collate (+ data.gat_bias for GAT)
    vs data.sparse_collate), wall clock;
  * h2d_padded_bytes / h2d_sparse_bytes: bytes copied to the device per step (label included).
LanczosNet runs with the collate's eigenpairs on both sides, GPNN partitions on the device on both sides.
SampledGraphSAGE (K = 40) trains from data.sage_collate (numpy's draws) on the padded side and from records
with a sample_key (draws on the device) on the other.
The GPU's name and power limit go into every line.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lanczosnetwork_b200 import configs, data, train  # noqa: E402
from lanczosnetwork_b200 import model as models  # noqa: E402
from bench_sparse_dropins import event_ms, gpu_info, wall_ms  # noqa: E402

MODELS = {
    'LanczosNet': lambda: models.LanczosNet(configs.qm8_lanczos_net()),
    'GCN': lambda: models.GCN(configs.qm8_gcn()),
    'DCNN': lambda: models.DCNN(configs.qm8_dcnn()),
    'ChebyNet': lambda: models.ChebyNet(configs.qm8_cheby_net()),
    'TrainableGAT': lambda: models.TrainableGAT(configs.qm8_gat()),
    'GGNN': lambda: models.GGNN(configs.qm8_ggnn()),
    'MPNN': lambda: models.MPNN(configs.qm8_mpnn()),
    'GPNN': lambda: models.GPNN(configs.qm8_gpnn()),
    'SampledGraphSAGE-Mean': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean')),
    'SampledGraphSAGE-Max': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='Max')),
    'SampledGraphSAGE-LSTM': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='LSTM')),
}
K = 20
SAGE_K = 40


def sage_collate(samples):
  return data.sage_collate(samples, SAGE_K, np.random.RandomState(0))


def padded_batch(name, samples, N):
  """(args, kwargs) of the padded forward as numpy arrays, and the label."""
  if name.startswith('SampledGraphSAGE'):
    c = sage_collate(samples)
    return [c['node_feat'], c['nn_idx'], c['nonempty_mask']], {'mask': c['node_mask']}
  c = data.collate(samples, K, num_nodes=N)
  L = data.gat_bias(c['L']) if name == 'TrainableGAT' else c['L']
  args = [c['node_feat'], L] + ([c['D'], c['V']] if name == 'LanczosNet' else [])
  return args, {'mask': c['node_mask']}


def records(name, samples):
  sp = data.sparse_collate(samples, K, eigs=(name == 'LanczosNet'))
  if name.startswith('SampledGraphSAGE'):
    sp['sample_key'] = np.array([1234, 0], np.int64)
  return {k: v for k, v in sp.items() if k not in ('label', 'num_edgetype')}


def pinned(x):
  return torch.from_numpy(x).pin_memory() if isinstance(x, np.ndarray) else x


def nbytes(ts):
  return int(sum(t.numel() * t.element_size() for t in ts if torch.is_tensor(t)))


def run(name, B, iters, dev, gpu):
  samples = data.synthetic_qm8_samples(B, seed=5)
  rec_np = records(name, samples)
  N = int(rec_np['N'])
  args_np, kw_np = padded_batch(name, samples, N)
  label_np = data.sparse_collate(samples, K, eigs=False)['label']
  row = {'model': name, 'B': B, 'N': N, 'gpu': gpu}

  def fresh():
    torch.manual_seed(0)
    mod = MODELS[name]().to(dev).train()
    return mod, torch.optim.Adam(mod.parameters(), lr=1e-4)

  # eager steps from device-resident inputs
  label = torch.from_numpy(label_np).to(dev)
  args_d = [torch.from_numpy(a).to(dev) for a in args_np]
  kw_d = {k: torch.from_numpy(v).to(dev) for k, v in kw_np.items()}
  rec_d = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else v) for k, v in rec_np.items()}
  mod, opt = fresh()

  def eager(fwd):
    def step():
      opt.zero_grad(set_to_none=True)
      _, loss = fwd()
      loss.backward()
      opt.step()
    return step
  row['eager_padded_ms'] = round(event_ms(eager(lambda: mod(*args_d, label=label, **kw_d)), iters), 4)
  row['eager_sparse_ms'] = round(event_ms(eager(lambda: mod.forward_sparse_train(rec_d, label=label)), iters), 4)

  # captured steps from pinned host memory
  label_h = pinned(label_np)
  args_h = [pinned(a) for a in args_np]
  kw_h = {k: pinned(v) for k, v in kw_np.items()}
  rec_h = {k: pinned(v) for k, v in rec_np.items()}
  mod, opt = fresh()
  step = train.GraphedStep(mod, opt, args_h, dict(kw_h, label=label_h))
  row['graphed_padded_ms'] = round(event_ms(lambda: step(*args_h, label=label_h, **kw_h), iters), 4)
  mod, opt = fresh()
  step = train.GraphedStep(mod, opt, (rec_h,), {'label': label_h}, sparse=True)
  row['graphed_sparse_ms'] = round(event_ms(lambda: step(rec_h, label=label_h), iters), 4)

  row['h2d_padded_bytes'] = nbytes(args_h + list(kw_h.values()) + [label_h])
  row['h2d_sparse_bytes'] = nbytes(list(rec_h.values()) + [label_h])
  if name.startswith('SampledGraphSAGE'):
    row['collate_padded_ms'] = round(wall_ms(lambda: sage_collate(samples)), 2)
  elif name == 'TrainableGAT':
    row['collate_padded_ms'] = round(wall_ms(lambda: data.gat_bias(data.collate(samples, K, num_nodes=N)['L'])), 2)
  else:
    row['collate_padded_ms'] = round(wall_ms(lambda: data.collate(samples, K, num_nodes=N)), 2)
  row['collate_sparse_ms'] = round(wall_ms(lambda: data.sparse_collate(samples, K, eigs=(name == 'LanczosNet'))), 2)
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, nargs='+', default=[64, 1024])
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--models', nargs='+', default=list(MODELS))
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_sparse_train: needs a CUDA device')
  dev = torch.device('cuda:0')
  gpu = gpu_info()
  for B in args.B:
    for name in args.models:
      print(json.dumps(run(name, B, args.iters, dev, gpu)), flush=True)


if __name__ == '__main__':
  main()
