"""The captured training step fed from records against the one fed from packed batches with labels in the blob.

    python tools/bench_packed_train.py [--B 64 1024] [--steps 20] [--rounds 3] [--models GCN GGNN ...]

Per model and batch size (seeded weights, Adam, a split of 4 B QM8-shaped molecules from
data.synthetic_qm8_samples, batches of B random molecules that all pad to N = 26), one JSON line with:
  * collate_records_ms / batch_packed_ms: host time per batch of data.sparse_collate against
    PackedMolecules(..., labels=True).batch into a pinned buffer (wall clock, best of 3 over the same indices);
  * records_bytes / blob_bytes: the bytes each format ships per step, labels included;
  * records_mol_s / packed_mol_s: molecules per second of a training loop that assembles every batch on the
    host and runs the captured step -- records: sparse_collate, torch.from_numpy (pageable tensors),
    GraphedStep(sparse=True); packed: PackedMolecules.batch into one of two pinned buffers, each refilled once
    the ``input_consumed`` event of the step that read it has completed, GraphedStep(packed=True).  The two
    loops alternate, ``--rounds`` times ``--steps`` batches each, every loop ends in a device synchronise, and
    the best round of each is reported with the packed loop's ratio to the records loop;
  * step_ms: the packed step's replay alone on a device-resident blob (CUDA events, no host work), the
    device time both loops are bounded by.
The first line names the GPU, its power limit and its maximum SM clock.  Exits without a CUDA device.
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

from lanczosnetwork_b200 import configs, data, train  # noqa: E402
from lanczosnetwork_b200 import model as models  # noqa: E402

MODELS = {
    'GCN': lambda: models.GCN(configs.qm8_gcn()),
    'GCNFP': lambda: models.GCNFP(configs.qm8_gcn()),
    'DCNN': lambda: models.DCNN(configs.qm8_dcnn()),
    'ChebyNet': lambda: models.ChebyNet(configs.qm8_cheby_net()),
    'TrainableGAT': lambda: models.TrainableGAT(configs.qm8_gat()),
    'KeyedGAT': lambda: models.KeyedGAT(configs.qm8_gat(dropout=0.1)),
    'GGNN': lambda: models.GGNN(configs.qm8_ggnn()),
    'MPNN': lambda: models.MPNN(configs.qm8_mpnn()),
    'GPNN': lambda: models.GPNN(configs.qm8_gpnn()),
    'SampledGraphSAGE-Mean': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean')),
    'SampledGraphSAGE-Max': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='Max')),
    'SampledGraphSAGE-LSTM': lambda: models.SampledGraphSAGE(configs.qm8_graphsage(agg_func='LSTM')),
    'LanczosNet': lambda: models.LanczosNet(configs.qm8_lanczos_net()),
    'LanczosNet-eigs': lambda: models.LanczosNet(configs.qm8_lanczos_net()),
}
K, N = 20, 26


def gpu_line():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
  return {'gpu': out[0] if out else torch.cuda.get_device_name(0)}


def keys(name):
  return {'sample_key': torch.tensor([1234, 0], dtype=torch.int64)} if name.startswith('SampledGraphSAGE') else {}


def records_batch(samples, idx, eigs, extra):
  sp = data.sparse_collate([samples[i] for i in idx], K, eigs=eigs)
  out = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sp.items()}
  label = out.pop('label')
  return dict(out, **extra), label


class PackedLoader(object):
  """PackedMolecules.batch into two pinned buffers, each refilled once the step that read it has copied it."""

  def __init__(self, pool, B, extra):
    self.pool, self.extra = pool, extra
    self.stage = [torch.empty(pool.max_bytes(B), dtype=torch.uint8).pin_memory() for _ in range(2)]
    self.done = [None, None]
    self.i = 0

  def batch(self, idx):
    s = self.i
    self.i ^= 1
    if self.done[s] is not None:
      self.done[s].synchronize()
    b = self.pool.batch(idx, out=self.stage[s].numpy())
    return s, dict(b, blob=self.stage[s][:b['blob'].size], **self.extra)

  def consumed(self, s, event):
    self.done[s] = event


def run_records(step, samples, idxs, eigs, extra):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for idx in idxs:
    rec, label = records_batch(samples, idx, eigs, extra)
    step(rec, label=label)
  torch.cuda.synchronize()
  return time.perf_counter() - t0


def run_packed(step, loader, idxs):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for idx in idxs:
    s, b = loader.batch(idx)
    step(b)
    loader.consumed(s, step.input_consumed)
  torch.cuda.synchronize()
  return time.perf_counter() - t0


def best_wall_ms(fn, idxs, reps=3):
  best = None
  for _ in range(reps):
    t0 = time.perf_counter()
    for idx in idxs:
      fn(idx)
    t = (time.perf_counter() - t0) * 1e3 / len(idxs)
    best = t if best is None else min(best, t)
  return best


def replay_ms(step, iters=20):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  step.graph.replay()
  start.record()
  for _ in range(iters):
    step.graph.replay()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) / iters


def bench(name, B, steps, rounds, dev):
  eigs = name == 'LanczosNet-eigs'
  samples = data.synthetic_qm8_samples(4 * B, seed=5)
  big = int(np.argmax([len(s['node_feat']) for s in samples]))
  pool = data.PackedMolecules(samples, K, eigs=eigs, labels=True)
  rng = np.random.RandomState(0)
  idxs = []
  for _ in range(steps):
    idx = rng.randint(0, len(samples), size=B)
    idx[rng.randint(B)] = big                      # every batch pads to N = 26: one capture per loop
    idxs.append(idx)
  extra = keys(name)
  stage = torch.empty(pool.max_bytes(B), dtype=torch.uint8).pin_memory().numpy()
  row = {'model': name, 'B': B, 'N': N}
  row['collate_records_ms'] = round(best_wall_ms(
      lambda i: data.sparse_collate([samples[j] for j in i], K, eigs=eigs), idxs[:10]), 3)
  row['batch_packed_ms'] = round(best_wall_ms(lambda i: pool.batch(i, out=stage), idxs[:10]), 3)
  rec0, label0 = records_batch(samples, idxs[0], eigs, extra)
  row['records_bytes'] = int(sum(v.numel() * v.element_size() for k, v in rec0.items() if torch.is_tensor(v)) +
                             label0.numel() * 4)
  row['blob_bytes'] = int(pool.batch(idxs[0])['blob'].size)
  torch.manual_seed(0)
  mods = [MODELS[name]().to(dev) for _ in range(2)]
  mods[1].load_state_dict(mods[0].state_dict())
  opts = [torch.optim.Adam(m.parameters(), lr=1e-3) for m in mods]
  rec_step = train.GraphedStep(mods[0], opts[0], (rec0,), {'label': label0}, sparse=True, edge_capacity=4 * B * N)
  loader = PackedLoader(pool, B, extra)
  s, b0 = loader.batch(idxs[0])
  pk_step = train.GraphedStep(mods[1], opts[1], (b0,), packed=True)
  # the first step of both from the same weights: the same loss
  _, l_r = rec_step(rec0, label=label0)
  _, l_p = pk_step(b0)
  loader.consumed(s, pk_step.input_consumed)
  row['first_loss_equal'] = bool(torch.equal(l_r, l_p))
  run_records(rec_step, samples, idxs[:3], eigs, extra)
  run_packed(pk_step, loader, idxs[:3])
  rec_t, pk_t = [], []
  for _ in range(rounds):
    rec_t.append(run_records(rec_step, samples, idxs, eigs, extra))
    pk_t.append(run_packed(pk_step, loader, idxs))
  row['records_mol_s'] = round(B * len(idxs) / min(rec_t), 1)
  row['packed_mol_s'] = round(B * len(idxs) / min(pk_t), 1)
  row['packed_over_records'] = round(min(rec_t) / min(pk_t), 3)
  row['step_ms'] = round(replay_ms(pk_step), 3)
  row['status'] = int(pk_step.status.item())
  del rec_step, pk_step, mods, opts
  torch.cuda.empty_cache()
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, nargs='+', default=[64, 1024])
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--models', nargs='+', default=list(MODELS))
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_packed_train: needs a CUDA device')
  dev = torch.device('cuda:0')
  print(json.dumps(gpu_line()), flush=True)
  for B in args.B:
    for name in args.models:
      print(json.dumps(bench(name, B, args.steps, args.rounds, dev)), flush=True)


if __name__ == '__main__':
  main()
