"""The drop-ins' records loop against their packed loop: forward_sparse from data.sparse_collate records
against forward_sparse from data.PackedMolecules blobs (no eigenpairs in either).

    python tools/bench_packed_dropins.py [--B 1024] [--steps 40] [--rounds 3] [--models GCN GGNN ...]

Per model (seeded weights, a split of 4 B QM8-shaped molecules from data.synthetic_qm8_samples, batches of B
random molecules), one JSON line with:
  * collate_records_ms / batch_packed_ms: host time per batch of data.sparse_collate(..., eigs=False) against
    PackedMolecules.batch into a pinned staging buffer (wall clock, best of 3 over the same index lists);
  * blob_bytes / records_bytes: the bytes each format ships per batch;
  * records_mol_s / records_pinned_mol_s / packed_mol_s: molecules per second of a loop that assembles every
    batch on the host and calls forward_sparse -- records: sparse_collate, torch.from_numpy, forward_sparse
    (pageable tensors); records_pinned: the same with every tensor copied to pinned memory first; packed:
    PackedMolecules.batch into one of two pinned staging buffers (a buffer is reused only after the forward
    that read it has finished), forward_sparse.  The three loops alternate, ``--rounds`` times ``--steps``
    batches each, and every loop ends in a device synchronise; the best round of each is reported, and the
    packed loop's ratio to each records loop.
A last line holds unpack_kernel_ms: lnb_records_unpack per batch (torch.profiler, after the timed loops).
The GPU's name and power limit go into every line.  Exits without a CUDA device.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from lanczosnetwork_b200 import configs, data, ops  # noqa: E402
from lanczosnetwork_b200 import model as models  # noqa: E402
from bench_sparse_dropins import gpu_info, profiled_kernel_ms  # noqa: E402

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
    'LanczosNet': lambda: models.LanczosNet(configs.qm8_lanczos_net()),
}
K = 20


def records_batch(samples, idx, key, pinned=False):
  sp = data.sparse_collate([samples[i] for i in idx], K, eigs=False)
  pin = (lambda t: t.pin_memory()) if pinned else (lambda t: t)
  out = {k: (pin(torch.from_numpy(v)) if isinstance(v, np.ndarray) else v) for k, v in sp.items()}
  out['sample_key'] = key
  return out


class PackedLoader(object):
  """PackedMolecules.batch into two pinned staging buffers, each reused once the forward that read it is done."""

  def __init__(self, pool, B, key):
    self.pool, self.key = pool, key
    self.stage = [torch.empty(pool.max_bytes(B), dtype=torch.uint8).pin_memory() for _ in range(2)]
    self.done = [None, None]
    self.i = 0

  def batch(self, idx):
    s = self.i
    self.i ^= 1
    if self.done[s] is not None:
      self.done[s].synchronize()
    b = self.pool.batch(idx, out=self.stage[s].numpy())
    return s, dict(b, blob=self.stage[s][:b['blob'].size], sample_key=self.key)

  def consumed(self, s):
    ev = torch.cuda.Event()
    ev.record()
    self.done[s] = ev


def run_records(mod, samples, idxs, key, pinned=False):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for idx in idxs:
    mod.forward_sparse(records_batch(samples, idx, key, pinned))
  torch.cuda.synchronize()
  return time.perf_counter() - t0


def run_packed(mod, loader, idxs):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for idx in idxs:
    s, b = loader.batch(idx)
    mod.forward_sparse(b)
    loader.consumed(s)
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


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, default=1024)
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--models', nargs='+', default=list(MODELS))
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_packed_dropins: needs a CUDA device')
  dev = torch.device('cuda:0')
  gpu = gpu_info()
  B = args.B
  samples = data.synthetic_qm8_samples(4 * B, seed=5)
  big = int(np.argmax([len(s['node_feat']) for s in samples]))
  pool = data.PackedMolecules(samples, K, eigs=False)
  rng = np.random.RandomState(0)
  idxs = []
  for _ in range(args.steps):
    idx = rng.randint(0, len(samples), size=B)
    idx[rng.randint(B)] = big                      # every batch pads to N = 26: one captured graph per loop
    idxs.append(idx)
  stage = torch.empty(pool.max_bytes(B), dtype=torch.uint8).pin_memory().numpy()
  host = {
      'collate_records_ms': round(best_wall_ms(lambda i: data.sparse_collate([samples[j] for j in i], K, eigs=False),
                                               idxs[:10]), 3),
      'batch_packed_ms': round(best_wall_ms(lambda i: pool.batch(i, out=stage), idxs[:10]), 3),
  }
  sp0 = data.sparse_collate([samples[j] for j in idxs[0]], K, eigs=False)
  host['records_bytes'] = int(sum(v.nbytes for k, v in sp0.items() if isinstance(v, np.ndarray) and k != 'label'))
  host['blob_bytes'] = int(pool.batch(idxs[0])['blob'].size)
  for name in args.models:
    torch.manual_seed(0)
    mod = MODELS[name]().to(dev).eval()
    key = torch.tensor([1234, 0], dtype=torch.int64)
    loader = PackedLoader(pool, B, key)
    row = dict({'model': name, 'B': B, 'N': 26, 'gpu': gpu}, **host)
    with torch.no_grad():
      # the same scores from both formats on the first batch, and both loops warmed up (captures)
      _, b = loader.batch(idxs[0])
      row['bit_equal'] = bool(torch.equal(mod.forward_sparse(b), mod.forward_sparse(records_batch(samples, idxs[0], key))))
      run_records(mod, samples, idxs[:3], key)
      run_records(mod, samples, idxs[:3], key, pinned=True)
      run_packed(mod, loader, idxs[:3])
      rec_t, pin_t, pk_t = [], [], []
      for _ in range(args.rounds):
        rec_t.append(run_records(mod, samples, idxs, key))
        pin_t.append(run_records(mod, samples, idxs, key, pinned=True))
        pk_t.append(run_packed(mod, loader, idxs))
      row['records_mol_s'] = round(B * len(idxs) / min(rec_t), 1)
      row['records_pinned_mol_s'] = round(B * len(idxs) / min(pin_t), 1)
      row['packed_mol_s'] = round(B * len(idxs) / min(pk_t), 1)
      row['packed_over_records'] = round(min(rec_t) / min(pk_t), 3)
      row['packed_over_records_pinned'] = round(min(pin_t) / min(pk_t), 3)
    print(json.dumps(row), flush=True)
  # the unpack kernel alone, profiled after the timed loops (the profiler slows the host)
  blob = torch.from_numpy(pool.batch(idxs[0])['blob']).to(dev)
  cap = (blob.numel() - data.packed_offsets(B, K).D) // 4
  print(json.dumps({'kernel': 'lnb_records_unpack', 'B': B, 'gpu': gpu, 'blob_bytes': host['blob_bytes'],
                    'unpack_kernel_ms': round(profiled_kernel_ms(
                        lambda: ops.records_unpack(blob, B, K, B * 26, cap), 50, ['records_unpack_kernel']), 4)}),
        flush=True)


if __name__ == '__main__':
  main()
