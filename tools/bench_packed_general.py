"""SparseLanczosNetGeneral (config/graph_lanczos_net.yaml) fed from records against packed batches of float
feature rows.

    python tools/bench_packed_general.py [--B 64 1024] [--steps 20] [--rounds 3]
    python tools/bench_packed_general.py --profile [--B 64 1024]

Per batch size: seeded weights and a split of 2 B graphs of data.synthetic_regression_graphs (the reference's
GraphData set: G(n, 0.5), 20 <= n <= 100, 10 features), batches of B random graphs that all pad to the
split's largest n.  One JSON line per batch size with:
  * fwd_{records,packed}_{eigs,noeigs}_ms: forward_sparse under torch.no_grad from pinned host tensors built
    before the loop (records of data.sparse_collate, or the blob of pack_sparse), per batch;
  * step_{sparse,packed}_ms: GraphedStep(sparse=True) on pinned records with the label beside them against
    GraphedStep(packed=True) on pinned labelled blobs, Adam, per step;
  * h2d_{records,packed}_{eigs,noeigs}_{bytes,copies} and h2d_step_{sparse,packed}_{bytes,copies}: what
    each crosses to the device per call, counted from the tensors each copies;
  * host_{collate,batch}_ms: data.sparse_collate against PackedMolecules(..., labels=True).batch into a pinned
    buffer (wall clock, best of 3 over the same indices).
Every timed row runs ``--steps`` calls ending in a device synchronise; the rows alternate within each of
``--rounds`` repeats and the best repeat of each is reported.  ``--profile`` instead times the prepare kernel,
atom-id packed (LanczosNet's QM8 blob of the same B) against feature packed, with torch.profiler over 50
launches each.  The first line names the GPU and its power limit, read in the same call.  Exits without a
CUDA device.
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

from lanczosnetwork_b200 import configs, data, ops, train  # noqa: E402
from lanczosnetwork_b200.model import SparseLanczosNetGeneral  # noqa: E402

K = 20


def gpu_line():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
  return {'gpu': out[0] if out else torch.cuda.get_device_name(0)}


def pinned(d):
  return {k: (torch.from_numpy(v).pin_memory() if isinstance(v, np.ndarray) else v) for k, v in d.items()}


def h2d(d, skip=('label',)):
  ts = [v for k, v in d.items() if torch.is_tensor(v) and k not in skip]
  return sum(t.numel() * t.element_size() for t in ts), len(ts)


def best_wall_ms(fn, idxs, reps=3):
  best = None
  for _ in range(reps):
    t0 = time.perf_counter()
    for idx in idxs:
      fn(idx)
    t = (time.perf_counter() - t0) * 1e3 / len(idxs)
    best = t if best is None else min(best, t)
  return best


def timed(fn, calls):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for c in calls:
    fn(c)
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) * 1e3 / len(calls)


def split(B, steps):
  samples = data.synthetic_regression_graphs(2 * B, seed=5)
  big = int(np.argmax([len(s['node_feat']) for s in samples]))
  rng = np.random.RandomState(0)
  idxs = []
  for _ in range(steps):
    idx = rng.randint(0, len(samples), size=B)
    idx[rng.randint(B)] = big                    # every batch pads to one N: one capture per row
    idxs.append(idx)
  return samples, idxs


def model(dev):
  torch.manual_seed(0)
  return SparseLanczosNetGeneral(configs.graph_lanczos_net()).to(dev)


def bench(B, steps, rounds, dev):
  samples, idxs = split(B, steps)
  row = {'B': B, 'N': int(max(len(s['node_feat']) for s in samples))}
  rows = {}
  for eigs in (True, False):
    tag = 'eigs' if eigs else 'noeigs'
    recs = [pinned(data.sparse_collate([samples[i] for i in idx], K, eigs=eigs)) for idx in idxs]
    pks = [pinned(data.pack_sparse(data.sparse_collate([samples[i] for i in idx], K, eigs=eigs))) for idx in idxs]
    row['h2d_records_%s_bytes' % tag], row['h2d_records_%s_copies' % tag] = h2d(recs[0])
    row['h2d_packed_%s_bytes' % tag], row['h2d_packed_%s_copies' % tag] = h2d(pks[0])
    mod = model(dev).eval()
    rows['fwd_records_%s_ms' % tag] = (lambda m, r: lambda: timed(m.forward_sparse, r))(mod, recs)
    rows['fwd_packed_%s_ms' % tag] = (lambda m, p: lambda: timed(m.forward_sparse, p))(mod, pks)
  pool = data.PackedMolecules(samples, K, labels=True)
  trs = [pinned(data.sparse_collate([samples[i] for i in idx], K)) for idx in idxs]
  labels = [t.pop('label') for t in trs]
  tps = [pinned(pool.batch(idx)) for idx in idxs]
  row['h2d_step_sparse_bytes'], row['h2d_step_sparse_copies'] = h2d(dict(trs[0], label=labels[0]), skip=())
  row['h2d_step_packed_bytes'], row['h2d_step_packed_copies'] = h2d(tps[0])
  m_s, m_p = model(dev), model(dev)
  m_p.load_state_dict(m_s.state_dict())
  st_s = train.GraphedStep(m_s, torch.optim.Adam(m_s.parameters(), lr=1e-3), (trs[0],), {'label': labels[0]},
                           sparse=True, edge_capacity=B * row['N'] * (row['N'] + 1) // 2)
  st_p = train.GraphedStep(m_p, torch.optim.Adam(m_p.parameters(), lr=1e-3), (tps[0],), packed=True)
  _, l_s = st_s(trs[0], label=labels[0])
  _, l_p = st_p(tps[0])
  row['first_loss_equal'] = bool(torch.equal(l_s, l_p))
  sparse_calls = list(zip(trs, labels))
  rows['step_sparse_ms'] = lambda: timed(lambda c: st_s(c[0], label=c[1]), sparse_calls)
  rows['step_packed_ms'] = lambda: timed(st_p, tps)
  with torch.no_grad():
    for fn in rows.values():                         # warm-up: captures and first replays
      fn()
    best = {k: None for k in rows}
    for _ in range(rounds):
      for k, fn in rows.items():
        t = fn()
        best[k] = t if best[k] is None else min(best[k], t)
  row.update({k: round(v, 3) for k, v in best.items()})
  row['status'] = int(st_p.status.item())
  stage = torch.empty(pool.max_bytes(B), dtype=torch.uint8).pin_memory().numpy()
  row['host_collate_ms'] = round(best_wall_ms(lambda i: data.sparse_collate([samples[j] for j in i], K), idxs[:10]), 3)
  row['host_batch_ms'] = round(best_wall_ms(lambda i: pool.batch(i, out=stage), idxs[:10]), 3)
  return row


def profile(B, dev, iters=50):
  from torch.profiler import ProfilerActivity, profile as tprof
  samples, idxs = split(B, 1)
  feat = torch.from_numpy(data.pack_sparse(data.sparse_collate([samples[i] for i in idxs[0]], K))['blob']).to(dev)
  N = int(max(len(samples[i]['node_feat']) for i in idxs[0]))
  atom_sp = data.sparse_collate(data.synthetic_qm8_samples(B, seed=5), K)
  atom = torch.from_numpy(data.pack_sparse(atom_sp)['blob']).to(dev)
  runs = {'atom_id_packed': lambda: ops.graph_prepare_sparse_packed(atom, B, atom_sp['N'], 7, K, want_dense=False),
          'feature_packed': lambda: ops.graph_prepare_sparse_packed(feat, B, N, 2, K, want_dense=True, feature_dim=10)}
  out = {'B': B}
  for name, fn in runs.items():
    fn()
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
      for _ in range(iters):
        fn()
      torch.cuda.synchronize()
    us = [e.device_time_total / e.count for e in prof.key_averages() if 'batch_prepare_sparse_kernel' in e.key]
    out[name + '_us'] = round(us[0], 2) if us else None
  out['atom_id_shape'] = [B, int(atom_sp['N']), 7]
  out['feature_shape'] = [B, N, 2]
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, nargs='+', default=[64, 1024])
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--profile', action='store_true')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_packed_general: needs a CUDA device')
  dev = torch.device('cuda:0')
  print(json.dumps(gpu_line()), flush=True)
  for B in args.B:
    print(json.dumps(profile(B, dev) if args.profile else bench(B, args.steps, args.rounds, dev)), flush=True)


if __name__ == '__main__':
  main()
