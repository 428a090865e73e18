"""GPNN's graph partition on the device (ops.spectral_partition) against the host partition of the
reference's collate, and the GPNN forward with device partitioning against operators passed in.

    python tools/bench_gpnn_partition.py [--batches 64 1024] [--iters 50]

  * device partition time at each batch size: CUDA events over a captured graph of one launch;
  * the GPNN forward (qm8_gpnn config, captured) given L_cluster / L_cut, and partitioning itself;
  * only if scipy and scikit-learn import: host time of the collate's per-graph partition, i.e.
    ``scipy.sparse.linalg.eigsh(L, k=P, which='LM', maxiter=N * 10000, tol=0, mode='normal')`` then
    ``sklearn.cluster.KMeans(n_clusters=P, random_state=1234).fit(V)``, on the same padded graphs.
Batches are data.synthetic_qm8_batch (QM8-shaped, N = 26).  Prints one JSON line per measurement.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lanczosnetwork_b200 import configs, data, ops  # noqa: E402
from lanczosnetwork_b200.model import GPNN  # noqa: E402


def graph_ms(fn, iters):
  """Mean ms per replay of fn captured as one CUDA graph."""
  fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    with torch.cuda.graph(g, stream=s):
      fn()
  torch.cuda.current_stream().wait_stream(s)
  for _ in range(3):
    g.replay()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    g.replay()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / iters


def event_ms(fn, iters):
  for _ in range(3):
    fn()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / iters


def host_ms(L0, P, limit=64):
  try:
    import scipy.sparse.linalg
    from sklearn.cluster import KMeans
  except ImportError:
    return None
  L0 = L0[:limit].astype(np.float64)
  t0 = time.perf_counter()
  for Lg in L0:
    N = Lg.shape[0]
    _, V = scipy.sparse.linalg.eigsh(Lg, k=P, which='LM', maxiter=N * 10000, tol=0, mode='normal')
    KMeans(n_clusters=P, random_state=1234).fit(V.real)
  return (time.perf_counter() - t0) * 1e3 / len(L0)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batches', type=int, nargs='+', default=[64, 1024])
  ap.add_argument('--iters', type=int, default=50)
  args = ap.parse_args()
  dev = torch.device('cuda:0')
  cfg = configs.qm8_gpnn()
  P = cfg.model.num_partition
  gpu = torch.cuda.get_device_name(dev)
  for B in args.batches:
    b = data.synthetic_qm8_batch(B, seed=5)
    L = torch.from_numpy(b['L']).to(dev)
    nf = torch.from_numpy(b['node_feat']).to(dev)
    mask = torch.from_numpy(b['node_mask']).to(dev)
    part_ms = graph_ms(lambda: ops.spectral_partition(L, P), args.iters)
    _, Lc, Lt, _ = ops.spectral_partition(L, P)
    torch.manual_seed(0)
    mod = GPNN(cfg).to(dev).eval()
    with torch.no_grad():
      given = event_ms(lambda: mod(nf, L, Lc, Lt, mask=mask), args.iters)
      device = event_ms(lambda: mod(nf, L, mask=mask), args.iters)
    per_graph = host_ms(b['L'][:, :, :, 0], P)
    print(json.dumps({'B': B, 'N': int(L.shape[1]), 'P': P, 'gpu': gpu,
                      'device_partition_ms': round(part_ms, 4),
                      'forward_given_operators_ms': round(given, 4),
                      'forward_device_partition_ms': round(device, 4),
                      'host_partition_ms_per_batch': None if per_graph is None else round(per_graph * B, 1)}))


if __name__ == '__main__':
  main()
