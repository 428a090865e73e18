"""Cost of the reference's eigenpairs on the device against the host preprocessing it replaces.

    python tools/bench_graph_eigs.py [--reps 50] [--steps 50] [--out result.json]

Reports, in one JSON document:
  * lnb_graph_eigs_sparse at B = 1024 QM8-shaped molecules (data.synthetic_qm8_samples, K = 20) and
    lnb_sym_eigs at the synthetic-graph shape (dataset/get_graph_data.py: G(n, 0.5), 20 <= n <= 100,
    N = 100, K = 20): ms per launch from CUDA events around a captured graph of ``--reps`` launches;
  * the host eigh of the same batches (numpy fp64, one process): eigh alone, and with the L4
    construction and the |lambda| sort of data.get_graph_laplacian_eigs;
  * LanczosNet.forward_sparse per step (CUDA-graph replay, resident batch) with host eigenpairs against
    device eigenpairs, and the bytes each batch form ships;
  * the card's name, power limit and SM clock limit, read in the same process.
Writes nothing into the tree unless --out points there."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from helpers import deterministic_state_dict  # noqa: E402
from lanczosnetwork_b200 import configs, data, ops  # noqa: E402
from lanczosnetwork_b200.model import LanczosNet  # noqa: E402


def card():
  out = {'name': torch.cuda.get_device_name(0)}
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    out['nvidia_smi'] = q
  except Exception as exc:      # the measurement stands; the record says the query failed
    out['nvidia_smi'] = 'query failed: %s' % exc
  return out


def graph_ms(fn, reps):
  """ms per call of ``fn`` from CUDA events around one replay of a graph holding ``reps`` calls."""
  fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for _ in range(reps):
      fn()
  g.replay()
  torch.cuda.synchronize()
  times = []
  for _ in range(5):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    e.record()
    torch.cuda.synchronize()
    times.append(a.elapsed_time(e) / reps)
  return {'ms_median': float(np.median(times)), 'ms_min': float(min(times)), 'ms_max': float(max(times))}


def host_eigh_ms(adjs, repeats=3):
  """Host fp64 eigh of every graph's simple-graph L4: alone, and with L4 construction + |lambda| sort."""
  L4 = [data.get_laplacian(a) for a in adjs]
  alone, full = [], []
  for _ in range(repeats):
    t0 = time.perf_counter()
    for m in L4:
      np.linalg.eigh(m)
    alone.append(1e3 * (time.perf_counter() - t0))
    t0 = time.perf_counter()
    for a in adjs:
      data.get_graph_laplacian_eigs(a)
    full.append(1e3 * (time.perf_counter() - t0))
  return {'eigh_ms_min': min(alone), 'eigh_l4_sort_ms_min': min(full)}


def eig_gflop(sizes, K):
  """fp64 GFLOP of the algorithm from shapes (an estimate, not measured): 4/3 n^3 for the
  tridiagonalisation, about 6 n^3 for QL with the rotations accumulated (two sweeps per eigenvalue),
  4 n^2 k for the back-transform of the kept columns."""
  n = np.asarray(sizes, np.float64)
  k = np.minimum(n, K)
  return float(((4.0 / 3.0) * n ** 3 + 6.0 * n ** 3 + 4.0 * n ** 2 * k).sum() / 1e9)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch-size', type=int, default=1024)
  ap.add_argument('--synth-batch', type=int, default=64)
  ap.add_argument('--reps', type=int, default=50)
  ap.add_argument('--steps', type=int, default=50)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_graph_eigs: needs a CUDA device')
  dev = torch.device('cuda:0')
  K, B = 20, args.batch_size
  res = {'card': card()}

  # ---- QM8 shape: bond lists -> eigenpairs -------------------------------------------------------
  rng = np.random.RandomState(3)
  sizes = data.synthetic_qm8_sizes(rng, B)
  mols = [data.synthetic_molecule(rng, n) for n in sizes]
  bare = [data.prepare_graph(a, nf, eigs=False) for nf, a in mols]
  sp0 = data.sparse_collate(bare, K, eigs=False)
  t = {k: torch.from_numpy(v).to(dev) for k, v in sp0.items() if isinstance(v, np.ndarray)}
  rows = int(sp0['node_ptr'][-1])
  N = sp0['N']

  def qm8():
    ops.graph_eigs_sparse(t['sizes'], t['node_ptr'], t['edge_ptr'], t['edges'], N, K,
                          num_edgetype=sp0['num_edgetype'], rows=rows)

  _, _, st = ops.graph_eigs_sparse(t['sizes'], t['node_ptr'], t['edge_ptr'], t['edges'], N, K,
                                   num_edgetype=sp0['num_edgetype'], rows=rows)
  res['qm8'] = {'B': B, 'N': N, 'K': K, 'mean_atoms': float(np.mean(sizes)), 'status_nonzero': int((st != 0).sum()),
                'kernel': graph_ms(qm8, args.reps), 'algorithm_gflop_fp64_estimate': eig_gflop(sizes, K),
                'host': host_eigh_ms([a.sum(axis=2) for _, a in mols])}

  # ---- synthetic-graph shape: dense padded operators -> eigenpairs ---------------------------------
  srng = np.random.RandomState(123)
  ssizes = srng.randint(20, 101, size=args.synth_batch)
  sadj = []
  for n in ssizes:
    a = np.triu(srng.rand(n, n) < 0.5, 1).astype(np.float64)
    sadj.append(a + a.T)
  Ns = 100
  L = np.zeros((args.synth_batch, Ns, Ns, 2), np.float32)
  for b, a in enumerate(sadj):
    n = a.shape[0]
    L[b, :n, :n, 0] = data.get_laplacian(a)
    L[b, :n, :n, 1] = L[b, :n, :n, 0]
  Ld = torch.from_numpy(L).to(dev)
  sz = torch.from_numpy(ssizes.astype(np.int32)).to(dev)
  res['synthetic'] = {'B': args.synth_batch, 'N': Ns, 'K': K,
                      'kernel': graph_ms(lambda: ops.sym_eigs(Ld, sz, K), args.reps),
                      'algorithm_gflop_fp64_estimate': eig_gflop(ssizes, K), 'host': host_eigh_ms(sadj)}

  # ---- LanczosNet.forward_sparse with host against device eigenpairs -------------------------------
  samples = data.synthetic_qm8_samples(B, seed=3)
  sp = data.sparse_collate(samples, K)
  sp_dev = data.sparse_collate(samples, K, eigs=False)
  mod = LanczosNet(configs.qm8_lanczos_net())
  mod.load_state_dict(deterministic_state_dict(mod, 1234))
  mod = mod.to(dev).eval()
  forms = {}
  with torch.no_grad():
    for name, s in (('host_eigenpairs', sp), ('device_eigenpairs', sp_dev)):
      batch = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) and k != 'label' else v)
               for k, v in s.items() if k != 'label'}
      for _ in range(5):
        mod.forward_sparse(batch)
      torch.cuda.synchronize()
      times = []
      for _ in range(5):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
          mod.forward_sparse(batch)
        e.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(e) / args.steps)
      shipped = sum(v.nbytes for k, v in s.items() if isinstance(v, np.ndarray) and k != 'label')
      forms[name] = {'ms_per_step_median': float(np.median(times)), 'ms_min': float(min(times)),
                     'ms_max': float(max(times)), 'record_bytes': int(shipped)}
  res['forward_sparse'] = dict(forms, B=B, graph_stats=mod.graph_stats())
  txt = json.dumps(res, indent=1)
  print(txt)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as fh:
      fh.write(txt)


if __name__ == '__main__':
  main()
