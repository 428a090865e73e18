"""The device's tile schedule (tile_assign_kernel, behind the next-fit table) is the host's
data.host_tile_schedule, on the dense and on the sparse prepare path.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import data

pytestmark = pytest.mark.gpu


def dev():
  return torch.device('cuda:0')


def ops():
  from lanczosnetwork_b200 import ops as _ops
  return _ops


def _schedule(prep, B):
  tiles = prep[4].cpu().numpy()
  return tiles[:B + 2], tiles[B + 2:B + 2 + 2 * B + 2]


def _check(prep, B, sizes=None, k_eff=None):
  gext = prep[3].cpu().numpy()
  table, sched = _schedule(prep, B)
  T = int(sched[0])
  want = data.host_tile_schedule(gext[:, 0], gext[:, 1])
  assert np.array_equal(sched[:T + 2 + B], want[:T + 2 + B])
  Tn = int(table[0])                           # the next-fit table is still there (entries past T + 1 undefined)
  assert np.array_equal(table[:Tn + 2], data.host_tile_table(gext[:, 0], gext[:, 1])[:Tn + 2])
  if sizes is not None:                        # the extents the host measures give the same schedule
    assert np.array_equal(want, data.host_tile_schedule(sizes, k_eff))
  return T


def _sparse(sp):
  t = {k: torch.from_numpy(v).to(dev()) for k, v in sp.items() if isinstance(v, np.ndarray)}
  return ops().graph_prepare_sparse(t['sizes'], t['node_ptr'], t['node_feat'], t['edge_ptr'], t['edges'],
                                    t['V_rows'], sp['N'], sp['num_edgetype'] + 1)[0]


def test_device_schedule_is_the_host_schedule_on_the_bench_batches():
  for seed in range(1000, 1008):
    samples = data.synthetic_qm8_samples(1024, seed)
    dense = data.collate(samples, 20)
    sp = data.sparse_collate(samples, 20)
    k_eff = data.ritz_extents(sp['V_rows'], sp['node_ptr'])
    prep_d = ops().graph_prepare(torch.from_numpy(dense['L']).to(dev()), torch.from_numpy(dense['V']).to(dev()))
    T = _check(prep_d, 1024, sp['sizes'], k_eff)
    assert T <= 130
    prep_s = _sparse(sp)
    _check(prep_s, 1024, sp['sizes'], k_eff)
    s0 = 1024 + 2                                # the schedules of the two paths, word for word
    assert torch.equal(prep_s[4][s0:s0 + T + 2 + 1024], prep_d[4][s0:s0 + T + 2 + 1024])


def test_device_schedule_is_the_host_schedule_on_random_multigraphs():
  rng = np.random.RandomState(11)
  for B, seed in ((2, 1), (3, 2), (37, 3), (200, 77), (700, 5)):
    samples = data.synthetic_qm8_samples(B, seed=seed)
    dense = data.collate(samples, 20)
    sp = data.sparse_collate(samples, 20)
    k_eff = data.ritz_extents(sp['V_rows'], sp['node_ptr'])
    _check(ops().graph_prepare(torch.from_numpy(dense['L']).to(dev()), torch.from_numpy(dense['V']).to(dev())),
           B, sp['sizes'], k_eff)
    _check(_sparse(sp), B, sp['sizes'], k_eff)
  # random extents up to a whole tile: n_eff in [0, 128], k_eff in [0, 32] (not multiples of 4), E1 = 2
  for B, N, K in ((300, 128, 32), (64, 40, 12), (2000, 8, 8)):
    n = rng.randint(0, N + 1, size=B)
    k = np.minimum(rng.randint(0, K + 1, size=B), n)
    L = np.zeros((B, N, N, 2), np.float32)
    Q = np.zeros((B, N, K), np.float32)
    for b in range(B):
      if n[b]:
        L[b, np.arange(n[b]), np.arange(n[b]), :] = 1.0
      Q[b, :n[b], :k[b]] = rng.rand(n[b], k[b]) + 0.5
    _check(ops().graph_prepare(torch.from_numpy(L).to(dev()), torch.from_numpy(Q).to(dev())), B, n, k)


def test_schedule_falls_back_to_the_next_fit_tiles_beyond_the_fused_kernels_shapes():
  # K > 32: the fused kernels do not run this batch; the schedule is the table in graph order
  B, N, K = 50, 10, 36
  rng = np.random.RandomState(4)
  L = np.zeros((B, N, N, 2), np.float32)
  L[:, np.arange(N), np.arange(N), :] = 1.0
  Q = rng.rand(B, N, K).astype(np.float32)
  prep = ops().graph_prepare(torch.from_numpy(L).to(dev()), torch.from_numpy(Q).to(dev()))
  table, sched = _schedule(prep, B)
  T = int(table[0])
  assert int(sched[0]) == T and np.array_equal(sched[1:T + 2], table[1:T + 2])
  assert np.array_equal(sched[T + 2:T + 2 + B], np.arange(B))
