"""The tile schedule of the fused convolution stack (first-fit decreasing, data.host_tile_schedule /
tile_assign_kernel): against a plain one-graph-at-a-time first-fit decreasing, on the bench batches,
and inside a packed batch."""
import numpy as np
from hypothesis import given, settings, strategies as st

from lanczosnetwork_b200 import data


def first_fit_decreasing(sizes, k_eff, rows=128, graphs=32):
  """One graph at a time: n_eff descending, k_eff descending, index ascending; lowest tile that fits."""
  tiles = []                                     # [sum n, sum k, [graph ids]]
  for i in sorted(range(len(sizes)), key=lambda i: (-sizes[i], -k_eff[i], i)):
    for t in tiles:
      if t[0] + sizes[i] <= rows and t[1] + k_eff[i] <= rows and len(t[2]) < graphs:
        t[0] += sizes[i]
        t[1] += k_eff[i]
        t[2].append(i)
        break
    else:
      tiles.append([sizes[i], k_eff[i], [i]])
  return [t[2] for t in tiles]


def unpack(sched, B):
  T = int(sched[0])
  starts = sched[1:T + 2]
  ids = sched[T + 2:T + 2 + B]
  return T, starts, ids


@settings(max_examples=200, deadline=None)
@given(st.lists(st.tuples(st.integers(1, 128), st.integers(0, 64)), min_size=0, max_size=300))
def test_host_tile_schedule_is_first_fit_decreasing(graphs):
  sizes = np.array([g[0] for g in graphs], np.int32)
  k_eff = np.array([min(g[1], g[0]) for g in graphs], np.int64)
  B = len(graphs)
  sched = data.host_tile_schedule(sizes, k_eff)
  assert sched.shape == (2 * B + 2,) and sched.dtype == np.int32
  T, starts, ids = unpack(sched, B)
  assert starts[0] == 0 and starts[-1] == B and np.all(np.diff(starts) >= 1) and (T == 0) == (B == 0)
  assert np.array_equal(np.sort(ids), np.arange(B))          # every graph exactly once
  assert np.all(sched[T + 2 + B:] == 0)
  for t in range(T):
    g = ids[starts[t]:starts[t + 1]]
    assert len(g) <= 32
    if len(g) > 1:                                           # a lone graph always fits
      assert sizes[g].sum() <= 128 and k_eff[g].sum() <= 128
  ref = first_fit_decreasing(sizes.tolist(), k_eff.tolist())
  assert [ids[starts[t]:starts[t + 1]].tolist() for t in range(T)] == ref


def test_host_tile_schedule_of_empty_graphs_and_identical_graphs():
  # empty graphs (n_eff = k_eff = 0) only count against the 32-graph limit
  sched = data.host_tile_schedule(np.zeros(70, np.int32), np.zeros(70, np.int64))
  T, starts, ids = unpack(sched, 70)
  assert T == 3 and starts.tolist() == [0, 32, 64, 70] and ids.tolist() == list(range(70))
  # 33 identical graphs of 4 nodes: the Ritz-row limit (4 x 32 = 128) and the graph limit bind together
  sched = data.host_tile_schedule(np.full(33, 4, np.int32), np.full(33, 4, np.int64))
  T, starts, ids = unpack(sched, 33)
  assert T == 2 and starts.tolist() == [0, 32, 33]


def _bench_batch(seed, B=1024, K=20):
  sp = data.sparse_collate(data.synthetic_qm8_samples(B, seed), K)
  return sp, data.ritz_extents(sp['V_rows'], sp['node_ptr'])


def test_bench_batches_fit_one_wave_of_an_h100():
  """The bench rotates through seeds 1000..1007 at B = 1024, K = 20: the schedule fits the 132 SMs
  in one wave (the next-fit table needs 142-143 tiles, two waves)."""
  for seed in range(1000, 1008):
    sp, k_eff = _bench_batch(seed)
    sched = data.host_tile_schedule(sp['sizes'], k_eff)
    assert int(sched[0]) <= 130, (seed, int(sched[0]))
    assert int(data.host_tile_table(sp['sizes'], k_eff)[0]) > 132


@settings(max_examples=25, deadline=None)
@given(st.integers(1, 40), st.integers(0, 10 ** 6), st.sampled_from([4, 20]))
def test_pack_sparse_carries_the_tile_schedule(B, seed, K):
  samples = data.synthetic_qm8_samples(B, seed=seed)
  sp = data.sparse_collate(samples, K)
  blob = data.pack_sparse(sp)['blob']
  hdr = blob[:64].view(np.int32)
  seg = blob[hdr[11]:hdr[11] + 4 * data.tile_segment_ints(B)].view(np.int32)
  assert hdr[12] >= hdr[11] + 4 * data.tile_segment_ints(B)
  k_eff = data.ritz_extents(sp['V_rows'], sp['node_ptr'])
  assert np.array_equal(seg[:B + 2], data.host_tile_table(sp['sizes'], k_eff))
  assert np.array_equal(seg[B + 2:], data.host_tile_schedule(sp['sizes'], k_eff))
  # the segments behind it depend on (B, K) only
  assert (int(hdr[11]), int(hdr[12])) == data.packed_offsets(B, K)[5:7]
