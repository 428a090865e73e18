"""Operators with long and uneven ELL rows, and a numpy restatement of graph_prepare's ELL layout, for
tests/test_gpu_long_ell_rows.py.  The convolution-stack kernel stages at most LB <= 255 ELL lines (one line =
one (channel, slot) pair, counted up to the tile's longest row of the channel) in shared memory and gathers
the rest from global memory; the molecule-like operators of the other sweeps (about four entries per row)
stay inside the budget.  These generators give every graph of a batch one row-length profile:

  dense     every pair of real nodes in every channel, the diagonal included (rows of length n)
  hub       about four entries per row, plus one or two hub nodes adjacent to every other node
  budget17  E1 = 16, the longest row of every channel exactly 17 entries: 272 lines
  budget19  the same with 19: 304 lines.  Both exceed 255, so some lines are never staged, and 17 * 19 = 323:
            a staging budget that splits neither case at a channel boundary splits a channel in one of them
  sparse    at most four entries per row
  empty     no real node

Values are signed, |v| in [0.25, 1], never zero.  This file checks the generators' invariants on the host."""
import numpy as np
import pytest

from lanczosnetwork_b200 import data

PROFILES = ('dense', 'hub', 'budget17', 'budget19', 'sparse', 'empty')


def _values(rng, shape):
  return (rng.uniform(0.25, 1.0, size=shape) * rng.choice([-1.0, 1.0], size=shape)).astype(np.float32)


def _cap_rows(rng, mask, longest):
  """Drop random entries of every row of mask [n, n] beyond `longest`."""
  for i in range(mask.shape[0]):
    cols = np.flatnonzero(mask[i])
    if len(cols) > longest:
      mask[i, rng.choice(cols, size=len(cols) - longest, replace=False)] = False
  return mask


def _graph_mask(rng, profile, n):
  """Non-zero pattern [n, n] of one channel of one graph."""
  if profile == 'dense':
    return np.ones((n, n), bool)
  sparse = rng.rand(n, n) < min(1.0, 4.0 / n)
  if profile == 'sparse':
    return _cap_rows(rng, sparse, 4)
  if profile == 'hub':
    for h in rng.choice(n, size=min(n, int(rng.randint(1, 3))), replace=False):
      sparse[h, :] = True
      sparse[:, h] = True
    return sparse
  longest = int(profile[len('budget'):])
  assert n >= longest, (profile, n)
  mask = _cap_rows(rng, sparse, longest)
  r = rng.randint(n)                                     # this channel's longest row, exactly `longest`
  mask[r] = False
  mask[r, rng.choice(n, size=longest, replace=False)] = True
  return mask


def operators(profiles, sizes, N, E1, seed):
  """L [B, N, N, E1] float32: graph b has sizes[b] real nodes and the row-length profile profiles[b] in
  every channel (a name from PROFILES; one name for every graph); zero outside the real nodes."""
  B = len(sizes)
  if isinstance(profiles, str):
    profiles = [profiles] * B
  rng = np.random.RandomState(seed)
  L = np.zeros((B, N, N, E1), np.float32)
  for b, (prof, n) in enumerate(zip(profiles, sizes)):
    n = int(n)
    if prof == 'empty' or n == 0:
      continue
    for e in range(E1):
      m = _graph_mask(rng, prof, n)
      L[b, :n, :n, e] = np.where(m, _values(rng, (n, n)), np.float32(0))
  return L


def mixed_tile(N):
  """(profiles, sizes) of a batch that the first-fit tile schedule packs into one tile: a dense graph,
  hub and sparse graphs of other sizes, and a graph without nodes (sum of sizes <= 128)."""
  profiles = ['sparse', 'dense', 'empty', 'hub', 'sparse', 'sparse', 'sparse']
  sizes = [N // 8 + 3, N // 2 - 4, 0, N // 8, N // 16, 5, 1]
  assert sum(sizes) <= 128
  return profiles, sizes


# ------------------------------------------------------------------------------------------
# graph_prepare's ELL rows, restated
# ------------------------------------------------------------------------------------------
def ell_rows(L, binarize=False):
  """lnb_graph_prepare's ELL rows of L [B, N, N, E1]: (val [B, E1, N(slot), N(row)], idx (uint8), ell_max
  [B, E1], n_eff [B]).  Row n of channel e lists the diagonal first (when non-zero), then the other
  non-zero columns ascending, then zero slots (value 0, column 0) up to ell_max[b, e], the longest row of
  the channel.  Slots past ell_max are not defined and hold 0 here."""
  B, N, _, E1 = L.shape
  val = np.zeros((B, E1, N, N), np.float32)
  idx = np.zeros((B, E1, N, N), np.uint8)
  emax = np.zeros((B, E1), np.int32)
  n_eff = np.zeros(B, np.int32)
  for b in range(B):
    for e in range(E1):
      for n in range(N):
        row = L[b, n, :, e]
        cols = np.flatnonzero(row)
        if len(cols) == 0:
          continue
        cols = np.concatenate([cols[cols == n], cols[cols != n]])
        val[b, e, :len(cols), n] = 1.0 if binarize else row[cols]
        idx[b, e, :len(cols), n] = cols
        emax[b, e] = max(emax[b, e], len(cols))
        n_eff[b] = max(n_eff[b], n + 1, cols.max() + 1)
  return val, idx, emax, n_eff


def lines(emax):
  """ELL lines of a tile of these graphs: the sum over channels of the channel's longest row."""
  return int(np.asarray(emax).max(axis=0).sum())


# ------------------------------------------------------------------------------------------
# generator invariants
# ------------------------------------------------------------------------------------------
def _row_lengths(L):
  return (L != 0).sum(axis=2)                            # [B, N, E1]


@pytest.mark.parametrize('profile', [p for p in PROFILES if p != 'empty'])
def test_profiles_keep_to_the_real_nodes_and_never_store_zero_by_value(profile):
  sizes = [20, 33, 19]
  L = operators(profile, sizes, 40, 3, seed=1)
  for b, n in enumerate(sizes):
    assert not L[b, n:].any() and not L[b, :, n:].any()
    nz = L[b, :n, :n][L[b, :n, :n] != 0]
    assert nz.size and np.abs(nz).min() >= 0.25 and np.abs(nz).max() <= 1.0
    assert (nz < 0).any() and (nz > 0).any()
  assert np.array_equal(L, operators(profile, sizes, 40, 3, seed=1))


def test_dense_rows_hold_every_real_pair():
  L = operators('dense', [128, 64, 1], 128, 2, seed=2)
  lens = _row_lengths(L)
  assert (lens[0] == 128).all() and (lens[1, :64] == 64).all() and (lens[1, 64:] == 0).all()
  assert (lens[2, 0] == 1).all() and (np.diagonal(L[0], axis1=0, axis2=1) != 0).all()


def test_hub_rows_are_few_and_full():
  L = operators('hub', [128, 100], 128, 7, seed=3)
  lens = _row_lengths(L)
  for b, n in enumerate((128, 100)):
    for e in range(7):
      full = np.flatnonzero(lens[b, :n, e] == n)
      assert 1 <= len(full) <= 2, (b, e, full)
      assert (L[b, :n, full, e] != 0).all()             # the hubs' columns are full too
      assert np.median(lens[b, :n, e]) <= 8


@pytest.mark.parametrize('longest', [17, 19])
def test_budget_crossing_rows_exceed_every_staging_budget(longest):
  sizes = [64, 40, 23, 64]
  L = operators('budget%d' % longest, sizes, 64, 16, seed=longest)
  _, _, emax, _ = ell_rows(L)
  assert (emax == longest).all(), emax                  # every channel of every graph
  assert lines(emax) == 16 * longest > 255


def test_one_budget_crossing_case_splits_a_channel_at_every_budget():
  """build_tables stages min(tmax_e, lines left) lines of each channel in channel order, so a budget LB
  (1 <= LB <= 255) ends inside a channel of longest row t unless t divides LB."""
  for lb in range(1, 256):
    assert lb % 17 or lb % 19, lb


def test_control_rows_are_short():
  L = operators('sparse', [64, 30, 64], 64, 1, seed=4)
  assert _row_lengths(L).max() <= 4 and lines(ell_rows(L)[2]) <= 4


def test_mixed_tile_is_one_tile_of_the_first_fit_schedule():
  for N in (64, 128):
    profiles, sizes = mixed_tile(N)
    L = operators(profiles, sizes, N, 7, seed=N)
    n_eff = ell_rows(L)[3]
    assert (n_eff <= sizes).all() and n_eff[profiles.index('empty')] == 0
    assert _row_lengths(L)[profiles.index('dense')].max() == sizes[profiles.index('dense')]
    for K in (8, 32):                                    # with Ritz vectors on every real node
      sched = data.host_tile_schedule(sizes, np.minimum(sizes, K))
      assert sched[0] == 1 and sched[2] == len(sizes), sched


def test_ell_restatement_orders_the_diagonal_first():
  L = np.zeros((1, 5, 5, 1), np.float32)
  L[0, 2, [0, 2, 4], 0] = [3, -1, 2]
  L[0, 4, [1, 3], 0] = [5, 6]
  val, idx, emax, n_eff = ell_rows(L)
  assert emax[0, 0] == 3 and n_eff[0] == 5
  assert idx[0, 0, :, 2].tolist() == [2, 0, 4, 0, 0] and val[0, 0, :, 2].tolist() == [-1, 3, 2, 0, 0]
  assert idx[0, 0, :, 4].tolist() == [1, 3, 0, 0, 0] and val[0, 0, :3, 4].tolist() == [5, 6, 0]
  assert ell_rows(L, binarize=True)[0][0, 0, :, 2].tolist() == [1, 1, 1, 0, 0]
