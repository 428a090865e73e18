"""The tile placement beside the filter-MLP chain changes no bit: the row list, the tile table and
schedule, the chain's coefficients and the scores equal those of the serial launch order (placement
inside graph_prepare, chain on every SM).  ``pytest -m gpu``."""
import contextlib

import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data

pytestmark = pytest.mark.gpu


def dev():
  return torch.device('cuda:0')


def ops():
  from lanczosnetwork_b200 import ops as _ops
  return _ops


@contextlib.contextmanager
def serial_order():
  """Every prepare writes its tiles itself, so the forward launches in the serial order."""
  o = ops()
  dense, sparse = o.graph_prepare, o.graph_prepare_sparse
  o.graph_prepare = lambda L, Q=None, binarize=False, defer_tiles=False: dense(L, Q, binarize)
  o.graph_prepare_sparse = lambda *a, defer_tiles=False, **kw: sparse(*a, **kw)
  try:
    yield
  finally:
    o.graph_prepare, o.graph_prepare_sparse = dense, sparse


def _defined_tiles(prep, B):
  """The words of `tiles` the fused kernels read: the next-fit table, and for B >= 2 the schedule."""
  t = prep[4].cpu()
  out = [t[:int(t[0]) + 2]]
  if B >= 2:
    s = t[B + 2:]
    out.append(s[:int(s[0]) + 2 + B])
  return out


def _assert_same_prep(a, b, B):
  assert torch.equal(a[3], b[3])
  assert torch.equal(a.nrows, b.nrows)
  n = int(a.nrows.item())
  assert torch.equal(a.rowmap[:n], b.rowmap[:n])
  for x, y in zip(_defined_tiles(a, B), _defined_tiles(b, B)):
    assert torch.equal(x, y)


def _deferred(prep, K):
  """Place the tiles of a deferred prepare on a side stream, joined back as the forward does."""
  assert prep.tiles_pending
  cur, side = torch.cuda.current_stream(), torch.cuda.Stream()
  side.wait_stream(cur)
  with torch.cuda.stream(side):
    ops().tile_assign(prep, K)
  cur.wait_stream(side)
  assert not prep.tiles_pending
  return prep


@pytest.mark.parametrize('B', [1024, 5, 1])
def test_deferred_prepare_writes_the_same_rows_and_tiles(B):
  samples = data.synthetic_qm8_samples(B, seed=70 + B)
  dense = data.collate(samples, 20)
  L, V = torch.from_numpy(dense['L']).to(dev()), torch.from_numpy(dense['V']).to(dev())
  serial = ops().graph_prepare(L, V)
  _assert_same_prep(_deferred(ops().graph_prepare(L, V, defer_tiles=True), 20), serial, B)
  sp = data.sparse_collate(samples, 20)
  t = {k: torch.from_numpy(v).to(dev()) for k, v in sp.items() if isinstance(v, np.ndarray)}
  args = (t['sizes'], t['node_ptr'], t['node_feat'], t['edge_ptr'], t['edges'], t['V_rows'], sp['N'],
          sp['num_edgetype'] + 1)
  sparse = _deferred(ops().graph_prepare_sparse(*args, defer_tiles=True)[0], 20)
  _assert_same_prep(sparse, ops().graph_prepare_sparse(*args)[0], B)
  _assert_same_prep(sparse, serial, B)
  if B <= 1:                                    # no schedule: the fused kernels run the next-fit table
    gext = serial[3].cpu().numpy()
    assert np.array_equal(_defined_tiles(sparse, B)[0].numpy(),
                          data.host_tile_table(gext[:, 0], gext[:, 1])[:int(sparse[4][0]) + 2])


def test_chain_coefficients_do_not_depend_on_the_grid():
  from lanczosnetwork_b200.model import LanczosNet
  from lanczosnetwork_b200.spectral_conv import ritz_filter_coefficients
  mod = LanczosNet(configs.qm8_lanczos_net()).to(dev()).eval()
  dense = data.collate(data.synthetic_qm8_samples(1024, seed=5), 20)
  D = torch.from_numpy(dense['D']).to(dev())
  prep = ops().graph_prepare(torch.from_numpy(dense['L']).to(dev()), torch.from_numpy(dense['V']).to(dev()))
  rows = prep.rowmap[:int(prep.nrows.item())].long()
  mlp = mod._filter_mlp_params()
  sms = torch.cuda.get_device_properties(dev()).multi_processor_count
  with torch.no_grad():
    ref = ritz_filter_coefficients(D, mod.long_diffusion_dist, mlp, mod._wcache, prep)[0]
    ref = ref.reshape(ref.shape[0], -1, ref.shape[3])[:, rows]
    for ctas in (sms - 1, 37, 1):
      got = ritz_filter_coefficients(D, mod.long_diffusion_dist, mlp, mod._wcache, prep, ctas=ctas)[0]
      assert torch.equal(got.reshape(got.shape[0], -1, got.shape[3])[:, rows], ref), ctas


def _models():
  from helpers import deterministic_state_dict
  from lanczosnetwork_b200.model import LanczosNet
  mods = []
  for _ in range(2):
    m = LanczosNet(configs.qm8_lanczos_net())
    m.load_state_dict(deterministic_state_dict(m, 1234))
    mods.append(m.to(dev()).eval())
  return mods


@pytest.mark.parametrize('B', [1024, 5, 1])
def test_scores_equal_the_serial_launch_order(B):
  new, old = _models()
  samples = data.synthetic_qm8_samples(B, seed=90 + B)
  dense = data.collate(samples, 20)
  args = [torch.from_numpy(dense[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')]
  mask = torch.from_numpy(dense['node_mask']).to(dev())
  sp = data.sparse_collate(samples, 20)
  sparse = {k: (torch.from_numpy(v).to(dev()) if isinstance(v, np.ndarray) else v) for k, v in sp.items()}
  pk = data.pack_sparse(sp)
  packed = dict(pk, blob=torch.from_numpy(pk['blob']).pin_memory())

  def run(mod):
    with torch.no_grad():
      mod.use_cuda_graph = False
      out = [mod(*args, mask=mask), mod.forward_sparse(sparse), mod.forward_sparse(packed)]
      mod.use_cuda_graph = True            # slot graph, then the zero-copy graph of the resident inputs
      out += [mod(*args, mask=mask) for _ in range(3)]
      out += [mod.forward_sparse(sparse) for _ in range(2)] + [mod.forward_sparse(packed) for _ in range(2)]
    torch.cuda.synchronize()
    return out

  got = run(new)
  with serial_order():
    want = run(old)
  assert new._graph_stats['replays'] > 0 and new._graph_stats['captures'] > 0
  for i, (a, b) in enumerate(zip(got, want)):
    assert torch.equal(a, b), i
  assert all(torch.equal(a, got[0]) for a in got), 'forward_sparse differs from forward'
