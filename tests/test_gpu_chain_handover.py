"""The filter-MLP chain's operand hand-overs (tc_gemm.cuh, operand_from_acc): the first stage is
computed inside produce() and every later hidden stage's operand is written by the consumers from
the previous step's accumulators.  Checked against fp64 for the widths the bench shape does not
take (S = 1 / 4 with Hd = 32 / 64 leave A stages of the four-deep ring unwritten; S > 8 chains three
consumer hand-overs per item), with and without a row list: listed rows match fp64, the others keep
their sentinel, and two launches give the same bits.  ``pytest -m gpu``."""
import pytest
import torch

from test_gpu_conv_envelope import _assert_mlp, _mlp_layers, _mlp_raw, dev, mlp_ref, ops

pytestmark = pytest.mark.gpu

CASES = [(S, Hd) for S in (1, 4, 8) for Hd in (32, 64, 128)] + [(16, 96), (32, 128)]


@pytest.mark.parametrize('row_list', [False, True], ids=['all-rows', 'row-list'])
@pytest.mark.parametrize('S,Hd', CASES, ids=['S%d-Hd%d' % c for c in CASES])
def test_chain_handover_matches_fp64(S, Hd, row_list):
  from lanczosnetwork_b200 import spectral_conv as sc
  R, nl = 700, 3                         # 6 row tiles x 3 layers: CTAs with several items and a layer change
  g = torch.Generator().manual_seed(100 * S + Hd + int(row_list))
  layers = _mlp_layers(g, nl, S, Hd)
  table = (torch.rand(R, S, generator=g) * 2 - 1).to(dev())
  w_hi, w_lo, bias_all = sc.WeightCache().split_mlp_chain('chain', layers)
  ref = mlp_ref(table, layers)
  if row_list:
    n = 411
    perm = torch.randperm(R, generator=g).int().to(dev())
    rowmap = torch.full((R,), -3, dtype=torch.int32, device=dev())
    rowmap[:n] = perm[:n]
    nrows = torch.tensor([n], dtype=torch.int32, device=dev())
    listed = torch.zeros(R, dtype=torch.bool, device=dev())
    listed[perm[:n].long()] = True
  else:
    rowmap = nrows = None
    listed = torch.ones(R, dtype=torch.bool, device=dev())
  sentinel = torch.full((nl, R, S), -4321.0, device=dev())
  out = _mlp_raw(table, w_hi, w_lo, bias_all, nl, rowmap, nrows, sentinel.clone())
  again = _mlp_raw(table, w_hi, w_lo, bias_all, nl, rowmap, nrows, sentinel.clone())
  what = 'S=%d Hd=%d row_list=%s' % (S, Hd, row_list)
  assert torch.equal(out, again), what
  assert torch.equal(out[:, ~listed], sentinel[:, ~listed]), what
  _assert_mlp(out[:, listed], ref[:, listed], what)
  if not row_list:                       # the plain entry point writes the same bits
    assert torch.equal(ops().ritz_filter_mlp(table, w_hi, w_lo, bias_all, nl), out), what
