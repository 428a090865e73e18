"""Host side of the device eigenpairs: records and batches without host eigenpairs, the graph key of
LanczosNet.forward_sparse for both batch forms, and the eigensolver ops' refusal of CPU tensors."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops, provider
from lanczosnetwork_b200.model import LanczosNet


def _samples(eigs):
  rng = np.random.RandomState(11)
  out = []
  for n in (5, 12, 26, 9):
    nf, adjs = data.synthetic_molecule(rng, n)
    out.append(data.prepare_graph(adjs, nf, label=rng.randn(1, 16), eigs=eigs))
  return out


def test_records_and_batch_without_eigenpairs():
  full, bare = _samples(True), _samples(False)
  for a, b in zip(full, bare):
    assert 'D_simple' not in b and 'V_simple' not in b
    assert set(a) - set(b) == {'D_simple', 'V_simple'}
    for k in b:
      assert np.array_equal(a[k], b[k]), k
  sp, sp0 = data.sparse_collate(full, 20), data.sparse_collate(bare, 20, eigs=False)
  assert 'D' not in sp0 and 'V_rows' not in sp0 and sp0['K'] == 20 and 'K' not in sp
  assert list(sp) == ['sizes', 'node_ptr', 'node_feat', 'edge_ptr', 'edges', 'D', 'V_rows', 'N', 'num_edgetype',
                      'label']
  for k in sp0:
    if k != 'K':
      assert np.array_equal(sp[k], sp0[k]) and np.asarray(sp[k]).dtype == np.asarray(sp0[k]).dtype, k
  # the dense collate still works from records without eigenpairs only where it needs none
  with pytest.raises(KeyError):
    data.collate(bare, 20)


class _KeyProbe(LanczosNet):
  """LanczosNet whose CUDA-graph front door records its key and inputs instead of running."""

  def _device(self):
    return torch.device('cpu')

  def _graph_forward(self, impl, inputs, extra_key=()):
    self.seen = (extra_key, inputs)
    return torch.zeros(1)


def _batch(sp):
  return {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sp.items()}


def test_forward_sparse_keys_the_two_batch_forms_apart():
  mod = _KeyProbe(configs.qm8_lanczos_net()).eval()
  sp = data.sparse_collate(_samples(True), 20)
  with torch.no_grad():
    mod.forward_sparse(_batch(sp))
    key, inputs = mod.seen
    assert key == ('sparse', sp['N'])                       # the existing form, keyed as before
    assert len(inputs) == 7 and inputs[5].tensor.shape == sp['V_rows'].shape
    assert inputs[2].capacity == 4 * sp['N'] and inputs[5].capacity == 4 * sp['N']
    mod.forward_sparse(_batch(data.sparse_collate(_samples(False), 20, eigs=False)))
    key0, inputs0 = mod.seen
  assert key0 == ('sparse_eigs', sp['N'], 20) and key0 != key
  assert len(inputs0) == 5 and inputs0[2].capacity == 4 * sp['N']


def test_eigensolver_ops_refuse_cpu_tensors():
  sp = _batch(data.sparse_collate(_samples(False), 20, eigs=False))
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.graph_eigs_sparse(sp['sizes'], sp['node_ptr'], sp['edge_ptr'], sp['edges'], sp['N'], 20)
  A = torch.eye(4).expand(2, 4, 4).contiguous()
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.sym_eigs(A, torch.tensor([4, 3], dtype=torch.int32), 4)
  with pytest.raises(RuntimeError, match='CUDA'):
    provider.exact_eigenpairs(A, torch.tensor([4, 3]), 4)


def test_eigensolver_kernels_do_not_spill():
  import os
  import re
  from lanczosnetwork_b200 import build
  log = os.path.join(build.HERE, 'build.log')
  if not os.path.exists(log):
    pytest.skip('no build.log: the library was not built in this tree')
  with open(log) as fh:
    txt = fh.read()
  reps = re.findall(r'Function properties for (\S*graph_eigs_kernel\S*)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores',
                    txt)
  assert len(reps) == 4, reps                   # warp / CTA variants of both producers
  assert all(int(s) == 0 for _, s in reps), reps
