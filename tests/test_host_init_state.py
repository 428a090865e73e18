"""CPU tests of the drop-in constructors: the seeded initial state of every class (state_dict keys, their
order, shapes and a digest of each tensor, against tests/golden/init_digests.json from
tests/golden/make_init_digests.py), the loss-name check, and DCNN's permuted weights following
``invalidate_caches``."""
import hashlib
import importlib.util
import json
import os

import pytest
import torch

from helpers import GOLDEN

_spec = importlib.util.spec_from_file_location('make_init_digests', os.path.join(GOLDEN, 'make_init_digests.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)

with open(os.path.join(GOLDEN, 'init_digests.json')) as _f:
  FIXTURE = json.load(_f)


@pytest.mark.parametrize('case', sorted(mk.CASES))
def test_seeded_initial_state_is_pinned(case):
  assert FIXTURE['seed'] == mk.SEED
  expected = FIXTURE['cases']['GAT' if case == 'TrainableGAT' else case]
  got = mk.init_state(case)
  assert [e[0] for e in got] == [e[0] for e in expected]           # keys and their order
  assert [e[1] for e in got] == [e[1] for e in expected]
  bad = [g[0] for g, e in zip(got, expected) if g[2] != e[2]]
  assert not bad, 'initial values changed: %s' % bad[:8]


@pytest.mark.parametrize('case', sorted(mk.CASES))
def test_unknown_loss_name_raises(case):
  with pytest.raises(ValueError, match='^Non-supported loss function!$'):
    mk.build(case, loss='Huber')


def test_dcnn_layer_weight_follows_invalidate_caches():
  """An edit through ``p.data`` bumps no version counter; invalidate_caches() must drop the permuted
  weight built from the old values."""
  from lanczosnetwork_b200 import configs
  from lanczosnetwork_b200.model import DCNN
  torch.manual_seed(0)
  mod = DCNN(configs.qm8_dcnn(num_layer=2, hidden_dim=[8, 8], diffusion_dist=[1, 2]))
  w = mod.filter[0].weight
  before = mod._layer_weight(0).clone()
  w.data.mul_(2.0)
  mod.invalidate_caches()
  after = mod._layer_weight(0)
  assert torch.equal(after, 2.0 * before)
  split = (mod.num_edgetype + 1) * (w.shape[1] // (mod.num_scale + mod.num_edgetype + 1))
  assert torch.equal(after, torch.cat([w.detach()[:, split:], w.detach()[:, :split]], dim=1))
