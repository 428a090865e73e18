"""GPNN drop-in, host side: the oracle against the reference's own outputs and gradients
(tests/golden/gpnn_qm8.npz, make_gpnn_golden.py), the partition operators against the reference's
partitions, the module's parameter surface, its refusals and the drop-in rebinding, and the unmodified
reference runner feeding the drop-in.  No GPU needed."""
import hashlib
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from helpers import ROOT, deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, dropin
from lanczosnetwork_b200.model import GPNN
from oracle import gpnn_oracle

REF = '/root/reference'
SMALL = dict(hidden_dim=32, num_prop=3, num_prop_cluster=2, num_prop_cut=1, aggregate_type='sum',
             update_func='RNN', output_dim=16)
CASES = (('config', {}, 0), ('small', SMALL, 1))


def _spec(cfg):
  m = cfg.model
  return gpnn_oracle.make_spec(m.num_prop, m.num_prop_cluster, m.num_prop_cut, m.aggregate_type, m.update_func,
                               cfg.dataset.num_bond_type)


def _params(cfg, seed):
  return deterministic_state_dict(GPNN(cfg), seed)


@pytest.mark.parametrize('prefix,over,dseed', CASES, ids=['config', 'small'])
def test_oracle_reproduces_the_reference_scores_and_loss(prefix, over, dseed):
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  cfg = configs.qm8_gpnn(**over)
  params = _params(cfg, int(gp['weight_seed']) + dseed)
  L = g['L'].copy()
  for mask, key in ((g['node_mask'], '%s_score' % prefix), (None, '%s_score_nomask' % prefix)):
    s32 = gpnn_oracle.gpnn_forward(params, _spec(cfg), g['node_feat'], L, gp['L_cluster'], gp['L_cut'], mask)
    np.testing.assert_allclose(s32.numpy(), gp[key], rtol=2e-5, atol=1e-6, err_msg=key)
    s64 = gpnn_oracle.gpnn_forward(params, _spec(cfg), g['node_feat'], L, gp['L_cluster'], gp['L_cut'], mask,
                                   dtype=torch.float64)
    np.testing.assert_allclose(s64.numpy(), gp[key], rtol=1e-4, atol=2e-5, err_msg=key)
    if mask is not None:
      loss = torch.nn.functional.mse_loss(s32, torch.from_numpy(g['label']))
      want = float(gp['%s_loss' % prefix])
      assert abs(float(loss) - want) <= 1e-5 * abs(want)
  assert np.array_equal(L, g['L'])                          # the oracle binarises a copy


@pytest.mark.parametrize('prefix,over,dseed', CASES, ids=['config', 'small'])
def test_oracle_fp64_autograd_reproduces_the_reference_gradients(prefix, over, dseed):
  """The reference ran in fp32, so its digests carry fp32 rounding through the recurrent steps; the
  bounds are those of the GGNN oracle's test (scaled by the gradient's own size)."""
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  cfg = configs.qm8_gpnn(**over)
  params = {k: v.double().requires_grad_(True) for k, v in _params(cfg, int(gp['weight_seed']) + dseed).items()}
  score = gpnn_oracle.gpnn_forward(params, _spec(cfg), g['node_feat'], g['L'], gp['L_cluster'], gp['L_cut'],
                                   g['node_mask'], dtype=torch.float64, cast=False)
  loss = torch.nn.functional.mse_loss(score, torch.from_numpy(g['label']).double())
  loss.backward()
  want_loss = float(gp['grad_%s_loss' % prefix])
  assert abs(float(loss.detach()) - want_loss) <= 1e-5 * want_loss
  names = [k for k in gp if k.startswith('grad_%s|' % prefix)]
  assert sorted(k.split('|', 1)[1] for k in names) == sorted(params)
  for k in names:
    name = k.split('|', 1)[1]
    want = gp[k]
    got = gpnn_oracle.grad_digest({name: params[name].grad})[name]
    scale = max(np.sqrt(want[1]), 1e-12)
    assert abs(got[0] - want[0]) <= 1e-4 * scale * np.sqrt(params[name].numel()), (k, got[0], want[0])
    assert abs(got[1] - want[1]) <= 3e-4 * want[1] + 1e-12, (k, got[1], want[1])
    np.testing.assert_allclose(got[2:], want[2:], rtol=0, atol=1e-4 * scale, err_msg=k)


def test_partition_operators_equal_the_reference_partitions():
  """The collate's get_L_cluster_cut, restated batch-wise: bit-identical on the reference's own partitions
  (padded nodes, stored with label -1, have no edges, so any label gives the same operators)."""
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  L_simple = g['L'][:, :, :, 0]
  c, t = data.partition_operators(L_simple, gp['partition_labels'])
  assert c.dtype == np.float32 and t.dtype == np.float32
  assert np.array_equal(c, gp['L_cluster']) and np.array_equal(t, gp['L_cut'])
  c1, t1 = data.partition_operators(L_simple[3], gp['partition_labels'][3])
  assert np.array_equal(c1, c[3]) and np.array_equal(t1, t[3])
  # every node, padded ones included, keeps a unit self-loop when it has no edge in that operator
  pad = ~g['node_mask'].astype(bool)
  assert np.all(c[pad[:, :, None].repeat(26, 2) & np.eye(26, dtype=bool)[None]] == 1.0)
  with pytest.raises(ValueError):
    data.partition_operators(L_simple, gp['partition_labels'][:, :5])


def test_module_surface_matches_the_reference():
  gp = load_golden('gpnn_qm8.npz')
  cfg = configs.qm8_gpnn()
  m = GPNN(cfg)
  assert sum(p.numel() for p in m.parameters()) == int(gp['num_params'])
  assert list(m.state_dict().keys()) == gp['keys'].tolist()
  shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
  assert shapes['update_func.weight_ih'] == (384, 896) and shapes['update_func_partition.weight_ih'] == (384, 128)
  assert shapes['state_func.0.weight'] == (512, 384) and shapes['state_func.2.weight'] == (128, 512)
  assert shapes['msg_func.6.0.weight'] == (128, 128) and shapes['input_func.0.weight'] == (128, 64)
  torch.manual_seed(int(gp['init_seed']))
  init = GPNN(cfg)
  h = hashlib.sha256()
  for name, t in init.state_dict().items():
    h.update(name.encode())
    h.update(t.detach().contiguous().numpy().tobytes())
  assert h.hexdigest() == str(gp['init_sha256'])
  # the message MLPs keep PyTorch's default initialisation, state_func and both cells' biases are zero
  assert init.msg_func[0][0].bias.abs().sum() > 0 and not init.state_func[0].bias.any()
  for cell in (init.update_func, init.update_func_partition):
    assert not cell.bias_ih.any() and not cell.bias_hh.any()


def test_refusals():
  with pytest.raises(AssertionError):
    GPNN(configs.qm8_gpnn(num_layer=2))
  with pytest.raises(AssertionError):
    GPNN(configs.qm8_gpnn(aggregate_type='max'))
  with pytest.raises(ValueError):
    GPNN(configs.qm8_gpnn(loss='hinge'))
  nf, L, P = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 4, 7), torch.zeros(2, 4, 4)
  m = GPNN(configs.qm8_gpnn(**SMALL))
  for grad in (False, True):                      # CPU module: no fallback, in inference or training
    with pytest.raises(RuntimeError, match='no CPU'):
      with torch.set_grad_enabled(grad):
        m(nf, L, P, P)
  mlp = GPNN(configs.qm8_gpnn(update_func='MLP'))
  shapes = {k: tuple(v.shape) for k, v in mlp.state_dict().items()}
  assert shapes['update_func.0.weight'] == (128, 896) and shapes['update_func_partition.0.weight'] == (128, 128)
  with pytest.raises(TypeError, match='2 positional arguments but 3'):
    with torch.no_grad():
      mlp(nf, L, P, P)
  with pytest.raises(UnboundLocalError):
    with torch.no_grad():
      GPNN(configs.qm8_gpnn(msg_func='embedding'))(nf, L, P, P)


def test_dropin_rebinds_gpnn_for_test_and_training_runs():
  for training in (False, True):
    ns = types.ModuleType('fake_runner')
    ns.GPNN = 'ref'
    dropin.patch_namespace(ns, training=training)
    assert ns.GPNN is GPNN
  assert 'GPNN' in dropin.DROPIN_CLASSES and 'GPNN' not in dropin.OPT_IN_CLASSES


SCRIPT = r'''
import os, pickle, sys
import numpy as np
import torch
repo, ref, work = sys.argv[1], sys.argv[2], sys.argv[3]
sys.path.insert(0, repo); sys.path.insert(0, os.path.join(repo, 'tests'))
from lanczosnetwork_b200 import data, dropin
from lanczosnetwork_b200 import model as b200_models

rng = np.random.RandomState(7)
pre = os.path.join(work, 'data', 'QM8', 'preprocess'); os.makedirs(pre)
for i, n in enumerate([9, 14, 5, 20, 11, 17, 8, 13]):
  nf, adjs = data.synthetic_molecule(rng, n)
  rec = data.prepare_graph(adjs, nf, label=rng.randn(1, 16))
  rec['label_weight'] = np.ones((1, 16))
  pickle.dump(rec, open(os.path.join(pre, 'QM8_preprocess_test_%07d.p' % i), 'wb'))
pickle.dump({'mean': np.zeros(16), 'std': np.ones(16)}, open(os.path.join(work, 'data', 'QM8', 'QM8_meta.p'), 'wb'))

dropin.install(ref, compat=True)
import runner.qm8_runner as qr
assert qr.GPNN is b200_models.GPNN, qr.GPNN

os.chdir(work)
from utils.arg_helper import get_config
config = get_config(os.path.join(ref, 'config', 'qm8_gpnn.yaml'), exp_dir=os.path.join(work, 'exp'))
config.use_gpu = False
config.test.batch_size = 4
from helpers import deterministic_state_dict
params = deterministic_state_dict(b200_models.GPNN(config), 77)
ckpt = os.path.join(work, 'model_snapshot_best.pth')
torch.save({'model': params, 'optimizer': {}, 'step': 0}, ckpt)
config.test.test_model = ckpt

seen = {}
orig_forward = b200_models.GPNN.forward
def spy(self, node_feat, L, L_cluster, L_cut, label=None, mask=None):
  seen['cls'] = type(self)
  seen['args'] = (node_feat.shape, L.clone(), L_cluster.clone(), L_cut.clone())
  return orig_forward(self, node_feat, L, L_cluster, L_cut, label=label, mask=mask)
b200_models.GPNN.forward = spy

try:
  qr.QM8Runner(config).test()
except RuntimeError as exc:
  assert 'CUDA' in str(exc) and 'no CPU' in str(exc), exc
else:
  raise SystemExit('the forward ran without CUDA: there must be no CPU fallback')
assert seen['cls'] is b200_models.GPNN
(B, N), L, Lc, Lt = seen['args']
assert B == 4 and tuple(L.shape) == (4, N, N, 7) and tuple(Lc.shape) == (4, N, N) and tuple(Lt.shape) == (4, N, N)
# the collate's partition operators: L4 of the cluster / cut parts of the simple graph, self-loops on every node
assert torch.all(torch.diagonal(Lc, dim1=1, dim2=2) > 0) and torch.all(torch.diagonal(Lt, dim1=1, dim2=2) > 0)
assert torch.equal((Lc + Lt - torch.diag_embed(torch.diagonal(Lc + Lt, dim1=1, dim2=2)) != 0),
                   (L[..., 0] - torch.diag_embed(torch.diagonal(L[..., 0], dim1=1, dim2=2)) != 0))
print('RUNNER_OK cpu')
'''


@pytest.mark.skipif(not os.path.isdir(REF), reason='reference checkout not present')
def test_reference_runner_feeds_the_dropin(tmp_path):
  script = tmp_path / 'drive_runner.py'
  script.write_text(SCRIPT)
  work = tmp_path / 'work'
  work.mkdir()
  env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
  proc = subprocess.run([sys.executable, str(script), ROOT, REF, str(work)], capture_output=True, text=True,
                        timeout=600, env=env)
  assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
  assert 'RUNNER_OK' in proc.stdout
