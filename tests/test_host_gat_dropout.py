"""KeyedGAT without a GPU: its surface and initial weights are GAT's, its key buffer stays out of the
state_dict (reference checkpoints load), the drop-in binds it only with --opt-in GAT --keyed-dropout, its key
checks fire before any device work, and the torch restatement of the mask rule (gat_dropout_oracle) agrees
word for word with the numpy Philox of sage_sample_oracle."""
import types

import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict
from lanczosnetwork_b200 import configs, dropin, ops, train
from lanczosnetwork_b200.model import GAT, KeyedGAT, TrainableGAT

import gat_dropout_oracle as oracle
import sage_sample_oracle

SMALL = dict(num_layer=2, num_heads=[3, 3], hidden_dim=[8, 8], output_dim=5)


def test_keyed_gat_has_the_surface_and_initial_weights_of_gat():
  for over in ({}, SMALL):
    cfg = configs.qm8_gat(**over)
    torch.manual_seed(1234)
    a = GAT(cfg)
    after_a = torch.randn(3)
    torch.manual_seed(1234)
    b = KeyedGAT(cfg)
    after_b = torch.randn(3)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(torch.equal(sa[k], sb[k]) for k in sa)
    assert torch.equal(after_a, after_b)                  # the same CPU random numbers were consumed
    b.load_state_dict(deterministic_state_dict(a, 7))     # strict: the key is not in the state_dict
    a.load_state_dict(b.state_dict())
    assert all(torch.equal(x, y) for x, y in zip(a.state_dict().values(), b.state_dict().values()))
  assert isinstance(b, TrainableGAT) and 'dropout_key' not in b.state_dict()
  assert b.dropout_key.dtype == torch.int64 and b.dropout_key.tolist() == [1234, 0]
  assert [n for n, _ in b.named_buffers()] == ['dropout_key']


def test_key_defaults_to_zero_seed_without_config_seed():
  cfg = configs.qm8_gat(**SMALL)
  cfg.seed = None
  assert KeyedGAT(cfg).dropout_key.tolist() == [0, 0]


@pytest.mark.parametrize('bad', [torch.zeros(2, dtype=torch.int32), torch.zeros(3, dtype=torch.int64), (1, 2),
                                 torch.zeros(1, 2, dtype=torch.int64)])
def test_dropout_key_checks_fire_before_device_work(bad):
  """The module sits on the CPU: any device work would raise RuntimeError instead of ValueError."""
  m = KeyedGAT(configs.qm8_gat(dropout=0.1, **SMALL)).train()
  nf, L = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 4, 7)
  with pytest.raises(ValueError, match='dropout_key'):
    m(nf, L, dropout_key=bad)
  for fn, args in ((ops.gat_dropout_project, (torch.zeros(4, 8), torch.zeros(6, 8), 3)),
                   (ops.gat_attention_dropout, (None,) * 7)):
    with pytest.raises(ValueError, match='dropout_key'):
      fn(*args, bad, 0.1, 0)


def test_keyed_gat_without_dropout_is_trainable_gat_and_has_no_cpu_path():
  m = KeyedGAT(configs.qm8_gat(dropout=0.1, **SMALL))
  nf, L = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 4, 7)
  for mode in (m.train(), m.eval()):
    with pytest.raises(RuntimeError, match='no CPU'):
      mode(nf, L)
  assert m.dropout_key.tolist() == [1234, 0]              # nothing ran, nothing advanced
  assert 'dropout_key' in train.GraphedStep._RECORD_KEYS


def test_dropin_binds_keyed_gat_only_with_the_gat_opt_in():
  for training in (False, True):
    ns = types.ModuleType('fake_runner')
    ns.GAT, ns.MPNN = 'ref', 'ref'
    dropin.patch_namespace(ns, training=training, opt_in=('GAT',), keyed_dropout=True)
    assert ns.GAT is KeyedGAT and ns.MPNN == 'ref'
    dropin.patch_namespace(ns, training=training, opt_in=('GAT',))
    assert ns.GAT is TrainableGAT
    with pytest.raises(ValueError, match='--opt-in GAT'):
      dropin.patch_namespace(ns, training=training, keyed_dropout=True)
    with pytest.raises(ValueError, match='--opt-in GAT'):
      dropin.patch_namespace(ns, training=training, opt_in=('MPNN',), keyed_dropout=True)
  with pytest.raises(ValueError, match='--opt-in GAT'):
    dropin.install(None, runner_modules=(), keyed_dropout=True)
  assert dropin.TRAINING_OPT_IN_CLASSES == ('GAT',) and dropin.OPT_IN_CLASSES == ('MPNN',)


def test_dropin_main_passes_the_keyed_dropout_flag(monkeypatch):
  seen = {}
  monkeypatch.setattr(dropin, 'install', lambda root, **kw: seen.update(kw, root=root) or [])
  monkeypatch.setattr(dropin.os, 'chdir', lambda path: None)
  fake = types.ModuleType('run_exp')
  fake.main = lambda: seen.update(argv=list(dropin.sys.argv))
  monkeypatch.setitem(dropin.sys.modules, 'run_exp', fake)
  monkeypatch.setattr(dropin.sys, 'argv', ['x'])
  dropin.main(['/ref', '-c', 'config/qm8_gat.yaml', '--opt-in', 'GAT', '--keyed-dropout'])
  assert seen['opt_in'] == ['GAT'] and seen['keyed_dropout'] is True and seen['training'] is True
  assert seen['argv'] == ['run_exp.py', '-c', 'config/qm8_gat.yaml']
  dropin.main(['/ref', '-c', 'config/qm8_gat.yaml', '--opt-in', 'GAT'])
  assert seen['keyed_dropout'] is False


@pytest.mark.parametrize('key', [(0, 0), (1234, 7), (2 ** 40 + 5, 2 ** 33 + 1), (-3, -1)])
def test_mask_words_match_the_numpy_philox(key):
  """words() over torch int64 against sage_sample_oracle.philox4x32_10 at counter (i >> 2, site, ctr lo,
  ctr hi), word i & 3, for indices across several counters and the three site kinds."""
  idx = torch.cat([torch.arange(0, 37), torch.tensor([2 ** 31 - 1, 2 ** 32 + 3, 2 ** 34 - 1])])
  seed, ctr = (int(v) & (2 ** 64 - 1) for v in key)
  for t, c, sigma in ((0, 0, 0), (3, 55, 1), (65535, 2 ** 14 - 1, 2)):
    st = oracle.site(t, c, sigma)
    got = oracle.words(torch.tensor(key, dtype=torch.int64), st, idx).numpy()
    i = idx.numpy().astype(np.uint64)
    ctrs = np.stack([i >> np.uint64(2), np.full_like(i, st), np.full_like(i, ctr & 0xffffffff),
                     np.full_like(i, ctr >> 32)], axis=-1)
    x = sage_sample_oracle.philox4x32_10(ctrs, np.array([seed & 0xffffffff, seed >> 32], np.uint64))
    want = x[np.arange(len(i)), (i & np.uint64(3)).astype(np.int64)]
    np.testing.assert_array_equal(got, want.astype(np.int64))


def test_mask_keeps_the_rule_fraction_and_scale():
  for p in (0.0, 0.1, 0.5, 0.9, 1.0):
    m = oracle.mask(torch.tensor([5, 9]), p, 1, 2, oracle.INPUT, (64, 128))
    kept = m != 0
    assert m.shape == (64, 128)
    if p == 1.0:
      assert not kept.any()
      continue
    assert torch.all(m[kept] == float(np.float32(1.0 / (1.0 - p))))
    assert abs(kept.double().mean().item() - (1.0 - p)) < 0.02
  assert oracle.threshold(0.5) == 2 ** 31 and oracle.threshold(1.0) == 2 ** 32


def test_masks_differ_across_sites_channels_layers_and_counters():
  key = torch.tensor([11, 3])
  base = oracle.mask(key, 0.5, 1, 2, oracle.ATT, (4, 9, 9))
  for other in (oracle.mask(key, 0.5, 1, 2, oracle.WH, (4, 9, 9)), oracle.mask(key, 0.5, 1, 3, oracle.ATT, (4, 9, 9)),
                oracle.mask(key, 0.5, 2, 2, oracle.ATT, (4, 9, 9)),
                oracle.mask(torch.tensor([11, 4]), 0.5, 1, 2, oracle.ATT, (4, 9, 9))):
    assert not torch.equal(base, other)
  assert torch.equal(base, oracle.mask(key.clone(), 0.5, 1, 2, oracle.ATT, (4, 9, 9)))
