"""Install the H100 drop-ins into an UNMODIFIED checkout of lrjconan/LanczosNetwork.

    python -m lanczosnetwork_b200.dropin /path/to/LanczosNetwork -c config/qm8_lanczos_net.yaml -t
    python -m lanczosnetwork_b200.dropin /path/to/LanczosNetwork -c config/qm8_gpnn.yaml --device-partition

What it does (see INTEGRATION.md):
  1. registers ``operators._ext`` / ``operators._ext.segment_reduction`` in ``sys.modules`` so
     ``from model import *`` of the reference works without building its THC-era extension
     (model/mpnn.py:6 -> operators/functions/unsorted_segment_sum.py:5);
  2. rebinds the classes of ``DROPIN_CLASSES`` (``LanczosNet``, ``AdaLanczosNet``, ``GCN``, ``GAT``, ``GraphSAGE``, ``GGNN``, ``GPNN``, ...)
     inside the runner modules' globals, because the runners resolve the class with ``eval(name)`` in their own
     namespace (runner/qm8_runner.py:59,288; runner/graph_runner.py:57,285), plus the classes of
     ``OPT_IN_CLASSES`` named with ``--opt-in NAME`` (repeatable; e.g. ``--opt-in MPNN``); ``--opt-in GAT``
     (``TRAINING_OPT_IN_CLASSES``) binds ``TrainableGAT`` under the name ``GAT``, and ``--opt-in GraphSAGE``
     (``LSTM_OPT_IN_CLASSES``) binds ``LSTMGraphSAGE`` (which takes ``agg_func: LSTM``) under the name
     ``GraphSAGE``, for training and test runs; ``--keyed-dropout`` with ``--opt-in GAT`` binds ``KeyedGAT``
     instead of ``TrainableGAT``, which trains with the config's ``dropout > 0`` (masks drawn on the device);
  3. with ``--device-partition`` (``install(..., device_partition=True)``), rebinds ``spectral_clustering``
     and ``get_L_cluster_cut`` in the dataset modules' globals (``DATASET_MODULES``) to stand-ins, so the GPNN
     collate never runs scikit-learn and ships empty [B,0,0] partition operators; the GPNN drop-in then
     partitions every batch on the device (``ops.spectral_partition``);
  4. runs the reference ``run_exp.main()`` unchanged (``--opt-in``, ``--keyed-dropout`` and
     ``--device-partition`` are removed from its argv).
"""
import importlib
import os
import sys

import numpy as np

from . import model as _models
from .operators import _ext as _ext_pkg

DROPIN_CLASSES = ('LanczosNet', 'AdaLanczosNet', 'LanczosNetGeneral', 'GCN', 'GCNFP', 'DCNN', 'ChebyNet',
                  'GAT', 'GraphSAGE', 'GGNN', 'GPNN')
# drop-ins that replace the reference class only when asked for (patch_namespace(opt_in=...), --opt-in)
OPT_IN_CLASSES = ('MPNN',)
# names whose drop-in becomes its trainable subclass ``Trainable<name>`` when asked for (opt_in=..., --opt-in);
# without the opt-in they keep their DROPIN_CLASSES behaviour
TRAINING_OPT_IN_CLASSES = ('GAT',)
# names whose drop-in becomes the subclass that also takes the LSTM aggregator, ``LSTM<name>``, when asked for
# (opt_in=..., --opt-in), for training and test runs; without the opt-in an LSTM config fails in the constructor
LSTM_OPT_IN_CLASSES = ('GraphSAGE',)
# modules whose GPNN collate calls the host partition (dataset/qm8.py:123-136, dataset/graph_data.py)
DATASET_MODULES = ('dataset.qm8', 'dataset.graph_data')


def register_native_op():
  """Make ``operators._ext.segment_reduction`` importable under the reference's module path."""
  sys.modules.setdefault('operators._ext', _ext_pkg)
  sys.modules.setdefault('operators._ext.segment_reduction', _ext_pkg.segment_reduction)
  ops_pkg = sys.modules.get('operators')
  if ops_pkg is not None:
    setattr(ops_pkg, '_ext', _ext_pkg)


def _check_opt_in(opt_in):
  unknown = [n for n in opt_in if n not in OPT_IN_CLASSES + TRAINING_OPT_IN_CLASSES + LSTM_OPT_IN_CLASSES]
  if unknown:
    raise ValueError('dropin: %s not in OPT_IN_CLASSES %s, TRAINING_OPT_IN_CLASSES %s or LSTM_OPT_IN_CLASSES %s'
                     % (', '.join(map(repr, unknown)), OPT_IN_CLASSES, TRAINING_OPT_IN_CLASSES,
                        LSTM_OPT_IN_CLASSES))
  return tuple(opt_in)


def _check_keyed_dropout(opt_in, keyed_dropout):
  if keyed_dropout and 'GAT' not in opt_in:
    raise ValueError("dropin: keyed_dropout (--keyed-dropout) binds KeyedGAT under the name GAT and needs "
                     "opt_in=('GAT',) (--opt-in GAT)")


def patch_namespace(module, training=False, opt_in=(), keyed_dropout=False):
  """Rebind the class names in ``module``'s globals to the H100 drop-ins: those of ``DROPIN_CLASSES``
  and those of ``opt_in`` (names from ``OPT_IN_CLASSES`` or ``TRAINING_OPT_IN_CLASSES``; any other name
  is a ValueError).  ``training=True`` (a run without ``-t``) rebinds only the classes that have a
  differentiable training path (every class but ``GAT``, which is inference only); a class without one
  keeps the reference's trainable class instead of failing on the first ``loss.backward()``.  A name of
  ``TRAINING_OPT_IN_CLASSES`` in ``opt_in`` is bound to ``Trainable<name>``, one of ``LSTM_OPT_IN_CLASSES`` to
  ``LSTM<name>``, in training and test runs.  ``keyed_dropout=True`` (only with ``GAT`` in ``opt_in``, else a
  ValueError) binds ``KeyedGAT`` under the name ``GAT`` instead of ``TrainableGAT``."""
  opt_in = _check_opt_in(opt_in)
  _check_keyed_dropout(opt_in, keyed_dropout)
  for name in DROPIN_CLASSES + tuple(n for n in opt_in if n in OPT_IN_CLASSES):
    if hasattr(module, name):
      cls = getattr(_models, name)
      if training and not hasattr(cls, '_train_impl'):
        continue
      setattr(module, name, cls)
  for name in opt_in:
    if name in TRAINING_OPT_IN_CLASSES and hasattr(module, name):
      keyed = keyed_dropout and name == 'GAT'
      setattr(module, name, getattr(_models, ('Keyed' if keyed else 'Trainable') + name))
    if name in LSTM_OPT_IN_CLASSES and hasattr(module, name):
      setattr(module, name, getattr(_models, 'LSTM' + name))
  return module


def _skip_spectral_clustering(L, K, seed=1234):
  """Stand-in for the collate's spectral_clustering: the partition runs on the device."""
  return np.zeros(L.shape[0], dtype=np.int32)


def _skip_cluster_cut(L, node_label):
  """Stand-in for the collate's get_L_cluster_cut: empty operators, stacked to [B,0,0] by the collate."""
  empty = np.zeros((0, 0), dtype=np.float32)
  return empty, empty.copy()


def patch_partition(module):
  """Rebind ``spectral_clustering`` / ``get_L_cluster_cut`` in ``module``'s globals to the stand-ins."""
  module.spectral_clustering = _skip_spectral_clustering
  module.get_L_cluster_cut = _skip_cluster_cut
  return module


def install(reference_root=None, runner_modules=('runner.qm8_runner', 'runner.graph_runner'),
            compat=False, training=False, opt_in=(), device_partition=False, keyed_dropout=False):
  """Returns the list of patched modules.  ``reference_root`` is put on sys.path if given.
  ``compat=True`` first installs the shims of ``lanczosnetwork_b200.compat`` (missing easydict /
  tensorboardX, PyYAML >= 6, numpy >= 2) so the 2019 checkout imports under a current stack.
  Raises ImportError when NO runner module could be imported and patched: the runners resolve
  the model class by name in their own namespace, so a silent miss would run the reference's
  classes while claiming the drop-in.  ``opt_in``, ``keyed_dropout``: see patch_namespace.  ``device_partition``: see patch_partition (the GPNN collate ships
  [B,0,0] operators and the GPNN drop-in partitions on the device)."""
  opt_in = _check_opt_in(opt_in)
  _check_keyed_dropout(opt_in, keyed_dropout)
  if compat:
    from . import compat as _compat
    _compat.install()
  if reference_root is not None:
    reference_root = os.path.abspath(reference_root)
    if reference_root not in sys.path:
      sys.path.insert(0, reference_root)
  register_native_op()
  patched = []
  ref_model = importlib.import_module('model')
  patched.append(patch_namespace(ref_model, training, opt_in, keyed_dropout))
  errors = []
  for name in runner_modules:
    try:
      mod = importlib.import_module(name)
    except ImportError as exc:      # e.g. tensorboardX absent: that runner cannot be used anyway
      errors.append('%s: %s' % (name, exc))
      continue
    patched.append(patch_namespace(mod, training, opt_in, keyed_dropout))
  if runner_modules and len(patched) == 1:
    raise ImportError('dropin.install: no runner module could be imported, nothing would call the '
                      'H100 classes (%s); pass compat=True for the shims of '
                      'lanczosnetwork_b200.compat' % '; '.join(errors))
  if device_partition:
    for name in DATASET_MODULES:
      patched.append(patch_partition(importlib.import_module(name)))
  return patched


def main(argv=None):
  argv = list(sys.argv[1:] if argv is None else argv)
  if not argv:
    raise SystemExit(__doc__)
  root = argv.pop(0)
  opt_in = []
  while '--opt-in' in argv:
    i = argv.index('--opt-in')
    if i + 1 >= len(argv):
      raise SystemExit('--opt-in needs a class name (one of %s)'
                       % (OPT_IN_CLASSES + TRAINING_OPT_IN_CLASSES + LSTM_OPT_IN_CLASSES,))
    opt_in.append(argv[i + 1])
    del argv[i:i + 2]
  device_partition = '--device-partition' in argv
  keyed_dropout = '--keyed-dropout' in argv
  argv = [a for a in argv if a not in ('--device-partition', '--keyed-dropout')]
  install(root, compat=True, training=('-t' not in argv and '--test' not in argv), opt_in=opt_in,
          device_partition=device_partition, keyed_dropout=keyed_dropout)
  os.chdir(root)
  sys.argv = ['run_exp.py'] + argv
  run_exp = importlib.import_module('run_exp')
  run_exp.main()


if __name__ == '__main__':
  main()
