"""ops.py enters the C library through ops._launch only: every entry it names there is one _lib binds, and no
other line of ops.py calls a library entry, guards a device or checks a status, except the size query
lnb_gat_dropout_project_slabs."""
import os
import re

from lanczosnetwork_b200 import _lib

OPS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'lanczosnetwork_b200', 'ops.py')


def _source():
  with open(OPS) as fh:
    return fh.read()


def test_every_launched_entry_is_bound():
  names = re.findall(r"_launch\('(lnb_\w+)'", _source())
  assert len(names) >= 50, names
  assert not set(names) - set(_lib.SIGNATURES), set(names) - set(_lib.SIGNATURES)


def test_no_entry_is_called_outside_launch():
  src = _source()
  assert re.findall(r'\.(lnb_\w+)\s*\(', src) == ['lnb_gat_dropout_project_slabs']
  assert src.count('_lib.check(') == 1 and src.count('torch.cuda.device(') == 1
