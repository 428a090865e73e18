"""Seeded initial state of every drop-in class: state_dict keys in order, shapes and a SHA-256 digest of
each tensor's bytes, for ``torch.manual_seed(SEED)`` followed by the constructor.

    python tests/golden/make_init_digests.py      # writes tests/golden/init_digests.json

The digests pin the construction and initialisation order (each drop-in mirrors the reference's, so a
seed gives the reference's initial weights); tests/test_host_init_state.py compares against them.  The
whole parameter set is too large for a fixture (LanczosNet alone holds 7 MB), hence digests.
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

import torch  # noqa: E402

from lanczosnetwork_b200 import configs  # noqa: E402
from lanczosnetwork_b200 import model as M  # noqa: E402

SEED = 1234
OUT = os.path.join(HERE, 'init_digests.json')

# name -> (class name, config factory name, model overrides)
CASES = {
    'LanczosNet': ('LanczosNet', 'qm8_lanczos_net', {}),
    'LanczosNetGeneral': ('LanczosNetGeneral', 'graph_lanczos_net', {}),
    'AdaLanczosNet': ('AdaLanczosNet', 'qm8_ada_lanczos_net', {}),
    'GCN': ('GCN', 'qm8_gcn', {}),
    'GCNFP': ('GCNFP', 'qm8_gcn', {}),
    'DCNN': ('DCNN', 'qm8_dcnn', {}),
    'ChebyNet': ('ChebyNet', 'qm8_cheby_net', {}),
    'GraphSAGE_Mean': ('GraphSAGE', 'qm8_graphsage', {'agg_func': 'Mean'}),
    'GraphSAGE_Max': ('GraphSAGE', 'qm8_graphsage', {'agg_func': 'Max'}),
    'GGNN_GRU': ('GGNN', 'qm8_ggnn', {'update_func': 'GRU'}),
    'GGNN_RNN': ('GGNN', 'qm8_ggnn', {'update_func': 'RNN'}),
    'GPNN_GRU': ('GPNN', 'qm8_gpnn', {'update_func': 'GRU'}),
    'GPNN_RNN': ('GPNN', 'qm8_gpnn', {'update_func': 'RNN'}),
    'MPNN_MLP': ('MPNN', 'qm8_mpnn', {'msg_func': 'MLP'}),
    'MPNN_embedding': ('MPNN', 'qm8_mpnn', {'msg_func': 'embedding'}),
    'GAT': ('GAT', 'qm8_gat', {}),
    'TrainableGAT': ('TrainableGAT', 'qm8_gat', {}),
}


def build(case, **extra):
  cls, factory, over = CASES[case]
  return getattr(M, cls)(getattr(configs, factory)(**dict(over, **extra)))


def init_state(case):
  """[[key, shape, sha256 of the contiguous tensor's bytes], ...] in state_dict order."""
  torch.manual_seed(SEED)
  mod = build(case)
  out = []
  for k, v in mod.state_dict().items():
    t = v.detach().contiguous()
    out.append([k, list(t.shape), hashlib.sha256(t.numpy().tobytes()).hexdigest()])
  return out


def main():
  digests = {case: init_state(case) for case in CASES}
  # TrainableGAT is GAT's constructor: one copy of its 2357 entries is stored, under GAT
  assert digests.pop('TrainableGAT') == digests['GAT']
  with open(OUT, 'w') as f:
    f.write('{"seed": %d, "cases": {\n' % SEED)
    f.write(',\n'.join('"%s": [\n%s]' % (case, ',\n'.join(json.dumps(e, separators=(',', ':')) for e in entries))
                       for case, entries in digests.items()))
    f.write('}}\n')
  print('wrote %s (%d cases)' % (OUT, len(digests)))


if __name__ == '__main__':
  main()
