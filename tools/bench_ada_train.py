"""AdaLanczosNet training steps: the base class (host start vector, GEMM chains for the Lanczos recurrence and
the powers of T) against KeyedAdaLanczosNet (device start vector, the Lanczos layer on lnb_lanczos_tridiag_train /
_backward, the powers on lnb_tridiag_powers / _backward), eager and captured.

    python tools/bench_ada_train.py [--B 64 1024] [--iters 10] [--repeats 5]

Per batch size (config qm8_ada_lanczos_net: 7 layers, K = 20, powers 5..30; seeded weights,
data.synthetic_qm8_samples, N = 26, Adam), one JSON line.  Every time is measured ``--repeats`` times, the rows
alternating within each repeat, and reported as median, min and max:
  * eager_base_ms / eager_keyed_ms: one eager step (forward, loss, backward, Adam) from device inputs;
  * graphed_padded_ms / graphed_sparse_ms: one train.GraphedStep replay of the keyed class from pinned
    host memory (padded batch with a start_key, or the records of data.sparse_collate), copies included;
  * lanczos_base_ms / lanczos_keyed_ms: the Lanczos layer alone, forward and backward on the step's operator
    (train._lanczos_train against train.lanczos_tridiag), and lanczos_share_base of the base step (medians);
  * forward_ms / forward_sparse_ms: keyed inference from pinned host memory, padded batch against records;
  * start_vector_us, powers_us, powers_backward_us, lanczos_train_us, lanczos_backward_us: the new kernels
    alone (CUDA events over windows of 1000-2000 launches);
Once per batch size: CUDA kernels per eager step and per Lanczos layer (torch.profiler), bytes host to device
per inference call, and the registers and spills of the new kernels from the build log.
The GPU's name and power limit go into every line.
"""
import argparse
import json
import os
import re
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lanczosnetwork_b200 import configs, data, ops, train  # noqa: E402
from lanczosnetwork_b200.model import AdaLanczosNet, KeyedAdaLanczosNet  # noqa: E402
from bench_sparse_dropins import event_ms, gpu_info  # noqa: E402

K = 20
N = 26
NEW_KERNELS = ('ada_start_vector_kernel', 'tridiag_powers_backward_kernel', 'lanczos_train_kernel')


def ptxas_report():
  log = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'lanczosnetwork_b200',
                     'build.log')
  out = {}
  if not os.path.exists(log):
    return out
  lines = open(log).read().splitlines()
  for i, line in enumerate(lines):
    for name in NEW_KERNELS:
      if 'Function properties for' in line and name in line:
        spill = re.search(r'(\d+) bytes spill stores', lines[i + 1])
        regs = re.search(r'Used (\d+) registers', lines[i + 2])
        out[name] = {'registers': int(regs.group(1)) if regs else None,
                     'spill_store_bytes': int(spill.group(1)) if spill else None}
  return out


def kernel_launches(fn):
  from torch.profiler import ProfilerActivity, profile
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and
             not e.name.startswith('Memcpy') and not e.name.startswith('Memset'))


def nbytes(*ts):
  return int(sum(t.numel() * t.element_size() for t in ts if torch.is_tensor(t)))


def pinned(x):
  return torch.from_numpy(np.ascontiguousarray(x)).pin_memory()


def row(B, iters, repeats, dev):
  samples = data.synthetic_qm8_samples(B, seed=B + 7)
  c = data.collate(samples, K, num_nodes=N)
  nf, L, mask = (pinned(c[k]) for k in ('node_feat', 'L', 'node_mask'))
  label = pinned(c['label'])
  dnf, dL, dmask, dlabel = (t.to(dev) for t in (nf, L, mask, label))
  sp = data.sparse_collate(samples, K, eigs=False)
  sp['N'] = N
  rec = {k: (pinned(v) if isinstance(v, np.ndarray) else v) for k, v in sp.items() if k != 'label'}
  rec['start_key'] = torch.tensor([1, 0], dtype=torch.int64).pin_memory()
  cfg = configs.qm8_ada_lanczos_net()
  torch.manual_seed(0)
  weights = AdaLanczosNet(cfg).state_dict()

  def fresh(cls):                     # modules on the device hold locks: build copies, do not deepcopy
    mod = cls(cfg)
    mod.load_state_dict(weights)
    return mod.to(dev).train()
  keyed = fresh(KeyedAdaLanczosNet)
  out = {'gpu': gpu_info(), 'B': B, 'N': N}

  def eager_step(mod):
    opt = torch.optim.Adam(mod.parameters(), lr=1e-4)

    def step():
      opt.zero_grad()
      mod(dnf, dL, label=dlabel, mask=dmask)[1].backward()
      opt.step()
    return step

  base_step, keyed_step = eager_step(fresh(AdaLanczosNet)), eager_step(fresh(KeyedAdaLanczosNet))
  out['launches_base'] = kernel_launches(base_step)
  out['launches_keyed'] = kernel_launches(keyed_step)

  # the Lanczos layer alone on the step's operator, forward and backward: AdaLanczosNet's recurrence on
  # train.bmm against the keyed class's two kernels
  with torch.no_grad():
    state = keyed.embedding.weight[dnf]
    adj = (dL[:, :, :, 0] != 0).float()
    Le = train._gaussian_laplacian_train(state, adj).contiguous()
  q1 = torch.randn(B, N, 1, device=dev)
  gT, gQ = torch.randn(B, K, K, device=dev), torch.randn(B, N, K, device=dev)

  def layer(fn):
    def run():
      A = Le.detach().requires_grad_(True)
      T, Q = fn(A, dmask, q1, K)
      ((T * gT).sum() + (Q * gQ).sum()).backward()
    return run
  lanczos_base, lanczos_keyed = layer(train._lanczos_train), layer(train.lanczos_tridiag)
  out['lanczos_launches_base'] = kernel_launches(lanczos_base)
  out['lanczos_launches_keyed'] = kernel_launches(lanczos_keyed)

  steps = {}
  for sparse in (False, True):
    mod = fresh(KeyedAdaLanczosNet)
    opt = torch.optim.Adam(mod.parameters(), lr=1e-4)
    if sparse:
      st = train.GraphedStep(mod, opt, (rec,), {'label': label}, sparse=True)
      steps['graphed_sparse_ms'] = lambda st=st: st(rec, label=label)
    else:
      key = torch.tensor([1, 0], dtype=torch.int64).pin_memory()
      st = train.GraphedStep(mod, opt, (nf, L), {'label': label, 'mask': mask, 'start_key': key})
      steps['graphed_padded_ms'] = lambda st=st, key=key: st(nf, L, label=label, mask=mask, start_key=key)

  inf = fresh(KeyedAdaLanczosNet).eval()
  key = torch.tensor([1, 0], dtype=torch.int64, device=dev)
  off = 0.3 * torch.diag_embed(torch.rand(B, K - 1, device=dev) - 0.5, 1)
  T = torch.diag_embed(torch.rand(B, K, device=dev) - 0.5) + off + off.transpose(1, 2)
  pw = keyed.long_diffusion_dist
  G = torch.randn(B, K, len(pw), K, device=dev)
  gq = torch.randn(B, N, K, device=dev)
  # (name, callable, calls per window, grad enabled); kernels get windows of >= 1000 launches
  timers = [('eager_base_ms', base_step, iters, True), ('eager_keyed_ms', keyed_step, iters, True),
            ('lanczos_base_ms', lanczos_base, iters, True), ('lanczos_keyed_ms', lanczos_keyed, iters * 10, True),
            ('graphed_padded_ms', steps['graphed_padded_ms'], iters, True),
            ('graphed_sparse_ms', steps['graphed_sparse_ms'], iters, True),
            ('forward_ms', lambda: inf(nf, L, mask=mask, start_key=rec['start_key']), iters * 10, False),
            ('forward_sparse_ms', lambda: inf.forward_sparse(rec), iters * 10, False),
            ('start_vector_us', lambda: ops.ada_start_vector(key, B, N), 2000, False),
            ('powers_us', lambda: ops.tridiag_powers(T, pw), 2000, False),
            ('powers_backward_us', lambda: ops.tridiag_powers_backward(T, G, pw), 2000, False),
            ('lanczos_train_us', lambda: ops.lanczos_tridiag_train(Le, dmask, q1, K), 1000, False),
            ('lanczos_backward_us', lambda: ops.lanczos_tridiag_backward(Le, dmask, q1, K, gT, gq), 1000, False)]
  vals = {name: [] for name, _, _, _ in timers}
  for _ in range(repeats):                        # the rows alternate within every repeat
    for name, fn, n, grad in timers:
      with torch.set_grad_enabled(grad):
        t = event_ms(fn, n)
      vals[name].append(t * 1e3 if name.endswith('_us') else t)
  for name, v in vals.items():
    out[name] = {'median': float(np.median(v)), 'min': float(min(v)), 'max': float(max(v))}
  out['repeats'] = repeats
  out['lanczos_share_base'] = out['lanczos_base_ms']['median'] / out['eager_base_ms']['median']
  out['h2d_padded_bytes'] = nbytes(nf, L, mask, rec['start_key'])
  out['h2d_sparse_bytes'] = nbytes(*[v for k, v in rec.items()])
  out['ptxas'] = ptxas_report()
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, nargs='+', default=[64, 1024])
  ap.add_argument('--iters', type=int, default=10)
  ap.add_argument('--repeats', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_ada_train: needs a CUDA device')
  dev = torch.device('cuda:0')
  for B in args.B:
    print(json.dumps(row(B, args.iters, args.repeats, dev)), flush=True)


if __name__ == '__main__':
  main()
