"""Per-phase clock64 timers of the whole-stack kernel on the bench workload, then the kernel alone
(CUDA events, 20 eager launches, median) with each LNB_DBG experiment bit (profiling aid)."""
import ctypes
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import bench  # noqa: E402
from lanczosnetwork_b200 import _lib, ops  # noqa: E402

dev = torch.device('cuda:0')
mod, params = bench.build_model()
mod = mod.to(dev).eval()
mod.use_cuda_graph = False
B = int(sys.argv[1]) if len(sys.argv) > 1 else bench.BATCH
b = bench.make_batches(1, B, 1000)[0]
t = {k: torch.from_numpy(b[k]).to(dev) for k in ('node_feat', 'L', 'D', 'V', 'node_mask')}
prof = torch.zeros(132 * 32, dtype=torch.int64, device=dev)
lib = _lib.load()
orig = ops.spectral_stack_forward
times = []


def probed(*a, **kw):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  _lib.check(lib.lnb_debug_set_prof(ctypes.c_void_p(prof.data_ptr())), 'set_prof')
  e0.record()
  r = orig(*a, **kw)
  e1.record()
  torch.cuda.synchronize()
  lib.lnb_debug_set_prof(None)
  times.append(e0.elapsed_time(e1) * 1e3)
  return r


with torch.no_grad():
  for _ in range(3):
    mod(t['node_feat'], t['L'], t['D'], t['V'], mask=t['node_mask'])
  torch.cuda.synchronize()
  ops.spectral_stack_forward = probed
  prof.zero_()
  mod(t['node_feat'], t['L'], t['D'], t['V'], mask=t['node_mask'])
  ops.spectral_stack_forward = orig
p = prof.cpu().reshape(132, 32).double()
# slot 3 (k-loop s0) includes computing U; slot 8 (k-loop s1) includes waiting for the consumers'
# V Z, which reads step 0's Z from the A ring; step 0 has no epilogue (slots 5 and 7 are edge steps)
names = ['stage issue', 'stage wait', '-', 'k-loop s0', 'pre_epi', 'acc wait s0', 'acc drain', 'store',
         'k-loop s1', 'acc wait s1', 'post_epi']
print('stack kernel %.1f us (with timers); clock64 totals per CTA (cycles)' % times[-1])
for i in (0, 1, 3, 4, 7, 8, 9, 10):
  print('  %-12s cta0 %8d cta1 %8d cta100 %8d  mean %8d  max %8d' % (names[i], p[0, i], p[1, i], p[100, i], p[:, i].mean(), p[:, i].max()))
for i, nm in [(22, 'pre_epi: wait for producers'), (16, 'stage: tables'), (17, 'stage: X/Q issue'), (18, 'stage: ELL lines'), (19, 'readout: wait'), (20, 'readout: W stage'), (21, 'readout: dots')]:
  print('  %-18s mean %8d  max %8d' % (nm, p[:, i].mean(), p[:, i].max()))
print('  sum cta0 %d, mean %d, max %d' % (p[0, :11].sum(), p[:, :11].sum(1).mean(), p[:, :11].sum(1).max()))
act = p[:, 12] > 0
print('  active CTAs %d; whole-CTA ns: mean %.0f max %.0f; cycles mean %.0f max %.0f; => %.3f GHz; start skew %.0f ns; first start->last end %.0f ns' % (
    act.sum(), p[act, 11].mean(), p[act, 11].max(), p[act, 12].mean(), p[act, 12].max(),
    p[act, 12].mean() / p[act, 11].mean(), p[act, 13].max() - p[act, 13].min(),
    (p[act, 13] + p[act, 11]).max() - p[act, 13].min()))

# the kernel alone on the same inputs: as built, MMAs skipped (2), W loads skipped (4), produce() skipped (8)
captured = []


def capture(*a, **kw):
  captured.append((a, kw))
  return orig(*a, **kw)


with torch.no_grad():
  ops.spectral_stack_forward = capture
  mod(t['node_feat'], t['L'], t['D'], t['V'], mask=t['node_mask'])
  ops.spectral_stack_forward = orig
  a, kw = captured[-1]
  for flag in (0, 2, 4, 8):
    os.environ['LNB_DBG'] = str(flag)
    for _ in range(3):
      orig(*a, **kw)
    ts = []
    for _ in range(20):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      orig(*a, **kw)
      e1.record()
      torch.cuda.synchronize()
      ts.append(e0.elapsed_time(e1))
    ts.sort()
    print('LNB_DBG=%d stack kernel alone: median %.3f ms (min %.3f, max %.3f)' % (flag, ts[10], ts[0], ts[-1]))
  os.environ.pop('LNB_DBG')
