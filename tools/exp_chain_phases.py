"""Filter-MLP chain kernel alone on the bench workload (QM8 LanczosNet, B = 1024), replayed from its own
CUDA graph, as built and with the skeleton's debug switches (LNB_DBG: 2 skips the MMAs, 4 the W loads,
8 produce(), 6 MMAs and W loads): what is left with the tensor side switched off is the CUDA-core and
hand-over work of the items (profiling aid; results are wrong with any switch set).

Then one eager launch with the PhaseTimer buffer registered (lnb_debug_set_prof): the clock64 totals per
CTA of every slot the chain fills.  Producer thread 0 times its own phases; the consumers' operand
hand-over (slot 14) is timed by the first consumer thread."""
import ctypes
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import bench  # noqa: E402
from lanczosnetwork_b200 import _lib, ops  # noqa: E402
from lanczosnetwork_b200.spectral_conv import ritz_filter_coefficients  # noqa: E402

dev = torch.device('cuda:0')
mod, _ = bench.build_model()
mod = mod.to(dev).eval()
bt = bench.make_batches(1, bench.BATCH, 1000)[0]
t = {k: torch.from_numpy(bt[k]).to(dev) for k in ('L', 'D', 'V')}
L, V, D = t['L'].float().contiguous(), t['V'].float().contiguous(), t['D'].float().contiguous()


def graph_time(fn, reps=50):
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(3):
      fn()
  torch.cuda.current_stream().wait_stream(s)
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    fn()
  for _ in range(3):
    g.replay()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(reps):
    g.replay()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / reps * 1e3


# PhaseTimer slots of tc_gemm_kernel as the chain (S <= 8) fills them: stage 1 is an odd sub-step
# (sub = 4 layer + stage), stage 2 an even one
SLOTS = [(1, 'step_begin: W1/W3 staging'), (8, 'k-loop stage 1'), (9, 'acc wait stage 1'),
         (3, 'k-loop stage 2'), (4, 'pre_epilogue'), (5, 'acc wait stage 2'), (7, 'epilogue stores'),
         (10, 'post_epilogue'), (14, 'consumers: operand hand-over')]

with torch.no_grad():
  prep = ops.graph_prepare(L, V)
  table = ops.ritz_power_table(D, mod.long_diffusion_dist)
  mlp = mod._filter_mlp_params()
  run = lambda: ritz_filter_coefficients(D, mod.long_diffusion_dist, mlp, mod._wcache, prep, table=table)
  for flag in (0, 2, 4, 8, 6):
    os.environ['LNB_DBG'] = str(flag)          # read when the kernel is launched (captured)
    us = graph_time(run)
    print('LNB_DBG=%d  filter MLP chain %.1f us' % (flag, us))
  os.environ.pop('LNB_DBG')

  nsm = torch.cuda.get_device_properties(dev).multi_processor_count
  prof = torch.zeros(nsm * 32, dtype=torch.int64, device=dev)
  lib = _lib.load()
  run()
  torch.cuda.synchronize()
  _lib.check(lib.lnb_debug_set_prof(ctypes.c_void_p(prof.data_ptr())), 'lnb_debug_set_prof')
  try:
    run()                                      # the first launch after registering copies the pointer
    torch.cuda.synchronize()
    prof.zero_()
    run()
    torch.cuda.synchronize()
  finally:
    _lib.check(lib.lnb_debug_set_prof(None), 'lnb_debug_set_prof')
  run()                                        # clears the kernel's copy of the pointer
  torch.cuda.synchronize()
  p = prof.cpu().reshape(nsm, 32).double()
  act = p[:, 12] > 0
  print('PhaseTimer, one launch with timers on: %d active CTAs; cycles per CTA (mean / max)' % int(act.sum()))
  for slot, name in SLOTS:
    print('  slot %2d  %-30s %9.0f %9.0f' % (slot, name, p[act, slot].mean(), p[act, slot].max()))
  prod = [s for s, _ in SLOTS if s != 14]
  print('  producer slots summed %9.0f; whole CTA %9.0f cycles, %.1f us (mean); %.3f GHz' % (
      p[act][:, prod].sum(1).mean(), p[act, 12].mean(), p[act, 11].mean() / 1e3,
      p[act, 12].mean() / p[act, 11].mean()))
