"""The ptxas report of the library build (lanczosnetwork_b200/build.log, written by build.py with
-Xptxas -v): every instantiation of the wgmma skeleton (tc_gemm_kernel) issues its MMAs
asynchronously and stays within its register budget.

ptxas serializes every wgmma of a kernel when it cannot keep the accumulators of the MMAs in flight
apart (C7511: a narrow MMA into part of a wider one's fragment) or has to wait for them in a
divergent path (C7518).  It says so in an info line, not an error, and the kernel still runs,
several times slower; this test turns that line into a failure."""
import os
import re

import pytest

from lanczosnetwork_b200 import build

LOG = os.path.join(build.HERE, 'build.log')
SKELETON = '_ZN3tcg14tc_gemm_kernel'
# one instantiation per policy: dense layer, filter-MLP chain, the three GRU updates, three stack variants
POLICIES = {'linear_tf32x3': 1, 'filter_mlp_chain': 1, 'ggnn_update': 1, 'mpnn_update': 1, 'gpnn_partition': 1,
            'spectral_conv_fused': 3}
MAX_REGISTERS = 168          # 384 threads, one CTA per SM
MAX_SPILL_STORES = 128       # bytes; the stack kernel's producers keep a few values on the stack


@pytest.fixture(scope='module')
def log():
  build.build()              # no-op when the library is current
  if not os.path.exists(LOG):
    pytest.fail('%s is missing: rebuild with python -m lanczosnetwork_b200.build --force' % LOG)
  with open(LOG) as fh:
    return fh.read()


def kernel_reports(text):
  """{mangled name: (registers, spill store bytes)} of every tc_gemm_kernel instantiation."""
  out = {}
  props = re.compile(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores'
                     r'.*\n.*Used (\d+) registers')
  for m in props.finditer(text):
    if m.group(1).startswith(SKELETON):
      out[m.group(1)] = (int(m.group(4)), int(m.group(3)))
  return out


def test_host_build_report_no_serialized_wgmma(log):
  bad = [l for l in log.splitlines() if 'C7511' in l or re.search(r'wgmma\S* instructions are serialized', l)]
  assert not bad, 'ptxas serialized wgmma:\n' + '\n'.join(bad)


def test_host_build_report_skeleton_resources(log):
  reps = kernel_reports(log)
  for src, n in POLICIES.items():
    found = [k for k in reps if src in k]
    assert len(found) == n, 'expected %d tc_gemm_kernel instantiation(s) from %s.cu, found %d' % (n, src, len(found))
  for name, (regs, spill) in reps.items():
    assert regs <= MAX_REGISTERS, '%s: %d registers' % (name, regs)
    assert spill <= MAX_SPILL_STORES, '%s: %d bytes of spill stores' % (name, spill)


def test_host_build_report_parser():
  text = ("ptxas info    : Function properties for _ZN3tcg14tc_gemm_kernelIN2_14linear_tf32x3E\n"
          "    40 bytes stack frame, 36 bytes spill stores, 48 bytes spill loads\n"
          "ptxas info    : Used 168 registers, used 3 barriers, 40 bytes cumulative stack size\n"
          "ptxas info    : Function properties for _Z5otherv\n"
          "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
          "ptxas info    : Used 32 registers\n")
  assert kernel_reports(text) == {'_ZN3tcg14tc_gemm_kernelIN2_14linear_tf32x3E': (168, 36)}
