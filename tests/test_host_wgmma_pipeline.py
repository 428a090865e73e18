"""The SASS of the wgmma skeleton (tc_gemm_kernel) as built: every instantiation issues its wgmma
asynchronously, and those without acc_init() keep one MMA group queued across k-blocks.

`wgmma.wait_group 1` is `WARPGROUP.DEPBAR.LE gsb0, 0x1` in SASS.  When ptxas serialises the wgmma
it fences every HGMMA on its own (`WARPGROUP.ARRIVE` before it, `WARPGROUP.DEPBAR.LE gsb0, 0x0`
after it); a kernel that is not serialised has one ARRIVE per group of 12 HGMMA.  The convolution
stack (SpectralPolicyT, the only policy with acc_init) waits for every group."""
import os
import re
import shutil
import subprocess

import pytest

from lanczosnetwork_b200 import build

SKELETON = '_ZN3tcg14tc_gemm_kernel'
WAITS_EVERY_GROUP = ('SpectralPolicyT',)        # acc_init(): see tc_gemm.cuh, kQueue


def cuobjdump():
  cand = os.path.join(os.path.dirname(build.nvcc_path()), 'cuobjdump')
  return cand if os.path.exists(cand) else shutil.which('cuobjdump')


@pytest.fixture(scope='module')
def sass():
  lib = build.build()
  tool = cuobjdump()
  if tool is None:
    pytest.fail('cuobjdump not found next to nvcc or on PATH')
  return subprocess.run([tool, '-sass', lib], check=True, capture_output=True, text=True).stdout


def functions(text):
  """{mangled name: SASS text} of every tc_gemm_kernel instantiation."""
  out = {}
  parts = re.split(r'\n\s*Function : (\S+)\n', text)
  for name, body in zip(parts[1::2], parts[2::2]):
    if name.startswith(SKELETON):
      out[name] = body
  return out


def test_host_wgmma_pipeline_sass(sass):
  funcs = functions(sass)
  assert len(funcs) == 8, 'expected 8 tc_gemm_kernel instantiations, found %d' % len(funcs)
  for name, body in funcs.items():
    n_mma = len(re.findall(r'\bHGMMA\.', body))
    n_arrive = len(re.findall(r'\bWARPGROUP\.ARRIVE\b', body))
    assert n_mma >= 12, '%s: %d HGMMA' % (name, n_mma)
    assert n_arrive * 12 <= n_mma, '%s: %d WARPGROUP.ARRIVE for %d HGMMA (serialised wgmma)' % (name, n_arrive, n_mma)
    queued = 'WARPGROUP.DEPBAR.LE gsb0, 0x1' in body
    if any(k in name for k in WAITS_EVERY_GROUP):
      assert not queued, '%s: unexpected wait_group 1' % name
    else:
      assert queued, '%s: no WARPGROUP.DEPBAR.LE gsb0, 0x1 (one MMA group queued)' % name


def test_host_wgmma_pipeline_parser():
  text = ('\n\tFunction : _ZN3tcg14tc_gemm_kernelIN2_1AEEE\n  HGMMA.64x128x8 ;\n'
          '\n\tFunction : _Z5otherv\n  MOV R1 ;\n')
  assert list(functions(text)) == ['_ZN3tcg14tc_gemm_kernelIN2_1AEEE']
