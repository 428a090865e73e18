"""The kernels' shape limits as the C header names them (LNB_MAX_*, LNB_*_MAX_*, LNB_*_MIN_*) and as ops
names them on the host: one Python constant of the same value per header limit and no other, and no CUDA
source keeping a private copy of a limit."""
import glob
import os
import re

from lanczosnetwork_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'lanczosnetwork_b200', 'csrc')
LIMIT = r'(?:\w+_)?(?:MAX|MIN)_\w+'

# constants of the CUDA sources with MAX or MIN in their name that are tile, layout or tuning choices of one
# kernel, not the limits of an entry point
PRIVATE = {
    'GMAX',            # graphs per packed tile of the convolution stack
    'RMAX',            # rows per packed tile (every graph of LNB_MAX_N fits one)
    'S0MAX',           # filter-MLP stage widths run on the CUDA cores instead of the tensor cores
    'S2V_GMAX',        # graphs per Set2Vec CTA
    'S2V_SMEM_MAX',    # Set2Vec's shared-memory budget per CTA
    'STACK_SAGE_MAX',  # a variant id of the stack kernel (GraphSAGE with Max aggregation)
    'PJ_RTMAX',        # row tiles per thread of the dropout projection
    'MAX_B_STAGES', 'MAX_A_STAGES',   # operand ring depths of the wgmma skeleton
    'SMEM_MAX',        # common.cuh: the shared-memory ceiling itself
}


def _header_limits():
  with open(os.path.join(ROOT, 'include', 'lanczosnet_b200.h')) as fh:
    return {m.group(1): int(m.group(2))
            for m in re.finditer(r'^#define LNB_(%s)\s+(\d+)\b' % LIMIT, fh.read(), re.M)}


def _sources():
  files = sorted(glob.glob(os.path.join(CSRC, '*.cu')) + glob.glob(os.path.join(CSRC, '*.cuh')))
  assert files
  for path in files:
    with open(path) as fh:
      yield os.path.basename(path), fh.read()


def test_every_header_limit_has_the_same_python_constant():
  header = _header_limits()
  assert 'MAX_N' in header and 'PARTITION_MIN_P' in header
  python = {name: v for name, v in vars(ops).items() if re.fullmatch(LIMIT, name) and isinstance(v, int)}
  assert set(header) == set(python), set(header) ^ set(python)
  for name, v in header.items():
    assert python[name] == v, (name, python[name], v)


def test_shared_memory_ceiling_matches():
  with open(os.path.join(CSRC, 'common.cuh')) as fh:
    m = re.search(r'constexpr int SMEM_MAX = (\d+) \* 1024;', fh.read())
  assert m and ops.SMEM_MAX == int(m.group(1)) * 1024


def test_no_source_keeps_a_private_limit():
  found = []
  for name, src in _sources():
    for decl in re.finditer(r'constexpr\s+(?:static\s+)?[\w:]+\s+([^;()]+);', src):
      for const in re.findall(r'(\w+)\s*=', decl.group(1)):
        if re.search(r'MAX|MIN', const) and const not in PRIVATE:
          found.append('%s: %s' % (name, const))
    if name != 'common.cuh' and re.search(r'\b227\s*\*\s*1024\b', src):
      found.append('%s: 227 * 1024 (use lnb::SMEM_MAX)' % name)
  assert not found, found
