"""Every atomic operation in the CUDA sources is on a short list, each with the reason it cannot change a
result's bits: integer counts, maxima and bit sets (whose value does not depend on the order of the
updates), work-queue cursors, profiler timers, and the fp32-atomic segment sum, whose exact,
order-independent twin runs under torch.use_deterministic_algorithms(True).  A new atomic, such as a
floating-point atomicAdd, fails here until someone decides it is acceptable and lists it."""
import collections
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'lanczosnetwork_b200', 'csrc')

CALL = re.compile(r'\b(atomic(?:Add|Sub|Max|Min|Or|And|Xor|Inc|Dec|CAS|Exch)\w*)\s*\(\s*&?\s*([\w.]+)')
ASM = re.compile(r'"[^"]*?\b((?:red|atom)\.[\w.]+)')

# (file, operation, target) -> (occurrences, why the result's bits cannot depend on the order of updates)
ALLOWED = {
    ('batch_prepare.cu', 'atomicOr', 'rowmask'): (2, 'adjacency bit set'),
    ('batch_prepare.cu', 'atomicMax', 's_max'): (1, 'integer maximum of ELL row lengths'),
    ('batch_prepare.cu', 'atomicMax', 's_ke'): (1, 'integer maximum of Ritz counts'),
    ('graph_eigs.cu', 'atomicOr', 'mk'): (2, 'bond-type bit set'),
    ('graph_sage.cu', 'atomicAdd', 'cnt'): (1, 'integer neighbour counts'),
    ('lanczos_fused.cu', 'atomicAdd', 'P.prof'): (3, 'profiler timers and counters, off unless requested'),
    ('lanczos_fused.cu', 'atomicAdd', 'ctl'): (2, 'work-queue cursor; each item is computed the same way by any CTA'),
    ('linear_tf32x3.cu', 'atomicAdd', 'p.counters'): (1, 'split-K arrival counter; partials are summed in a fixed order'),
    ('sage_sample.cu', 'atomicOr', 'adj'): (2, 'adjacency bit set'),
    ('sage_sample.cu', 'atomicMax', 's_max'): (1, 'integer maximum of ELL row lengths'),
    ('sage_sample.cu', 'atomicMax', 's_ne'): (1, 'integer maximum of node extents'),
    ('sage_sample.cu', 'atomicMax', 's_maxT'): (1, 'integer maximum of transposed row lengths'),
    ('segment_reduction.cu', 'red.global.add.v4.f32', ''):
        (1, 'the fp32-atomic segment sum; its exact twin is lnb_unsorted_segment_sum_exact'),
    ('segment_reduction.cu', 'atomicAdd', 'dst'):
        (1, 'the fp32-atomic segment sum; its exact twin is lnb_unsorted_segment_sum_exact'),
    ('segment_reduction.cu', 'atomicOr', 'fl'): (2, 'exact segment sum: NaN / Inf flag bits'),
    ('segment_reduction.cu', 'atomicMax', 'ex'): (1, 'exact segment sum: integer exponent maximum'),
    ('segment_reduction.cu', 'atomicAdd', 'acc'): (1, 'exact segment sum: int64 fixed-point accumulator'),
    ('spectral_conv_fused.cu', 'atomicMax', 's_max'): (1, 'integer maximum of ELL row lengths'),
    ('spectral_conv_fused.cu', 'atomicMax', 's_ext'): (2, 'integer maxima of node and Ritz extents'),
    ('spectral_conv_fused.cu', 'atomicAdd', 'hist'): (1, 'integer histogram of row lengths'),
    ('spectral_partition.cu', 'atomicOr', 'mk'): (2, 'bond-type bit set'),
    ('spectral_partition.cu', 'atomicOr', 'adj'): (2, 'adjacency bit set'),
    ('tc_gemm.cuh', 'atomicAdd', 'buf'): (1, 'profiler timer, off unless requested'),
    ('tc_gemm.cuh', 'atomicAdd', 'g_prof'): (2, 'profiler timers, off unless requested'),
}


def _code(src):
  """The source without its comments."""
  src = re.sub(r'/\*.*?\*/', lambda m: '\n' * m.group(0).count('\n'), src, flags=re.S)
  return re.sub(r'//[^\n]*', '', src)


def atomics(name, src):
  """Counter of (file, operation, target) over the atomic calls and red. / atom. instructions in src."""
  found = collections.Counter()
  code = _code(src)
  for m in CALL.finditer(code):
    found[(name, m.group(1), m.group(2))] += 1
  for m in ASM.finditer(code):
    found[(name, m.group(1), '')] += 1
  return found


def _all_sources():
  files = sorted(glob.glob(os.path.join(CSRC, '*.cu')) + glob.glob(os.path.join(CSRC, '*.cuh')))
  assert files
  found = collections.Counter()
  for path in files:
    with open(path) as fh:
      found += atomics(os.path.basename(path), fh.read())
  return found


def test_every_atomic_is_allowed():
  found = _all_sources()
  extra = {k: n for k, n in found.items() if n > ALLOWED.get(k, (0, ''))[0]}
  assert not extra, 'atomics not on the list (or more of them than listed): %s' % extra


def test_every_allowed_atomic_still_exists():
  found = _all_sources()
  stale = {k: (v[0], found.get(k, 0)) for k, v in ALLOWED.items() if found.get(k, 0) != v[0]}
  assert not stale, stale


def test_a_new_float_atomic_is_found():
  src = '''
  __global__ void k(float* out, const float* x, float* y) {
    // atomicAdd(out, 1.f) in a comment is not code
    atomicAdd(&out[threadIdx.x], x[0]);
    asm volatile("red.global.add.f32 [%0], %1;" :: "l"(y), "f"(x[1]));
    atomicExch(y, 0.f);
  }'''
  assert atomics('graph_ops.cu', src) == collections.Counter({
      ('graph_ops.cu', 'atomicAdd', 'out'): 1, ('graph_ops.cu', 'red.global.add.f32', ''): 1,
      ('graph_ops.cu', 'atomicExch', 'y'): 1})
  # a second float atomicAdd beside the listed one in segment_reduction.cu is one too many
  with open(os.path.join(CSRC, 'segment_reduction.cu')) as fh:
    src = fh.read()
  more = atomics('segment_reduction.cu', src + '\n__device__ void f(float* dst) { atomicAdd(dst, 1.f); }\n')
  assert more[('segment_reduction.cu', 'atomicAdd', 'dst')] > ALLOWED[('segment_reduction.cu', 'atomicAdd', 'dst')][0]
