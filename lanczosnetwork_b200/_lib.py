"""ctypes binding of liblanczosnet_b200.so (C ABI declared in include/lanczosnet_b200.h).

There is NO CPU fallback: if the shared object is missing this module raises at first use
with the build command; every op raises RuntimeError on a non-zero status.
"""
import ctypes
import os
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'liblanczosnet_b200.so')

c_f32p = ctypes.c_void_p
c_stream = ctypes.c_void_p
c_int = ctypes.c_int
c_i64 = ctypes.c_int64


class GemmDesc(ctypes.Structure):
  """lnb_gemm_desc (include/lanczosnet_b200.h)."""
  _fields_ = [
      ('A', ctypes.c_void_p), ('a_sb', c_i64), ('a_sz', c_i64), ('a_sm', c_i64), ('a_sk', c_i64),
      ('B', ctypes.c_void_p), ('b_sb', c_i64), ('b_sz', c_i64), ('b_sk', c_i64), ('b_sn', c_i64),
      ('C', ctypes.c_void_p), ('c_sb', c_i64), ('c_sz', c_i64), ('c_sm', c_i64), ('c_sn', c_i64),
      ('kscale', ctypes.c_void_p), ('s_sb', c_i64), ('s_sz', c_i64), ('s_sk', c_i64),
      ('bias', ctypes.c_void_p), ('bias_sz', c_i64),
      ('batch', ctypes.c_int32), ('nz', ctypes.c_int32), ('M', ctypes.c_int32),
      ('N', ctypes.c_int32), ('K', ctypes.c_int32), ('relu', ctypes.c_int32),
      ('alpha', ctypes.c_float), ('beta', ctypes.c_float),
      ('addend', ctypes.c_void_p), ('d_sb', c_i64), ('d_sz', c_i64), ('d_sm', c_i64), ('d_sn', c_i64),
  ]


class SpectralStack(ctypes.Structure):
  """lnb_spectral_stack (include/lanczosnet_b200.h)."""
  _fields_ = [
      ('X', ctypes.c_void_p), ('node_ids', ctypes.c_void_p), ('emb_table', ctypes.c_void_p),
      ('Q', ctypes.c_void_p), ('coeff', ctypes.c_void_p), ('coeff_layer_stride', c_i64),
      ('ell_val', ctypes.c_void_p), ('ell_idx', ctypes.c_void_p), ('ell_max', ctypes.c_void_p),
      ('gext', ctypes.c_void_p), ('tiles', ctypes.c_void_p),
      ('W_hi', ctypes.c_void_p), ('W_lo', ctypes.c_void_p), ('bias', ctypes.c_void_p),
      ('out_state', ctypes.c_void_p),
      ('W_out', ctypes.c_void_p), ('b_out', ctypes.c_void_p), ('w_att', ctypes.c_void_p),
      ('b_att', ctypes.c_void_p), ('mask', ctypes.c_void_p), ('score', ctypes.c_void_p),
      ('Din', ctypes.c_int32 * 8),
      ('num_layers', ctypes.c_int32), ('Kw', ctypes.c_int32), ('emb_rows', ctypes.c_int32),
      ('P', ctypes.c_int32), ('write_pad', ctypes.c_int32),
      ('B', ctypes.c_int32), ('N', ctypes.c_int32), ('E1', ctypes.c_int32), ('K', ctypes.c_int32),
      ('S', ctypes.c_int32), ('H', ctypes.c_int32), ('relu', ctypes.c_int32),
  ]


# name -> (restype, argtypes): every symbol include/lanczosnet_b200.h declares
SIGNATURES = {
    'lnb_abi_version': (c_int, []),
    'lnb_last_error': (ctypes.c_char_p, []),
    'lnb_launch_count': (c_i64, []),
    'lnb_unsorted_segment_sum_forward':
        (c_int, [c_stream, c_f32p, ctypes.c_void_p, ctypes.POINTER(c_int), c_int, c_f32p]),
    'lnb_unsorted_segment_sum_backward':
        (c_int, [c_stream, c_f32p, ctypes.c_void_p, ctypes.POINTER(c_int), c_int, c_f32p]),
    'lnb_unsorted_segment_sum_exact':
        (c_int, [c_stream, c_f32p, ctypes.c_void_p, ctypes.POINTER(c_int), c_int, ctypes.c_void_p,
                 ctypes.c_void_p, ctypes.c_void_p, c_f32p]),
    'lnb_batched_gemm': (c_int, [c_stream, ctypes.POINTER(GemmDesc)]),
    'lnb_split_tf32': (c_int, [c_stream, c_f32p, c_i64, c_f32p, c_f32p]),
    'lnb_linear_tf32x3':
        (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_linear_tf32x3_splitk':
        (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_f32p, c_int,
                 c_f32p, ctypes.c_void_p]),
    'lnb_linear_tf32x3_grouped':
        (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_graph_prepare': (c_int, [c_stream, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_f32p,
                                  ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                  ctypes.c_void_p, ctypes.c_void_p, c_int]),
    'lnb_tile_assign': (c_int, [c_stream, ctypes.c_void_p, c_int, c_int, ctypes.c_void_p]),
    'lnb_graph_prepare_sparse': (c_int, [c_stream] + [ctypes.c_void_p] * 7 + [c_int] * 5 +
                                 [ctypes.c_void_p] * 11),
    'lnb_graph_prepare_sparse_packed': (c_int, [c_stream] + [ctypes.c_void_p] * 2 + [c_int] * 5 +
                                        [ctypes.c_void_p] * 11),
    'lnb_records_unpack': (c_int, [c_stream, ctypes.c_void_p, c_i64, c_int, c_int, c_i64, c_i64] +
                           [ctypes.c_void_p] * 8),
    'lnb_records_unpack_labels': (c_int, [c_stream, ctypes.c_void_p, c_i64, c_int, c_int, c_i64, c_i64] +
                                  [ctypes.c_void_p] * 8 + [c_int, ctypes.c_void_p]),
    'lnb_graph_prepare_sparse_features': (c_int, [c_stream] + [ctypes.c_void_p] * 7 + [c_int] * 6 +
                                          [ctypes.c_void_p] * 11),
    'lnb_graph_prepare_sparse_features_packed': (c_int, [c_stream] + [ctypes.c_void_p] * 2 + [c_int] * 6 +
                                                 [ctypes.c_void_p] * 11),
    'lnb_records_unpack_features': (c_int, [c_stream, ctypes.c_void_p, c_i64, c_int, c_int, c_int, c_i64, c_i64] +
                                    [ctypes.c_void_p] * 8 + [c_int, ctypes.c_void_p]),
    'lnb_spectral_conv_fused':
        (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, ctypes.c_void_p, ctypes.c_void_p,
                 ctypes.c_void_p, ctypes.c_void_p, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int,
                 c_int, c_int, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_spectral_stack_forward': (c_int, [c_stream, ctypes.POINTER(SpectralStack)]),
    'lnb_sage_operators': (c_int, [c_stream, ctypes.c_void_p, c_f32p, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_sage_stack_forward': (c_int, [c_stream, ctypes.POINTER(SpectralStack), c_int]),
    'lnb_neighbour_max': (c_int, [c_stream, c_f32p, c_f32p, ctypes.c_void_p, ctypes.c_void_p, c_int, c_int,
                                  c_int, c_int, c_f32p, ctypes.c_void_p]),
    'lnb_sage_sample_sparse': (c_int, [c_stream] + [ctypes.c_void_p] * 6 + [c_int] * 5 + [ctypes.c_void_p] * 12),
    'lnb_ritz_rowmap': (c_int, [c_stream, ctypes.c_void_p, c_int, c_int, ctypes.c_void_p, ctypes.c_void_p]),
    'lnb_ritz_filter_mlp': (c_int, [c_stream, c_f32p, ctypes.c_void_p, ctypes.c_void_p, c_f32p, c_f32p,
                                    c_f32p, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_ritz_filter_mlp_ctas': (c_int, [c_stream, c_f32p, ctypes.c_void_p, ctypes.c_void_p, c_f32p, c_f32p,
                                         c_f32p, c_int, c_int, c_int, c_int, c_f32p, c_int]),
    'lnb_debug_set_prof': (c_int, [ctypes.c_void_p]),
    'lnb_debug_set_max_ctas': (c_int, [c_int]),
    'lnb_embedding_rows': (c_int, [c_stream, ctypes.c_void_p, c_f32p, c_i64, c_int, c_int, c_f32p]),
    'lnb_ritz_power_table': (c_int, [c_stream, c_f32p, c_i64, ctypes.POINTER(c_int), c_int, c_f32p]),
    'lnb_readout': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, ctypes.c_void_p,
                            c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_gat_attention': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p,
                                  c_int, c_int, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_gat_attention_backward': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p,
                                           c_f32p, c_int, c_int, c_int, c_int, c_int, c_int, c_f32p, c_f32p]),
    'lnb_gat_attention_dropout': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p,
                                          c_int, c_int, c_int, c_int, c_int, c_int, ctypes.c_void_p,
                                          ctypes.c_double, c_int, c_f32p]),
    'lnb_gat_attention_dropout_backward':
        (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int,
                 c_int, c_int, c_int, ctypes.c_void_p, ctypes.c_double, c_int, c_f32p, c_f32p]),
    'lnb_gat_dropout_project': (c_int, [c_stream, c_f32p, c_f32p, c_int, c_int, c_int, c_int, ctypes.c_void_p,
                                        ctypes.c_double, c_int, c_f32p]),
    'lnb_gat_dropout_project_slabs': (c_int, [c_int, c_int, c_int, c_int]),
    'lnb_gat_dropout_project_backward': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int,
                                                 ctypes.c_void_p, ctypes.c_double, c_int, c_f32p, c_f32p, c_f32p]),
    'lnb_ggnn_update': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, ctypes.c_void_p, ctypes.c_void_p, c_f32p,
                                c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_sage_lstm_step': (c_int, [c_stream, c_f32p, ctypes.c_void_p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p,
                                   c_f32p, c_int, c_int, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_mpnn_update': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, ctypes.c_void_p, ctypes.c_void_p, c_f32p,
                                c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_gpnn_partition_update': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p,
                                          ctypes.c_void_p, ctypes.c_void_p, c_f32p, c_f32p, c_f32p, c_f32p,
                                          c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    'lnb_mpnn_edge_aggregate': (c_int, [c_stream, c_f32p, c_f32p, ctypes.c_void_p, ctypes.c_void_p, c_int, c_int,
                                        c_int, c_int, c_f32p]),
    'lnb_mpnn_edge_aggregate_backward':
        (c_int, [c_stream, c_f32p, c_f32p, c_f32p, ctypes.c_void_p, ctypes.c_void_p, c_f32p, ctypes.c_void_p,
                 ctypes.c_void_p, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_ell_messages': (c_int, [c_stream, c_f32p, c_i64] + [ctypes.c_void_p] * 5 + [c_int] * 6 +
                         [c_f32p, c_i64, c_int]),
    'lnb_ell_messages_adjoint': (c_int, [c_stream, c_f32p, c_i64] + [ctypes.c_void_p] * 5 + [c_int] * 6 +
                                 [c_f32p, c_i64]),
    'lnb_set2vec': (c_int, [c_stream, c_f32p, ctypes.c_void_p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p,
                            c_int, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_operator_chain': (c_int, [c_stream, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_int, c_int,
                                   ctypes.POINTER(c_int), c_f32p, c_i64, c_i64, c_int]),
    'lnb_graph_messages': (c_int, [c_stream, c_f32p, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_int,
                                   c_int, c_int, c_int, ctypes.POINTER(c_int), c_int, c_f32p, c_i64, c_i64]),
    'lnb_gaussian_laplacian': (c_int, [c_stream, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_f32p]),
    'lnb_lanczos_ritz': (c_int, [c_stream, c_f32p, ctypes.c_void_p, c_f32p, c_int, c_int, c_int, c_int,
                                 c_f32p, c_f32p, c_f32p, c_f32p, ctypes.c_void_p, c_f32p, c_f32p,
                                 ctypes.c_void_p]),
    'lnb_graph_eigs_sparse': (c_int, [c_stream] + [ctypes.c_void_p] * 5 + [c_int] * 4 + [ctypes.c_void_p] * 3),
    'lnb_sym_eigs': (c_int, [c_stream, c_f32p, c_i64, ctypes.c_void_p, c_int, c_int, c_int, c_f32p, c_f32p,
                             ctypes.c_void_p]),
    'lnb_spectral_partition_draws': (c_int, [c_int]),
    'lnb_spectral_partition': (c_int, [c_stream, c_f32p, c_i64, c_int, c_int, c_int] + [ctypes.c_void_p] * 6),
    'lnb_spectral_partition_sparse': (c_int, [c_stream] + [ctypes.c_void_p] * 4 + [c_int] * 4 +
                                      [ctypes.c_void_p] * 9),
    'lnb_gat_bias_sparse': (c_int, [c_stream] + [ctypes.c_void_p] * 3 + [c_int] * 3 + [ctypes.c_void_p]),
    'lnb_tridiag_powers':(c_int, [c_stream, c_f32p, c_int, c_int, ctypes.POINTER(c_int), c_int,
                                   c_f32p]),
    'lnb_lanczos_tridiag_train': (c_int, [c_stream, c_f32p, ctypes.c_void_p, c_f32p, c_int, c_int, c_int,
                                          c_f32p, c_f32p, c_f32p, c_f32p, ctypes.c_void_p]),
    'lnb_lanczos_tridiag_backward': (c_int, [c_stream, c_f32p, ctypes.c_void_p, c_f32p, c_int, c_int, c_int,
                                             c_f32p, c_f32p, c_f32p, c_f32p, c_f32p]),
    'lnb_tridiag_powers_backward': (c_int, [c_stream, c_f32p, c_f32p, c_int, c_int, ctypes.POINTER(c_int), c_int,
                                            c_f32p]),
    'lnb_ada_start_vector': (c_int, [c_stream, ctypes.c_void_p, c_int, c_int, c_f32p]),
    'lnb_symmetrize_filters': (c_int, [c_stream, c_f32p, c_int, c_int, c_int, c_f32p]),
}

_lock = threading.Lock()
_lib = None


def load():
  """Load (once) and return the ctypes handle.  Fails loudly if the library is not built."""
  global _lib
  if _lib is not None:
    return _lib
  with _lock:
    if _lib is None:
      if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'liblanczosnet_b200.so is not built (%s). Build it with '
            '`python -m lanczosnetwork_b200.build` (nvcc, sm_90a). There is no CPU fallback.'
            % LIB_PATH)
      lib = ctypes.CDLL(LIB_PATH)
      for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if a declared symbol is missing
        fn.restype = res
        fn.argtypes = args
      if lib.lnb_abi_version() != 1:
        raise RuntimeError('liblanczosnet_b200.so ABI mismatch; rebuild')
      _lib = lib
  return _lib


def check(status, what):
  if status != 0:
    msg = load().lnb_last_error()
    raise RuntimeError('%s failed (status %d): %s' % (what, status, (msg or b'').decode()))


_replayed = [0]


def note_graph_replay(num_kernels):
  """Kernels launched by a CUDA-graph replay never pass through the library's host-side launch
  counter; the module records how many kernel nodes the captured forward holds."""
  _replayed[0] += int(num_kernels)


def launch_count():
  """Kernels of this library launched from this process: direct launches (counted in C) plus
  kernel nodes of replayed CUDA graphs."""
  return int(load().lnb_launch_count()) + _replayed[0]
