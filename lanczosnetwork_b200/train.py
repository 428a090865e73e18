"""Training path (SURVEY 8f1): the forward AND backward of the spectral-convolution models as
``torch.autograd.Function``s whose arithmetic runs in this library's CUDA kernels.

The reference trains through autograd over ``torch.bmm`` / ``nn.Linear``
(runner/qm8_runner.py:188-259, ``train_loss.backward()`` at :247).  Here every contraction of the
forward and of its adjoint goes through the C ABI:

  * dense layers ``act(x W^T + b)`` and their two adjoint products (``g W`` and ``g^T x``): the
    wgmma 3xTF32 kernel (lnb_linear_tf32x3) -- the big Linear of the graph-conv layer is 97 % of
    the flops of a training step -- or, for layers too small to amortise that kernel's set-up, the
    strided fp32 GEMM reading W / W^T / g^T in place;
  * operator products ``L_e X``, ``L_e^T G`` (channel-innermost operators read in place through
    their strides), ``V^T X``, ``V diag(f) U`` and their adjoints: the strided batched GEMM
    (lnb_batched_gemm);
  * the embedding gradient, GraphSAGE Max's gradient and the LSTM aggregator's row gather adjoint: the
    scatter-add of the reference's own ``unsorted_segment_sum`` op (ops.segment_sum_forward): fp32 atomics
    (lnb_unsorted_segment_sum_forward), or, under ``torch.use_deterministic_algorithms(True)``, the exact
    order-independent sum (lnb_unsorted_segment_sum_exact), which makes every training step bit-reproducible.

PyTorch supplies what it supplies everywhere in this package -- tensor memory, streams, the autograd
tape -- plus the pointwise glue of the adjoint (ReLU masks, sigmoid gate, masked mean, the loss).
The training forward is the UNFUSED formulation (activations have to exist to be differentiated);
the one-launch fused stack remains the inference path.  Gradients are checked against
``torch.autograd`` over the fp64 CPU oracle in tests/test_gpu_train.py, and function by function
across the shapes they accept in tests/test_gpu_train_envelope.py.
"""
import collections

import torch

from . import ops

__all__ = ['dense', 'EllOperator', 'ell_operator', 'operator_messages', 'spectral_messages', 'embedding', 'ritz_stack_train',
           'dcnn_train', 'cheby_train', 'gated_readout', 'bmm', 'lanczos_tridiag', 'tridiag_powers', 'ada_train', 'neighbour_max', 'sage_train',
           'lstm_messages', 'ggnn_train', 'gpnn_train', 'recurrent_cell', 'edge_aggregate', 'set2vec_train', 'mpnn_train', 'gat_attention',
           'gat_train', 'GraphedStep']

_EPS = 1.1920928955078125e-07       # np.finfo(np.float32).eps (ada_lanczos_net.py:8)


def _pad_cols(x, mult=4):
  k = x.shape[1]
  if k % mult == 0:
    return x.contiguous()
  return torch.nn.functional.pad(x, (0, mult - k % mult)).contiguous()


def _matmul_nt(a, w):
  """a [M,K] @ w[N,K]^T on the wgmma 3xTF32 kernel; K is zero padded to a multiple of 4."""
  a, w = _pad_cols(a.float()), _pad_cols(w.float())
  w_hi, w_lo = ops.split_tf32(w)
  return ops.linear_tf32x3(a, w_hi, w_lo, None, False)


# Below this many flops (2 M N K) a dense layer is launch bound on the persistent wgmma kernel (
# allocation, barrier set-up, operand splits, padded / transposed copies for its two adjoint products):
# the strided fp32 GEMM reads W, W^T, g^T in place and is exact fp32.  At the reference's batch size (64
# molecules) this is every layer but the graph-conv Linear, which keeps 95 % of the flops on the tensor cores.
_SMALL_DENSE_FLOPS = 1.5e8


def _small_gemm(A, a_str, Bm, b_str, M, N, K, bias=None, relu=False):
  C = torch.empty((M, N), device=A.device, dtype=torch.float32)
  ops.bgemm(A, (0, 0) + a_str, Bm, (0, 0) + b_str, C, (0, 0, N, 1), 1, 1, M, N, K, bias=bias, relu=relu)
  return C


class _Dense(torch.autograd.Function):
  """y = act(x W^T + b): nn.Linear (+ ReLU) of model/lanczos_net.py:109-113,180-181,188-189."""

  @staticmethod
  def forward(ctx, x, weight, bias, relu):
    M, K = x.shape
    N = weight.shape[0]
    ctx.small = 2.0 * M * N * K < _SMALL_DENSE_FLOPS
    if ctx.small:
      x, weight = x.float().contiguous(), weight.float().contiguous()
      y = _small_gemm(x, (K, 1), weight, (1, K), M, N, K, bias.float().contiguous() if bias is not None else None, relu)
    else:
      xp, wp = _pad_cols(x.float()), _pad_cols(weight.float())
      w_hi, w_lo = ops.split_tf32(wp)
      y = ops.linear_tf32x3(xp, w_hi, w_lo, bias, relu)
    ctx.relu = bool(relu)
    ctx.save_for_backward(x, weight, y if relu else None)
    ctx.has_bias = bias is not None
    return y

  @staticmethod
  def backward(ctx, gy):
    x, weight, y = ctx.saved_tensors
    gy = gy.contiguous()
    if ctx.relu:
      gy = gy * (y > 0).to(gy.dtype)
    gx = gw = gb = None
    M, K = x.shape
    N = weight.shape[0]
    if ctx.needs_input_grad[0]:                                     # g W
      gx = (_small_gemm(gy, (N, 1), weight, (K, 1), M, K, N) if ctx.small
            else _matmul_nt(gy, weight.t())[:, :K])
    if ctx.needs_input_grad[1]:                                     # g^T x
      # few output tiles, long contraction over the rows: the tensor-core kernel wins at every size
      gw = _matmul_nt(gy.t(), x.t())[:, :K]
    if ctx.has_bias and ctx.needs_input_grad[2]:
      gb = gy.sum(dim=0)
    return gx, gw, gb, None


def dense(x, weight, bias, relu=False):
  return _Dense.apply(x, weight, bias, relu)


class _OperatorMessages(torch.autograd.Function):
  """msg[b, n, e*D:(e+1)*D] = (L[b, :, :, e] X[b])[n]   for the channels e in ``channels``
  (model/lanczos_net.py:177-178); adjoint: gX = sum_e L_e^T g_e."""

  @staticmethod
  def forward(ctx, L, X, c0, nc):
    B, N, D = X.shape
    E1 = L.shape[3]
    X = X.contiguous()
    msg = torch.empty((B, N, nc * D), device=X.device, dtype=torch.float32)
    ops.bgemm(L, (N * N * E1, 1, N * E1, E1), X, (N * D, 0, D, 1), msg, (N * nc * D, D, nc * D, 1),
              B, nc, N, D, N, a_off=c0)
    ctx.save_for_backward(L)
    ctx.c0, ctx.nc = c0, nc
    return msg

  @staticmethod
  def backward(ctx, g):
    (L,) = ctx.saved_tensors
    B, N, E1 = L.shape[0], L.shape[1], L.shape[3]
    nc = ctx.nc
    D = g.shape[2] // nc
    g = g.contiguous()
    tmp = torch.empty((B, nc, N, D), device=g.device, dtype=torch.float32)
    # A[m = column c][k = row r] = L[b, r, c, e]: the transpose through swapped strides
    ops.bgemm(L, (N * N * E1, 1, E1, N * E1), g, (N * nc * D, D, nc * D, 1), tmp,
              (nc * N * D, N * D, D, 1), B, nc, N, D, N, a_off=ctx.c0)
    return None, tmp.sum(dim=1), None, None


class EllOperator(collections.namedtuple('EllOperator', 'prep prep_t weight')):
  """Operators [B,N,N,E1] held as ELL rows instead of a dense tensor: ``prep`` (ops.graph_prepare /
  graph_prepare_sparse / spectral_partition_sparse), ``prep_t`` the ELL rows of the transposed operators
  (the adjoint reads them), ``weight`` optional row weights [B,N,E1] (the ``avg`` aggregations) or None.
  The training functions that take a dense L take this too; their products then run on
  ops.ell_messages / ell_messages_adjoint."""

  @property
  def shape(self):
    B, E1, N = self.prep[0].shape[0], self.prep[0].shape[1], self.prep[0].shape[2]
    return (B, N, N, E1)


def ell_operator(prep, prep_t=None):
  """EllOperator of ``prep``; ``prep_t`` defaults to ``prep`` itself, right for symmetric operators (the
  bond-list records: every bond is listed once and both entries of a pair get the same value)."""
  return EllOperator(prep, prep if prep_t is None else prep_t, None)


def _row_sums(op):
  """sum_j L_e[b, n, j] as [B,N,E1], in ELL slot order: ops.ell_messages of a ones column."""
  B, N, _, E1 = op.shape
  ones = torch.ones((B * N, 1), device=op.prep[0].device, dtype=torch.float32)
  return ops.ell_messages(ones, op.prep).reshape(B, N, E1)


def _rows_view(g, width):
  """g as a view the ELL kernels read in place (unit column stride, row stride >= width), else a copy."""
  if g.dim() == 2 and (g.shape[1] <= 1 or g.stride(1) == 1) and (g.shape[0] <= 1 or g.stride(0) >= width):
    return g
  return g.contiguous()


class _EllMessages(torch.autograd.Function):
  """``_OperatorMessages`` over an EllOperator: X [B*N, D] -> [B*N, nc*D] (lnb_ell_messages); adjoint
  gX = sum_e L_e^T (w_e . g_e) over the transposed rows (lnb_ell_messages_adjoint).  On 0/1 or unweighted
  operators both directions give the dense path's bits."""

  @staticmethod
  def forward(ctx, X, op, c0, nc):
    ctx.op, ctx.c0, ctx.nc, ctx.D = op, c0, nc, X.shape[1]
    return ops.ell_messages(_rows_view(X, X.shape[1]), op.prep, c0, nc, w=op.weight)

  @staticmethod
  def backward(ctx, g):
    g = _rows_view(g, ctx.nc * ctx.D)
    op, D, nc = ctx.op, ctx.D, ctx.nc
    if nc == 1:
      return ops.ell_messages_adjoint(g, op.prep_t, D, ctx.c0, 1, w=op.weight), None, None, None
    # one product per channel, summed by the same torch reduction over the same [B, nc, N, D] layout as
    # _OperatorMessages: the per-channel products are the dense path's bits, so the sum is too
    B, N = op.shape[0], op.shape[1]
    tmp = torch.stack([ops.ell_messages_adjoint(g[:, k * D:(k + 1) * D], op.prep_t, D, ctx.c0 + k, 1,
                                                w=op.weight).view(B, N, D) for k in range(nc)], dim=1)
    return tmp.sum(dim=1).reshape(B * N, D), None, None, None


class _EllChannelMessages(torch.autograd.Function):
  """[A_e m_e]_e as [B*N, E1*D] over an EllOperator, one message per channel: every channel's product is
  written straight into its column block (no concatenation); the adjoint reads g's blocks in place."""

  @staticmethod
  def forward(ctx, op, *msgs):
    D = msgs[0].shape[1]
    out = torch.empty((msgs[0].shape[0], len(msgs) * D), device=msgs[0].device, dtype=torch.float32)
    for e, m in enumerate(msgs):
      ops.ell_messages(_rows_view(m, D), op.prep, e, 1, w=op.weight, out=out, col0=e * D)
    ctx.op, ctx.D, ctx.E1 = op, D, len(msgs)
    return out

  @staticmethod
  def backward(ctx, g):
    D = ctx.D
    g = _rows_view(g, ctx.E1 * D)
    return (None,) + tuple(ops.ell_messages_adjoint(g[:, e * D:(e + 1) * D], ctx.op.prep_t, D, e, 1, w=ctx.op.weight)
                           for e in range(ctx.E1))


def _operator(L):
  """The operators as the training functions read them: an EllOperator as is, a dense L as fp32."""
  return L if isinstance(L, EllOperator) else L.float().contiguous()


def operator_messages(L, X, c0=0, nc=None):
  """[L_e X]_{c0 <= e < c0 + nc} as [B,N,nc*D] for a dense L [B,N,N,E1] or an EllOperator."""
  nc = L.shape[3] - c0 if nc is None else nc
  if isinstance(L, EllOperator):
    B, N, D = X.shape
    return _EllMessages.apply(X.reshape(B * N, D), L, c0, nc).reshape(B, N, nc * D)
  return _OperatorMessages.apply(L, X, c0, nc)


class _SpectralMessages(torch.autograd.Function):
  """msg[b, n, s*D:(s+1)*D] = (V diag(F[:, :, s]) V^T X)[b, n]  in factored form
  (model/lanczos_net.py:114-123,172-175); F = filter coefficients [B,K,S] (differentiable: they are
  the output of the learned spectral filter), V is data."""

  @staticmethod
  def forward(ctx, V, X, F):
    B, N, D = X.shape
    K, S = V.shape[2], F.shape[2]
    X, F = X.contiguous(), F.contiguous()
    U = torch.empty((B, K, D), device=X.device, dtype=torch.float32)
    ops.bgemm(V, (N * K, 0, 1, K), X, (N * D, 0, D, 1), U, (K * D, 0, D, 1), B, 1, K, D, N)
    msg = torch.empty((B, N, S * D), device=X.device, dtype=torch.float32)
    ops.bgemm(V, (N * K, 0, K, 1), U, (K * D, 0, D, 1), msg, (N * S * D, D, S * D, 1), B, S, N, D, K,
              kscale=F, s_str=(K * S, 1, S))
    ctx.save_for_backward(V, U, F)
    return msg

  @staticmethod
  def backward(ctx, g):
    V, U, F = ctx.saved_tensors
    B, N, K = V.shape
    S = F.shape[2]
    D = U.shape[2]
    g = g.contiguous()
    T = torch.empty((B, S, K, D), device=g.device, dtype=torch.float32)        # T_s = V^T g_s
    ops.bgemm(V, (N * K, 0, 1, K), g, (N * S * D, D, S * D, 1), T, (S * K * D, K * D, D, 1),
              B, S, K, D, N)
    gF = (T * U.unsqueeze(1)).sum(dim=3).permute(0, 2, 1).contiguous()         # [B,K,S]
    gU = (T * F.permute(0, 2, 1).unsqueeze(3)).sum(dim=1).contiguous()         # [B,K,D]
    gX = torch.empty((B, N, D), device=g.device, dtype=torch.float32)
    ops.bgemm(V, (N * K, 0, K, 1), gU, (K * D, 0, D, 1), gX, (N * D, 0, D, 1), B, 1, N, D, K)
    return None, gX, gF


def spectral_messages(V, X, F):
  return _SpectralMessages.apply(V, X, F)


class _Embedding(torch.autograd.Function):
  """state = table[ids] (model/lanczos_net.py:154); the gradient of the table is the scatter-add of
  the reference's own unsorted_segment_sum op.  An id outside [0, rows) reads a zero row, so its
  gradient row belongs to no table row: the segment sum skips it."""

  @staticmethod
  def forward(ctx, ids, table):
    ctx.save_for_backward(ids)
    ctx.rows = table.shape[0]
    return ops.embedding_rows(ids, table)

  @staticmethod
  def backward(ctx, g):
    (ids,) = ctx.saved_tensors
    D = g.shape[-1]
    flat = g.reshape(1, -1, D).contiguous()
    return None, ops.segment_sum_forward(flat, ids.reshape(1, -1), ctx.rows)[0]


def embedding(ids, table):
  return _Embedding.apply(ids.long(), table)


def _dropout(model, x):
  """The reference's dropout after every layer / propagation step, on the tape in training mode."""
  if model.training and model.dropout > 0.0:
    x = torch.nn.functional.dropout(x, model.dropout, True)
  return x


def _short_walk(L, state, dist):
  """[L_0^k X for k in dist, ascending k]: the walk over channel 0 (lanczos_net.py:164-169)."""
  msgs, walk = [], state
  for step in range(1, max(dist, default=0) + 1):
    walk = operator_messages(L, walk, 0, 1)
    if step in dist:
      msgs.append(walk)
  return msgs


def _conv_layer(model, t, msgs):
  """Graph-convolution layer t on its messages [B,N,*]: concatenated, Linear ``filter[t]`` + ReLU, dropout."""
  B, N = msgs[0].shape[0], msgs[0].shape[1]
  msg = torch.cat(msgs, dim=2) if len(msgs) > 1 else msgs[0]
  lin = model.filter[t]
  return _dropout(model, dense(msg.reshape(B * N, -1), lin.weight, lin.bias, True).reshape(B, N, -1))


def _filter_mlp(seq, h):
  """The four-layer spectral filter MLP ``seq`` (Linear, ReLU, ..., Linear) in the dense kernel."""
  for i in (0, 2, 4, 6):
    h = dense(h, seq[i].weight, seq[i].bias, i != 6)
  return h


def _input_state(model, node_ids, table):
  """h = input_func(table[node_ids]) [B*N, D] of GGNN / GPNN / MPNN."""
  x = embedding(node_ids, table)
  lin = model.input_func[0]
  return dense(x.reshape(-1, x.shape[-1]), lin.weight, lin.bias, False)


def _row_normalised(A):
  """A / (rowsum + float32 eps): the ``avg`` aggregation of GGNN, GPNN and MPNN.  An EllOperator gets
  the row weights 1 / (rowsum + eps) instead, its row sums in ELL slot order."""
  if isinstance(A, EllOperator):
    return A._replace(weight=1.0 / (_row_sums(A) + _EPS))
  return A / (A.sum(dim=2, keepdim=True) + _EPS)


def _channel_messages(A, msgs):
  """[A_e m_e]_e as [B*N, E1*D] for the per-channel messages m_e [B*N, D] (an iterable, consumed in
  channel order)."""
  if isinstance(A, EllOperator):
    return _EllChannelMessages.apply(A, *list(msgs))
  B, N = A.shape[0], A.shape[1]
  agg = torch.cat([operator_messages(A, m.reshape(B, N, -1), e, 1) for e, m in enumerate(msgs)], dim=2)
  return agg.reshape(B * N, -1)


def ritz_stack_train(model, state, node_ids, L, D, V, mask):
  """Differentiable convolution stack + readout of LanczosNet / LanczosNetGeneral / GCN
  (model/lanczos_net.py:125-199): same math, same parameter tensors as the inference path.  L: dense
  [B,N,N,E1] or an EllOperator."""
  L = _operator(L)
  if node_ids is not None:
    state = embedding(node_ids, model.embedding.weight)
  else:
    state = state.float().contiguous()
  B = state.shape[0]
  S = model.num_scale_long
  table = None
  if S > 0:
    V = V.float().contiguous()
    table = ops.ritz_power_table(D.float().contiguous(), model.long_diffusion_dist)   # [B,K,S], data
    K = table.shape[1]
  for t in range(model.num_layer):
    msgs = _short_walk(L, state, model.short_diffusion_dist)
    if S > 0:
      if model.spectral_filter_kind == 'MLP':
        F = _filter_mlp(model.spectral_filter[t], table.reshape(B * K, S)).reshape(B, K, S)
      else:
        F = table
      msgs.append(spectral_messages(V, state, F))
    msgs.append(operator_messages(L, state))
    state = _conv_layer(model, t, msgs)
  return gated_readout(model, state, mask)


def gated_readout(model, state, mask, head=None):
  """Gated masked-mean readout shared by all models (lanczos_net.py:185-194): the two Linears in the
  library's dense kernel, the pointwise gate / mean on the autograd tape.  ``head`` is the output
  Linear, by default ``model.filter[model.num_layer]`` (GGNN passes its ``output_func[0]``)."""
  B, N = state.shape[0], state.shape[1]
  if head is None:
    head = model.filter[model.num_layer]
  att = model.att_func[0]
  flat = state.reshape(B * N, -1)
  y = dense(flat, head.weight, head.bias, False).reshape(B, N, -1)
  gate = torch.sigmoid(dense(flat, att.weight, att.bias, False)).reshape(B, N, 1)
  y = y * gate
  if mask is None:
    return y.mean(dim=1)
  m = (mask != 0).to(y.dtype).unsqueeze(2)
  return (y * m).sum(dim=1) / m.sum(dim=1)


def dcnn_train(model, node_ids, L, mask):
  """Differentiable DCNN (model/dcnn.py:64-124): per layer the edge-type products, then the walk
  L_0^k X for k in diffusion_dist, concatenated EDGES FIRST (:98), Linear + ReLU.  L: dense or an
  EllOperator."""
  L = _operator(L)
  state = embedding(node_ids, model.embedding.weight)
  dist = set(model.diffusion_dist)
  for t in range(model.num_layer):
    state = _conv_layer(model, t, [operator_messages(L, state)] + _short_walk(L, state, dist))
  return gated_readout(model, state, mask)


def cheby_train(model, node_ids, L, mask):
  """Differentiable ChebyNet (model/cheby_net.py:64-124): s_0 = L_0 X, s_k = 2 L_0 s_{k-1} - s_{k-2}
  with s_{-1} = X (the reference's index -1 is its LAST slot, :88-93), bond-type products for e >= 1,
  cat(edges + [s_0 .. s_{order-1}] + [X]) (:99), Linear + ReLU.  L: dense or an EllOperator."""
  L = _operator(L)
  state = embedding(node_ids, model.embedding.weight)
  E1 = L.shape[3]
  order = model.polynomial_order
  for t in range(model.num_layer):
    scale = [None] * (order + 1)
    scale[-1] = state
    scale[0] = operator_messages(L, state, 0, 1)
    for kk in range(1, order):
      scale[kk] = 2.0 * operator_messages(L, scale[kk - 1], 0, 1) - scale[kk - 2]
    state = _conv_layer(model, t, ([operator_messages(L, state, 1, E1 - 1)] if E1 > 1 else []) + scale)
  return gated_readout(model, state, mask)


class _NeighbourMax(torch.autograd.Function):
  """msg[b, n, e*D + f] = max over the neighbours m drawn for row n of channel e of X[b, m, f]: the Max
  aggregator of model/graph_sage.py:141-146 (a row with nonempty = 0 gives 0).  ``prep`` is
  ops.graph_prepare of the count-weighted operators (ops.sage_operators): their ELL rows list the
  distinct neighbours drawn.  The gradient goes to the argmax node (ties: lowest index), scatter-added
  per feature with the library's segment sum."""

  @staticmethod
  def forward(ctx, X, prep):
    msg, arg = ops.neighbour_max(X, prep)
    ctx.save_for_backward(arg)
    ctx.dims = tuple(X.shape)
    return msg

  @staticmethod
  def backward(ctx, g):
    (arg,) = ctx.saved_tensors
    B, N, D = ctx.dims
    b = torch.arange(B, device=g.device).view(B, 1, 1, 1)
    f = torch.arange(D, device=g.device).view(1, 1, 1, D)
    seg = torch.where(arg >= 0, (b * N + arg.long()) * D + f, -1)       # -1: empty row, skipped
    gx = ops.segment_sum_forward(g.reshape(1, -1, 1), seg.reshape(1, -1), B * N * D)
    return gx.view(B, N, D), None


def neighbour_max(X, prep):
  return _NeighbourMax.apply(X.float(), prep)


def sage_train(model, node_ids, M, mask, prep=None, samples=None):
  """Differentiable GraphSAGE (model/graph_sage.py:98-175): embedding -> num_layer - 1 layers of
  [messages of every channel] -> Linear + ReLU -> row / (||row|| + eps) -> dropout -> gated readout
  with the head filter[num_layer].  Mean messages are M_e X on the count-weighted operators M
  [B,N,N,E1] (ops.sage_operators); Max messages come from ``neighbour_max`` on the ELL lists of M
  (``prep``, built here when not given).  M may be an EllOperator instead (its ``prep_t`` the rows of the
  transposed M, which the Mean adjoint reads; Max takes ``prep`` from it).  LSTM messages (``lstm_messages``
  with the cell agg_func[t]) read ``samples`` = (nn_idx, nonempty_mask) instead; M is then unused."""
  lstm = model.agg_func_name == 'LSTM'
  if isinstance(M, EllOperator):
    prep = M.prep if prep is None else prep
  elif not lstm:
    M = M.float().contiguous()
  state = embedding(node_ids, model.embedding.weight)
  B, N = state.shape[0], state.shape[1]
  if model.agg_func_name == 'Max' and prep is None and model.num_layer > 1:
    prep = ops.graph_prepare(M)
  for t in range(model.num_layer - 1):
    if lstm:
      msg = lstm_messages(model.agg_func[t], state, *samples)
    else:
      msg = neighbour_max(state, prep) if model.agg_func_name == 'Max' else operator_messages(M, state)
    lin = model.filter[t]
    y = dense(msg.reshape(B * N, -1), lin.weight, lin.bias, True)
    y = y / (torch.norm(y, 2, dim=1, keepdim=True) + _EPS)
    state = _dropout(model, y.reshape(B, N, -1))
  return gated_readout(model, state, mask)


class _LstmPointwise(torch.autograd.Function):
  """The pointwise part of torch's LSTMCell: from the pre-activations G = [i f g o] [R, 4D] and c [R, D]
  (None: zero), c' = sigmoid(f) c + sigmoid(i) tanh(g), h' = sigmoid(o) tanh(c').  Saves G, c and c' only
  (the gates are recomputed in the backward), so the tape of K steps holds about 6D floats per row and
  step."""

  @staticmethod
  def forward(ctx, G, c):
    i, f, g, o = G.chunk(4, dim=1)
    si, sf, tg, so = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    c2 = si * tg if c is None else sf * c + si * tg
    h2 = so * torch.tanh(c2)
    ctx.save_for_backward(G, c, c2)
    return h2, c2

  @staticmethod
  def backward(ctx, gh, gc2):
    G, c, c2 = ctx.saved_tensors
    i, f, g, o = G.chunk(4, dim=1)
    si, sf, tg, so = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    tc = torch.tanh(c2)
    gc = gc2 + gh * so * (1 - tc * tc)
    gi = gc * tg * si * (1 - si)
    gf = gc * c * sf * (1 - sf) if c is not None else torch.zeros_like(gi)
    gg = gc * si * (1 - tg * tg)
    go = gh * tc * so * (1 - so)
    return torch.cat([gi, gf, gg, go], dim=1), (gc * sf if c is not None and ctx.needs_input_grad[1] else None)


def lstm_messages(cell, state, nn_idx, nonempty):
  """The LSTM aggregator of one GraphSAGE layer (model/graph_sage.py:131-140) on the tape, for every
  channel at once: the sequences s = (b*N + n)*E1 + e run ``cell`` (an nn.LSTMCell) over
  x_t = state[b, nn_idx[b, n, t, e]] from h = c = 0.  The input product is hoisted out of the gather:
  P = state W_ih^T once per layer, then per step P[ids] (the row gather of ``embedding``, whose adjoint is
  the segment sum; an id outside [0, N) reads a zero row, like x = 0) + b_ih + b_hh + h W_hh^T and the
  pointwise cell.  state [B, N, D], nn_idx [B, N, K, E1], nonempty [B, N, 1].  Returns the messages
  [B*N, E1*D]: the final h of channel e in column block e, times nonempty."""
  B, N, D = state.shape
  K, E1 = nn_idx.shape[2], nn_idx.shape[3]
  P = dense(state.reshape(B * N, D), cell.weight_ih, None, False)                 # [B*N, 4D]
  bias = cell.bias_ih + cell.bias_hh
  idx = nn_idx.long()
  rows = torch.where((idx >= 0) & (idx < N), idx + N * torch.arange(B, device=idx.device).view(B, 1, 1, 1),
                     torch.full_like(idx, -1))                                     # global rows, -1: zero
  h = c = None
  for t in range(K):
    G = embedding(rows[:, :, t, :].reshape(-1), P) + bias
    if h is not None:
      G = G + dense(h, cell.weight_hh, None, False)
    h, c = _LstmPointwise.apply(G, c)
  return (h.reshape(B, N, E1 * D) * nonempty.reshape(B, N, 1).to(h.dtype)).reshape(B * N, E1 * D)


def recurrent_cell(kind, cell, x, h):
  """The update cell of GGNN / GPNN on the tape: torch's GRUCell (``kind == 'GRU'``) or the relu RNNCell,
  with both products in the library's dense kernel."""
  gi = dense(x, cell.weight_ih, cell.bias_ih, False)
  gh = dense(h, cell.weight_hh, cell.bias_hh, False)
  if kind == 'GRU':                                                            # torch's GRUCell
    i_r, i_z, i_n = gi.chunk(3, dim=1)
    h_r, h_z, h_n = gh.chunk(3, dim=1)
    r = torch.sigmoid(i_r + h_r)
    z = torch.sigmoid(i_z + h_z)
    n = torch.tanh(i_n + r * h_n)
    return (h - n) * z + n
  return torch.relu(gi + gh)                                                   # RNNCell, relu


def _ggnn_operators(L, aggregate_type):
  """The 0/1 pattern of L, row-normalised by (nnz + float32 eps) for ``avg``: a new tensor.  An
  EllOperator must already hold the pattern (graph_prepare(..., binarize=True)); ``avg`` gives it row
  weights."""
  if isinstance(L, EllOperator):
    return _row_normalised(L) if aggregate_type == 'avg' else L
  A = (L != 0).float()
  if aggregate_type == 'avg':
    A = _row_normalised(A)
  return A.contiguous()


def _ggnn_prop(model, A, h):
  """One GGNN propagation step (model/ggnn.py:143-171, model/gpnn.py:164-190) of h [B*N, D] over the
  operators A [B,N,N,E1]: the first message layers of all channels as one dense layer against their weights
  concatenated on the tape, the second layers, A_e m_e, then ``model.update_func``."""
  first = [seq[0] for seq in model.msg_func]
  w1 = torch.cat([l.weight for l in first], dim=0)
  b1 = torch.cat([l.bias for l in first], dim=0)
  hw = first[0].weight.shape[0]
  hid = dense(h, w1, b1, True)                                                 # [B*N, E1 * 128]
  second = [seq[2] for seq in model.msg_func]
  agg = _channel_messages(A, (dense(hid[:, e * hw:(e + 1) * hw], second[e].weight, second[e].bias, False)
                              for e in range(A.shape[3])))
  return recurrent_cell(model.update_func_name, model.update_func, agg, h)


def ggnn_train(model, node_ids, L, mask):
  """Differentiable GGNN (model/ggnn.py:122-197): embedding -> input_func -> num_prop steps of
  [per-channel message MLP -> A_e m_e -> GRU / RNN cell -> dropout] -> gated readout with the head
  ``output_func``.  A_e is the 0/1 pattern of L_e, row-normalised by (nnz + float32 eps) for ``avg``;
  both are new tensors (the caller's L is not modified).  The first message layers of all channels run
  as one dense layer against their weights concatenated on the tape."""
  A = _ggnn_operators(L, model.aggregate_type)
  B, N = A.shape[0], A.shape[1]
  h = _input_state(model, node_ids, model.embedding.weight)
  D = h.shape[1]
  for _ in range(model.num_prop):
    h = _dropout(model, _ggnn_prop(model, A, h))
  return gated_readout(model, h.reshape(B, N, D), mask, head=model.output_func[0])


def gpnn_train(model, node_ids, L, L_cluster, L_cut, mask):
  """Differentiable GPNN (model/gpnn.py:141-251): embedding -> input_func -> num_prop steps of
  [num_prop_cluster (num_prop_cut) steps of msg_func[0] -> P m -> partition cell over the cluster (cut)
  operator, both chains from the same state -> state_func on [state | cluster | cut] -> the GGNN step over
  the 0/1 pattern of L -> dropout] -> gated readout with the head ``output_func``.  P is the valued
  partition operator, row-normalised by (rowsum + float32 eps) for ``avg``; all operators are new tensors
  (the caller's L, L_cluster and L_cut are not modified).  With an EllOperator L (the 0/1 pattern),
  ``L_cluster`` is the EllOperator of the two-channel [L_cluster, L_cut] and ``L_cut`` is None."""
  A = _ggnn_operators(L, model.aggregate_type)
  if isinstance(L_cluster, EllOperator):
    P = L_cluster
  else:
    P = torch.stack([L_cluster, L_cut], 3).float()
  if model.aggregate_type == 'avg':
    P = _row_normalised(P)
  if not isinstance(P, EllOperator):
    P = P.contiguous()
  B, N = A.shape[0], A.shape[1]
  h = _input_state(model, node_ids, model.embedding.weight)
  D = h.shape[1]
  m1, m2 = model.msg_func[0][0], model.msg_func[0][2]
  s1, s2 = model.state_func[0], model.state_func[2]
  for _ in range(model.num_prop):
    chains = []
    for e, count in enumerate((model.num_prop_cluster, model.num_prop_cut)):
      s = h
      for _ in range(count):
        m = dense(dense(s, m1.weight, m1.bias, True), m2.weight, m2.bias, False)
        agg = operator_messages(P, m.reshape(B, N, D), e, 1).reshape(B * N, D)
        s = recurrent_cell(model.update_func_name, model.update_func_partition, agg, s)
      chains.append(s)
    s = dense(dense(torch.cat([h] + chains, dim=1), s1.weight, s1.bias, True), s2.weight, s2.bias, False)
    h = _dropout(model, _ggnn_prop(model, A, s))
  return gated_readout(model, h.reshape(B, N, D), mask, head=model.output_func[0])


class _EdgeAggregate(torch.autograd.Function):
  """S_e[i] = w_i sum_j A_e[i,j] relu(P_e[j] + Q_e[i]) from PQ [B*N, E1*128] (lnb_mpnn_edge_aggregate); the
  adjoint gathers over the ELL rows of the operators and of their transposes (``prep_t``), without atomics."""

  @staticmethod
  def forward(ctx, PQ, prep, prep_t, avg):
    PQ = PQ.contiguous()
    ctx.save_for_backward(PQ)
    ctx.prep, ctx.prep_t, ctx.avg = prep, prep_t, avg
    return ops.mpnn_edge_aggregate(PQ, prep, avg)

  @staticmethod
  def backward(ctx, gS):
    (PQ,) = ctx.saved_tensors
    return ops.mpnn_edge_aggregate_backward(PQ, gS.contiguous(), ctx.prep, ctx.prep_t, ctx.avg), None, None, None


def edge_aggregate(PQ, prep, prep_t, avg):
  return _EdgeAggregate.apply(PQ.float(), prep, prep_t, bool(avg))


def set2vec_train(model, X, mask):
  """Set2Vec (model/set2set.py:60-100) of every graph at once, then output_func: the Linears in the
  library's dense kernel, the attention over each graph's set as a softmax with the nodes outside the set
  filled with -inf (an empty set reads 0).  X [B,N,D]."""
  s2v = model.att_func
  B, N, D = X.shape
  lin = [seq[0] for seq in s2v.LSTM.gates()]
  wg = torch.cat([l.weight for l in lin], dim=0)
  bg = torch.cat([l.bias for l in lin], dim=0)
  inset = (torch.ones((B, N), device=X.device, dtype=torch.bool) if mask is None
           else (mask != 0).reshape(B, N))
  hidden = X.new_zeros((B, 2 * D))
  mem = X.new_zeros((B, D))
  for _ in range(s2v.num_step_encoder):
    f, i, o, c = dense(hidden, wg, bg, False).chunk(4, dim=1)
    mem = torch.sigmoid(f) * mem + torch.sigmoid(i) * torch.tanh(c)
    h = torch.sigmoid(o) * torch.tanh(mem)
    u = dense(h, s2v.W_1.t(), None, False)
    energy = dense(torch.tanh(u.unsqueeze(1) + X).reshape(B * N, D), s2v.W_2.t(), None, False).reshape(B, N)
    energy = energy.masked_fill(~inset, float('-inf'))
    top = energy.detach().max(dim=1, keepdim=True)[0]
    top = torch.where(torch.isfinite(top), top, torch.zeros_like(top))
    a = torch.exp(energy - top)
    total = a.sum(dim=1, keepdim=True)
    a = a / torch.where(total > 0, total, torch.ones_like(total))
    read = bmm(a.unsqueeze(1), X).reshape(B, D)
    hidden = torch.cat([h, read], dim=1)
  head = model.output_func[0]
  return dense(hidden, head.weight, head.bias, False)


def mpnn_train(model, node_ids, L, mask):
  """Differentiable MPNN (model/mpnn.py:110-212): embedding -> input_func -> num_prop steps of [messages
  -> GRU cell -> dropout] -> Set2Vec -> output_func.  ``MLP`` messages: PQ = dense(h, [W1a_e ; W1b_e]),
  S = edge_aggregate(PQ), agg_e = S_e W2_e^T + (w nnz_e) b2_e; ``embedding`` messages: A_e (h E_e) as in
  ggnn_train.  A_e is the 0/1 pattern of L_e (row-normalised by nnz + float32 eps for ``avg``); the
  caller's L is not modified.  An EllOperator L must hold the pattern (graph_prepare(..., binarize=True));
  its ``prep`` / ``prep_t`` then feed edge_aggregate directly."""
  ell = isinstance(L, EllOperator)
  A = L if ell else (L != 0).float()
  nnz = _row_sums(A) if ell else A.sum(dim=2)                                  # [B,N,E1]
  avg = model.aggregate_type == 'avg'
  B, N, E1 = A.shape[0], A.shape[1], A.shape[3]
  h = _input_state(model, node_ids, model.node_embedding.weight)
  D = h.shape[1]
  if model.msg_func_name == 'MLP':
    if ell:
      prep, prep_t = L.prep, L.prep_t
    else:
      zeros = torch.zeros((B, N, 4), device=L.device, dtype=torch.float32)
      prep = ops.graph_prepare(L, zeros, binarize=True)
      prep_t = ops.graph_prepare(L.transpose(1, 2), zeros, binarize=True)
    deg = (nnz * (1.0 / (nnz + _EPS)) if avg else nnz).reshape(B * N, E1)     # w_i nnz_e(i)
    first = [seq[0] for seq in model.edge_func]
    second = [seq[2] for seq in model.edge_func]
    w_pq = torch.cat([w for l in first for w in (l.weight[:, :D], l.weight[:, D:])], dim=0)
    b_pq = torch.cat([b for l in first for b in (torch.zeros_like(l.bias), l.bias)], dim=0)
    hw = first[0].weight.shape[0]
  else:
    if avg:
      A = _row_normalised(A)
    if not ell:
      A = A.contiguous()
    w_msg = model.edge_embedding.weight.view(E1, D, D).transpose(1, 2).reshape(E1 * D, D)    # stacked E_e^T
  for _ in range(model.num_prop):
    if model.msg_func_name == 'MLP':
      S = edge_aggregate(dense(h, w_pq, b_pq, False), prep, prep_t, avg)       # [B*N, E1*64]
      agg = torch.cat([dense(S[:, e * hw:(e + 1) * hw], second[e].weight, None, False) +
                       deg[:, e:e + 1] * second[e].bias for e in range(E1)], dim=1)
    else:
      msg = dense(h, w_msg, None, False)
      agg = _channel_messages(A, (msg[:, e * D:(e + 1) * D] for e in range(E1)))
    h = _dropout(model, recurrent_cell('GRU', model.update_func, agg, h))
  return set2vec_train(model, h.reshape(B, N, D), mask)


class _GatAttention(torch.autograd.Function):
  """One GAT layer after the projection (lnb_gat_attention) and its adjoint (lnb_gat_attention_backward).
  Only the inputs are saved: the backward recomputes the attention weights ([B, C, N, N], 10 MB per layer
  at B = 64) and h (ELU'(h) = exp(h) for h <= 0; out + 1 loses it where ELU(h) rounds towards -1)."""

  @staticmethod
  def forward(ctx, Wh, bias, a1, a2, c1, c2, sb, last):
    Wh = Wh.contiguous()
    out = ops.gat_attention(Wh, bias, a1, a2, c1, c2, sb, last=last)
    ctx.save_for_backward(Wh, bias, a1, a2, c1, c2, sb)
    ctx.last = last
    return out

  @staticmethod
  def backward(ctx, gout):
    Wh, bias, a1, a2, c1, c2, sb = ctx.saved_tensors
    gWh, ga1, ga2, gc1, gc2, gsb = ops.gat_attention_backward(gout.contiguous(), Wh, bias, a1, a2, c1, c2, sb,
                                                              last=ctx.last)
    return gWh, None, ga1, ga2, gc1, gc2, gsb, None


def gat_attention(Wh, bias, a1, a2, c1, c2, sb, last=False):
  """Differentiable ``ops.gat_attention`` in Wh, a1, a2, c1, c2 and sb; ``bias`` is data."""
  return _GatAttention.apply(Wh.float(), bias.float().contiguous(), a1.float().contiguous(),
                             a2.float().contiguous(), c1.float().contiguous(), c2.float().contiguous(),
                             sb.float().contiguous(), bool(last))


class _GatAttentionDropout(torch.autograd.Function):
  """``_GatAttention`` with the attention and Wh dropout of layer t (lnb_gat_attention_dropout and its
  adjoint).  The backward draws the masks again from the saved device copy of the key the forward drew with
  (the module advances its own key after the forward)."""

  @staticmethod
  def forward(ctx, Wh, bias, a1, a2, c1, c2, sb, key, p, t, last):
    Wh = Wh.contiguous()
    out = ops.gat_attention_dropout(Wh, bias, a1, a2, c1, c2, sb, key, p, t, last=last)
    ctx.save_for_backward(Wh, bias, a1, a2, c1, c2, sb, key)
    ctx.p, ctx.t, ctx.last = p, t, last
    return out

  @staticmethod
  def backward(ctx, gout):
    Wh, bias, a1, a2, c1, c2, sb, key = ctx.saved_tensors
    gWh, ga1, ga2, gc1, gc2, gsb = ops.gat_attention_dropout_backward(gout.contiguous(), Wh, bias, a1, a2, c1, c2,
                                                                      sb, key, ctx.p, ctx.t, last=ctx.last)
    return gWh, None, ga1, ga2, gc1, gc2, gsb, None, None, None, None


class _GatDropoutProject(torch.autograd.Function):
  """Wh = per-channel (X * M_c s) W_c^T of layer t (lnb_gat_dropout_project) and its adjoint
  (lnb_gat_dropout_project_backward), which draws the input masks again from the saved key copy."""

  @staticmethod
  def forward(ctx, X, W, C, key, p, t):
    X, W = X.contiguous(), W.contiguous()
    ctx.save_for_backward(X, W, key)
    ctx.C, ctx.p, ctx.t = C, p, t
    return ops.gat_dropout_project(X, W, C, key, p, t)

  @staticmethod
  def backward(ctx, gWh):
    X, W, key = ctx.saved_tensors
    gX, gW = ops.gat_dropout_project_backward(X, W, gWh.contiguous(), ctx.C, key, ctx.p, ctx.t)
    return gX, gW, None, None, None, None


def gat_train(model, node_ids, bias, mask, dropout_key=None):
  """Differentiable GAT (model/gat.py:125-201): embedding -> per layer the head weights
  of all (E+1) * heads channels stacked in concat order c = jj * heads + ii on the tape, ONE ``dense``
  projection, a1 / a2 / c1 / c2 stacked likewise, ``gat_attention`` -> gated readout with the head
  ``output_func``.  Every channel reads ``bias_{ii}_{E}_{t}`` (the reference's shared state_bias list),
  so that parameter's gradient sums over all E+1 channels and the other ``bias_{ii}_{jj}_{t}`` get
  none (``grad`` stays None, as in the reference).  ``bias`` is the collate's attention bias
  [B,N,N,E+1] (data.gat_bias).

  ``dropout_key`` (int64 [2] CUDA tensor, (seed, counter)): the reference's three dropout sites with
  p = model.dropout, masks drawn on the device by the rule of the C header -- the projection becomes
  ``_GatDropoutProject`` (each channel's own input mask) and the attention ``_GatAttentionDropout``.  The
  Functions keep a copy of the key, so the caller may advance it once the forward is issued.  Without a key
  there is no dropout."""
  bias = bias.float().contiguous()
  if dropout_key is not None:
    dropout_key = dropout_key.detach().clone()
    p = float(model.dropout)
  state = embedding(node_ids, model.embedding.weight)
  B, N = state.shape[0], state.shape[1]
  E = model.num_edgetype
  for t in range(model.num_layer):
    mods = [(jj, ii) for jj in range(E + 1) for ii in range(model.num_heads[t])]
    w = torch.cat([model.filter[t][jj][ii].weight for jj, ii in mods], dim=0)          # [C*F, Din]
    if dropout_key is not None:
      x = state.reshape(B * N, -1).float()
      Wh = _GatDropoutProject.apply(x, w.float(), len(mods), dropout_key, p, t).reshape(B, N, -1)
    else:
      Wh = dense(state.reshape(B * N, -1), w, None, False).reshape(B, N, -1)
    a1 = torch.cat([model.att_net_1[t][jj][ii].weight for jj, ii in mods], dim=0)       # [C, F]
    a2 = torch.cat([model.att_net_2[t][jj][ii].weight for jj, ii in mods], dim=0)
    c1 = torch.cat([model.att_net_1[t][jj][ii].bias for jj, ii in mods], dim=0)         # [C]
    c2 = torch.cat([model.att_net_2[t][jj][ii].bias for jj, ii in mods], dim=0)
    sb = torch.stack([getattr(model, 'bias_%d_%d_%d' % (ii, E, t)) for _, ii in mods], dim=0)
    last = t == model.num_layer - 1
    if dropout_key is not None:
      state = _GatAttentionDropout.apply(Wh.float(), bias, a1.float().contiguous(), a2.float().contiguous(),
                                         c1.float().contiguous(), c2.float().contiguous(), sb.float().contiguous(),
                                         dropout_key, p, t, last)
    else:
      state = gat_attention(Wh, bias, a1, a2, c1, c2, sb, last=last)
  return gated_readout(model, state, mask, head=model.output_func[0])


class _BMM(torch.autograd.Function):
  """C[b] = A[b] @ Bm[b] on the strided batched GEMM, differentiable in both operands
  (gA = g Bm^T, gB = A^T g through swapped strides -- no transposed copies)."""

  @staticmethod
  def forward(ctx, A, Bm):
    A, Bm = A.contiguous(), Bm.contiguous()
    nb, M, K = A.shape
    N = Bm.shape[2]
    C = torch.empty((nb, M, N), device=A.device, dtype=torch.float32)
    ops.bgemm(A, (M * K, 0, K, 1), Bm, (K * N, 0, N, 1), C, (M * N, 0, N, 1), nb, 1, M, N, K)
    ctx.save_for_backward(A, Bm)
    return C

  @staticmethod
  def backward(ctx, g):
    A, Bm = ctx.saved_tensors
    nb, M, K = A.shape
    N = Bm.shape[2]
    g = g.contiguous()
    gA = gB = None
    if ctx.needs_input_grad[0]:            # [M,N] @ [N,K]: B operand = Bm^T via (k stride 1, n stride N)
      gA = torch.empty_like(A)
      ops.bgemm(g, (M * N, 0, N, 1), Bm, (K * N, 0, 1, N), gA, (M * K, 0, K, 1), nb, 1, M, K, N)
    if ctx.needs_input_grad[1]:            # [K,M] @ [M,N]: A operand = A^T via (m stride 1, k stride K)
      gB = torch.empty_like(Bm)
      ops.bgemm(A, (M * K, 0, 1, K), g, (M * N, 0, N, 1), gB, (K * N, 0, N, 1), nb, 1, K, N, M)
    return gA, gB


def bmm(A, Bm):
  return _BMM.apply(A.float(), Bm.float())


def _gaussian_laplacian_train(x, adj):
  """Learned operator of model/ada_lanczos_net.py:101-137 on the autograd tape: Gaussian kernel of the
  embedding distances (sigma^2 = mean over all N^2 pairs, padded ones included), masked by the
  adjacency, symmetrically normalised."""
  diff = x.unsqueeze(1) - x.unsqueeze(2)
  dist2 = (diff * diff).sum(dim=3)
  sigma2 = dist2.reshape(dist2.shape[0], -1).mean(dim=1).reshape(-1, 1, 1)
  A = torch.exp(-dist2 / sigma2) * adj
  rs = A.sum(dim=2, keepdim=True)
  d = (rs + (rs == 0).to(A.dtype)).pow(-0.5)
  return d * A * d.transpose(1, 2)


def _lanczos_train(A, mask, q1, K):
  """Differentiable K-step Lanczos with the reference's rules (model/ada_lanczos_net.py:139-247);
  operator products through ``bmm``, re-orthogonalisation as two block Gram-Schmidt passes (the
  formulation of the inference kernel), the acceptance / masking logic as data (no gradient)."""
  B, N = A.shape[0], A.shape[1]
  iters = min(N, K)
  q = q1.reshape(B, N, 1).to(A.dtype)
  nreal = torch.full((B,), N, device=A.device, dtype=torch.long)
  if mask is not None:
    fm = (mask != 0).reshape(B, N, 1).to(A.dtype)
    q = q * fm
    nreal = fm.sum(dim=1).reshape(B).long()
  q = q / q.norm(dim=1, keepdim=True)
  basis, alphas, betas, valids = [q], [], [], []
  prev, beta_prev = torch.zeros_like(q), torch.zeros((B, 1, 1), device=A.device, dtype=A.dtype)
  ok = torch.ones((B, 1, 1), device=A.device, dtype=A.dtype)
  for i in range(iters):
    cur = basis[i]
    z = bmm(A, cur)
    a = (cur * z).sum(dim=1, keepdim=True)
    z = z - a * cur - beta_prev * prev
    if i > 0:
      Qb = torch.cat(basis[:i], dim=2)                               # [B,N,i]
      scale = 1.0 / ((Qb * Qb).sum(dim=1, keepdim=True) + _EPS)       # [B,1,i]
      for _ in range(2):
        c = bmm(Qb.transpose(1, 2), z) * scale.transpose(1, 2)       # [B,i,1]
        z = z - bmm(Qb, c)
    b = z.norm(dim=1, keepdim=True)
    ok = ok * (b.detach() >= 1.0e-4).to(A.dtype)
    valids.append(ok)
    alphas.append(a)
    betas.append(b)
    basis.append(z * ok / (b + _EPS))
    prev, beta_prev = cur, b
  alpha = torch.cat(alphas, dim=1).squeeze(2)
  valid = torch.cat(valids, dim=1).squeeze(2)
  idx = torch.minimum(valid.sum(dim=1).long(), nreal)
  col = torch.arange(iters, device=A.device).unsqueeze(0)
  valid = valid * (col < idx.unsqueeze(1)).to(A.dtype)
  alpha = alpha * valid
  T = torch.diag_embed(alpha)
  if iters > 1:
    beta = torch.cat(betas[:-1], dim=1).squeeze(2) * valid[:, :-1]
    T = T + torch.diag_embed(beta, offset=1) + torch.diag_embed(beta, offset=-1)
  Q = torch.cat(basis[:iters], dim=2)
  row = torch.arange(N, device=A.device).reshape(1, N, 1)
  Q = Q * (valid.unsqueeze(1) * (row < idx.reshape(B, 1, 1)).to(A.dtype))
  if iters < K:
    T = torch.nn.functional.pad(T, (0, K - iters, 0, K - iters))
    Q = torch.nn.functional.pad(Q, (0, K - iters))
  return T, Q


class _TridiagPowers(torch.autograd.Function):
  """out[b, r, s, c] = (T_b ** powers[s])[r, c] on lnb_tridiag_powers (one launch), its adjoint on
  lnb_tridiag_powers_backward (one launch)."""

  @staticmethod
  def forward(ctx, T, powers):
    T = T.contiguous()
    ctx.save_for_backward(T)
    ctx.powers = powers
    return ops.tridiag_powers(T, powers)

  @staticmethod
  def backward(ctx, g):
    T, = ctx.saved_tensors
    return ops.tridiag_powers_backward(T, g.contiguous(), ctx.powers), None


def tridiag_powers(T, powers):
  """Differentiable powers of the tridiagonal T [B,K,K] -> [B,K,S,K] (the layout of ops.tridiag_powers).
  The forward reads the three diagonals of T for every product after the first, as the kernel does.
  ValueError outside ops.tridiag_powers_backward_supported."""
  powers = [int(p) for p in powers]
  if not ops.tridiag_powers_backward_supported(T.shape[1], powers):
    raise ValueError('tridiag_powers: K=%d with powers up to %d is outside lnb_tridiag_powers_backward'
                     % (T.shape[1], max(powers)))
  return _TridiagPowers.apply(T.float(), powers)


class _LanczosTridiag(torch.autograd.Function):
  """(T, Q) of the K-step Lanczos recurrence on lnb_lanczos_tridiag_train, its adjoint on
  lnb_lanczos_tridiag_backward (one launch each): the backward recomputes the forward with the same code, so
  it differentiates the tape the forward returned.  Gradients flow to A only."""

  @staticmethod
  def forward(ctx, A, mask, q1, K):
    A = A.contiguous()
    out = ops.lanczos_tridiag_train(A, mask, q1, K)
    ctx.save_for_backward(A, mask, q1)
    ctx.K = K
    return out['T'], out['Q']

  @staticmethod
  def backward(ctx, gT, gQ):
    A, mask, q1 = ctx.saved_tensors
    K = ctx.K
    if gT is None:
      gT = torch.zeros((A.shape[0], K, K), device=A.device, dtype=torch.float32)
    if gQ is None:
      gQ = torch.zeros((A.shape[0], A.shape[1], K), device=A.device, dtype=torch.float32)
    return ops.lanczos_tridiag_backward(A, mask, q1, ctx.K, gT, gQ), None, None, None


def lanczos_tridiag(A, mask, q1, K):
  """Differentiable Lanczos layer of the training path: the formulation of ``_lanczos_train`` (same rules,
  two block Gram-Schmidt passes) in one forward and one backward launch.  A [B,N,N], mask [B,N] or None,
  q1 [B,N] or [B,N,1] -> (T [B,K,K], Q [B,N,K]).  ValueError outside ops.lanczos_tridiag_train_supported."""
  B, N = A.shape[0], A.shape[1]
  if not ops.lanczos_tridiag_train_supported(N, K):
    raise ValueError('lanczos_tridiag: N=%d K=%d outside 1 <= N <= %d, 1 <= K <= %d'
                     % (N, K, ops.LANCZOS_TRAIN_MAX_N, ops.LANCZOS_MAX_K))
  q1 = q1.reshape(B, N).float().contiguous()
  if mask is not None:
    mask = (mask != 0).to(torch.uint8).contiguous()
  return _LanczosTridiag.apply(A.float(), mask, q1, int(K))


def ada_train(model, node_ids, L, mask, q1, powers_fn=None, lanczos_fn=None):
  """Differentiable AdaLanczosNet (model/ada_lanczos_net.py:288-368): embedding -> learned Gaussian
  Laplacian -> Lanczos -> learned filter on the powers of T (the 4096-wide MLP on the wgmma dense
  kernel) -> graph convolutions with [short walk | Q G_s Q^T X | L_e X] messages -> gated readout.
  ``powers_fn(T, dist)`` -> [B,K,S,K] (dist ascending), when given, replaces the chain of ``bmm`` products that forms the
  powers of T, and ``lanczos_fn(A, mask, q1, K)`` -> (T, Q) replaces ``_lanczos_train`` (the defaults are
  AdaLanczosNet's own formulation)."""
  L = L.float().contiguous()
  state = embedding(node_ids, model.embedding.weight)
  B, N = state.shape[0], state.shape[1]
  K, S = model.num_eig_vec, model.num_scale_long
  powers = Q = None
  if S > 0:
    adj = (L[:, :, :, 0] != 0).to(torch.float32)                    # ada_lanczos_net.py:310-311
    Le = _gaussian_laplacian_train(state, adj)
    T, Q = (lanczos_fn or _lanczos_train)(Le, mask, q1.to(L.device), K)
    if powers_fn is not None:
      P4 = powers_fn(T, sorted(model.long_diffusion_dist))          # [B,K,S,K], ascending like the chain below
      powers = P4.reshape(B, K, S * K)
      plist = P4.unbind(dim=2)
    else:
      plist, cur = [], T
      for p in range(1, max(model.long_diffusion_dist) + 1):        # T^p by repeated products (:262-270)
        if p in model.long_diffusion_dist:
          plist.append(cur)
        if p < max(model.long_diffusion_dist):
          cur = bmm(cur, T)
      powers = torch.cat(plist, dim=2)                              # [B,K,S*K]: index r, s*K + c (:274)
  for t in range(model.num_layer):
    msgs = _short_walk(L, state, model.short_diffusion_dist)
    if S > 0:
      if model.spectral_filter_kind == 'MLP':
        G = _filter_mlp(model.spectral_filter[t], powers.reshape(B, K * S * K))
        G = G.reshape(B, K, K, S)                                   # index r, c, s (:275)
        G = ((G + G.transpose(1, 2)) * 0.5).permute(0, 3, 1, 2)     # [B,S,K,K]
      else:
        G = torch.stack(plist, dim=1)
      D = state.shape[2]
      U = bmm(Q.transpose(1, 2), state)                             # [B,K,D]
      W = bmm(G.reshape(B * S, K, K), U.unsqueeze(1).expand(B, S, K, D).reshape(B * S, K, D))
      M = bmm(Q.unsqueeze(1).expand(B, S, N, K).reshape(B * S, N, K), W)      # [B*S,N,D]
      msgs.append(M.reshape(B, S, N, D).permute(0, 2, 1, 3).reshape(B, N, S * D))
    msgs.append(operator_messages(L, state))
    state = _conv_layer(model, t, msgs)
  return gated_readout(model, state, mask)


class GraphedStep:
  """One optimisation step -- forward, loss, backward, optimizer update -- of a drop-in module captured
  in ONE CUDA graph and replayed per batch (the loop body of runner/qm8_runner.py:226-259:
  ``optimizer.zero_grad(); _, loss = model(...); loss.backward(); optimizer.step()``).

  At the reference's batch size (64 molecules, config/qm8_lanczos_net.yaml:33) a training step is a few
  hundred small launches and launch-bound in eager mode; the replayed graph removes the host from the
  loop.  Inputs are copied into static device buffers (shapes are fixed at capture: pad every batch to
  the same node count -- padded nodes are masked and have zero operator rows, so the padding does not
  change a real node's value).  The optimizer must support capture (``torch.optim.Adam`` /
  ``AdamW`` get ``capturable=True`` here; plain SGD needs nothing).  The warm-up iterations torch needs
  before capture are rolled back (parameters and optimizer state restored in place), so constructing
  the object does not advance training.  Not for AdaLanczosNet (its start vector is drawn on the
  host each call); KeyedAdaLanczosNet draws it on the device and is captured like the others.  The
  segment sums of the backward read ``torch.are_deterministic_algorithms_enabled()`` when the step is
  captured: a step captured under ``torch.use_deterministic_algorithms(True)`` replays the exact,
  order-independent sum whatever the flag is at replay, and one captured without it replays the atomic sum."""

  def __init__(self, model, optimizer, args, kwargs=None, warmup=3, sparse=False, edge_capacity=None,
               packed=False):
    """``sparse=True``: ``args`` is ``(batch,)``, the records of data.sparse_collate as torch tensors, and the
    step is ``model.forward_sparse_train(batch, label=label)``.  ``node_feat`` gets a static buffer of B*N
    rows, ``edges`` one of ``edge_capacity`` rows (default: the ``Ragged`` bucket of the first batch), and a
    replay copies only the rows present, so one capture serves every batch with the same B, N and K.

    ``packed=True``: ``args`` is ``(batch,)``, a packed batch WITH its labels (data.pack_sparse(...,
    label=True), data.PackedMolecules(..., labels=True)), and no ``label=`` is passed.  Each call is one copy
    of the blob's own bytes into a static blob of ``packed_capacity`` bytes, then the replay: the blob is
    split on the device (lnb_records_unpack_labels) and the model's training entry from records runs on it,
    with ``model.loss_func`` on the unpacked labels.  One capture serves every batch with the same (B, N, K,
    P, eigs).  Keys (``sample_key``, ``dropout_key``) travel beside the blob, as in ``sparse=True``.  For GCN,
    GCNFP, DCNN, ChebyNet, TrainableGAT, KeyedGAT, GGNN, MPNN, GPNN, SampledGraphSAGE and LanczosNet (blobs of
    atom ids, with or without eigenpairs) and SparseLanczosNetGeneral (blobs of float feature rows,
    data.PackedMolecules of GraphData samples: lnb_records_unpack_features splits them).  Every call checks the
    header on the host before copying (a pinned blob in place, a device blob with a small synchronous copy) and
    raises ValueError, leaving parameters and optimizer
    state untouched, rather than step on a batch the device would refuse.  ``step.status`` is the unpack's
    status (device int32 [1], 0 = copied).  ``step.input_consumed`` is a new CUDA event per call, recorded
    after that call's copy: a loader refills the host buffer it passed only once that event has completed
    (with two pinned buffers, keep each call's event beside its buffer)."""
    kwargs = dict(kwargs or {})
    if packed:
      if sparse:
        raise ValueError('GraphedStep: sparse=True and packed=True exclude each other')
      takes = getattr(model, '_takes_packed_training', None)
      if takes is None or not takes(args[0] if len(args) == 1 and isinstance(args[0], dict) else {}):
        raise TypeError('GraphedStep(packed=True) trains GCN, GCNFP, DCNN, ChebyNet, TrainableGAT, KeyedGAT, GGNN, '
                        'MPNN, GPNN, SampledGraphSAGE and LanczosNet from packed batches of atom ids, and '
                        'SparseLanczosNetGeneral from packed batches of float feature rows; %s is not among them'
                        % type(model).__name__)
      self._check_packed_args(args, kwargs)
      checked = model._check_packed_train(args[0])
      model._sparse_inputs(args[0])                          # the model's own checks (its keys)
    elif sparse:
      if not hasattr(model, '_train_records'):
        raise TypeError('GraphedStep(sparse=True) needs a drop-in module with forward_sparse_train; %s has none'
                        % type(model).__name__)
      if len(args) != 1 or not isinstance(args[0], dict) or 'blob' in args[0]:
        raise ValueError('GraphedStep(sparse=True) takes one argument: the data.sparse_collate records (batch,)')
      model._sparse_inputs(args[0])                          # forward_sparse's batch checks
    elif not hasattr(type(model), '_train_impl') or type(model).__name__ == 'AdaLanczosNet':
      raise TypeError('GraphedStep needs a drop-in module with a host-free training forward')
    if not packed and kwargs.get('label') is None:
      raise ValueError('GraphedStep captures the loss: pass label=')
    if sparse:
      from .model._common import Ragged
      edges = args[0]['edges']
      cap = Ragged(edges, edge_capacity).capacity            # ValueError if the first batch does not fit
    dev = model._device()
    if dev.type != 'cuda':
      raise RuntimeError('GraphedStep needs the module on a CUDA device')
    model.train()
    self.model, self.optimizer, self.sparse, self.packed = model, optimizer, bool(sparse), bool(packed)
    if packed:
      self._args = [self._static_packed(args[0], dev, *checked)]
      self.input_consumed = None
    elif sparse:
      self._args = [self._static_records(args[0], dev, cap)]
    else:
      self._args = [self._static(a, dev) for a in args]
    self._kwargs = {k: self._static(v, dev) for k, v in kwargs.items()}
    for group in optimizer.param_groups:
      if 'capturable' in group:
        group['capturable'] = True
    for st in optimizer.state.values():                      # a resumed Adam keeps ``step`` on the host
      if torch.is_tensor(st.get('step')) and st['step'].device != dev:
        st['step'] = st['step'].to(dev)
    params = [p for g in optimizer.param_groups for p in g['params']]
    saved_p = [p.detach().clone() for p in params]
    saved_s = {id(p): {k: v.detach().clone() for k, v in optimizer.state.get(p, {}).items() if torch.is_tensor(v)}
               for p in params}
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
      for _ in range(max(int(warmup), 1)):
        self._body()
    torch.cuda.current_stream(dev).wait_stream(side)
    self.graph = torch.cuda.CUDAGraph()
    optimizer.zero_grad(set_to_none=True)
    with torch.cuda.graph(self.graph, stream=side):          # same stream as the warm-up: the parameters'
      self.score, self.loss = self._body(zero=False)         # AccumulateGrad nodes were created on it
    with torch.no_grad():                                    # roll the warm-up steps back, in place
      for p, sp in zip(params, saved_p):
        p.copy_(sp)
        for k, v in optimizer.state.get(p, {}).items():
          if torch.is_tensor(v):
            old = saved_s[id(p)].get(k)
            v.copy_(old) if old is not None else v.zero_()
    self.replays = 0

  @staticmethod
  def _static(x, dev):
    return x.detach().to(dev).clone() if torch.is_tensor(x) else x

  # the ragged record arrays: static buffers of more rows than a batch fills, only the rows present copied
  _RAGGED = ('node_feat', 'edges', 'V_rows')
  _RECORD_KEYS = ('sizes', 'node_ptr', 'node_feat', 'edge_ptr', 'edges', 'N', 'K', 'V_rows', 'D', 'sample_key', 'start_key',
                  'dropout_key')

  def _static_records(self, batch, dev, cap):
    B, N = int(batch['sizes'].shape[0]), int(batch['N'])
    rows = {'node_feat': B * N, 'edges': cap, 'V_rows': B * N}
    out = {}
    for k in self._RECORD_KEYS:
      if k not in batch:
        continue
      v = batch[k]
      if k in self._RAGGED:
        out[k] = torch.zeros((rows[k],) + tuple(v.shape[1:]), dtype=v.dtype, device=dev)
        out[k][:v.shape[0]].copy_(v)
      else:
        out[k] = self._static(v, dev)
    return out

  def _copy_records(self, batch, kwargs):
    """Checks ``batch`` and the tensor ``kwargs`` (the label) against the captured buffers, ValueError before
    anything is copied; then copies the rows present and the kwargs."""
    static = self._args[0]
    for k, dst in self._kwargs.items():
      if torch.is_tensor(dst):
        src = kwargs.get(k)
        if not torch.is_tensor(src) or tuple(src.shape) != tuple(dst.shape):
          raise ValueError('GraphedStep was captured for %s %s, got %s'
                           % (k, tuple(dst.shape), tuple(src.shape) if torch.is_tensor(src) else src))
    if set(k for k in self._RECORD_KEYS if k in batch) != set(static):
      raise ValueError('GraphedStep was captured for records with %s, got %s'
                       % (sorted(static), sorted(k for k in self._RECORD_KEYS if k in batch)))
    for k, dst in static.items():
      src = batch[k]
      if not torch.is_tensor(dst):
        if int(src) != dst:
          raise ValueError('GraphedStep was captured for %s=%d, got %d' % (k, dst, int(src)))
      elif k in self._RAGGED:
        if src.shape[0] > dst.shape[0] or tuple(src.shape[1:]) != tuple(dst.shape[1:]) or src.dtype != dst.dtype:
          raise ValueError('GraphedStep: %s %s does not fit the captured buffer %s (%s)'
                           % (k, tuple(src.shape), tuple(dst.shape), dst.dtype))
      elif tuple(src.shape) != tuple(dst.shape) or src.dtype != dst.dtype:
        raise ValueError('GraphedStep was captured for %s %s, got %s' % (k, tuple(dst.shape), tuple(src.shape)))
    for k, dst in static.items():
      if torch.is_tensor(dst):
        (dst[:batch[k].shape[0]] if k in self._RAGGED else dst).copy_(batch[k], non_blocking=True)
    for k, dst in self._kwargs.items():
      if torch.is_tensor(dst):
        dst.copy_(kwargs[k], non_blocking=True)

  _PACKED_KEYS = ('sample_key', 'dropout_key')

  @staticmethod
  def _check_packed_args(args, kwargs):
    if len(args) != 1 or not isinstance(args[0], dict) or 'blob' not in args[0]:
      raise ValueError('GraphedStep(packed=True) takes one argument: the packed batch (batch,) of '
                       'data.pack_sparse(..., label=True) or data.PackedMolecules(..., labels=True)')
    if kwargs:
      raise ValueError('GraphedStep(packed=True): the labels travel in the blob; got %s=' % ', '.join(sorted(kwargs)))

  def _static_packed(self, batch, dev, hdr, N, eigs):
    self._packed_shape = (hdr.B, N, hdr.K, eigs, hdr.P)
    blob = torch.zeros(self.model._packed_capacity(hdr.B, N, hdr.K, eigs, hdr.total, label_dim=hdr.P),
                       dtype=torch.uint8, device=dev)
    blob[:hdr.total].copy_(batch['blob'][:hdr.total])
    out = {'blob': blob, 'B': hdr.B, 'N': N, 'K': hdr.K, 'eigs': eigs, 'F': hdr.F}
    for k in self._PACKED_KEYS:
      if k in batch:
        out[k] = self._static(batch[k], dev)
    return out

  def _copy_packed(self, args, kwargs):
    """Checks a packed batch on the host against the captured one -- ValueError before anything is copied --
    then copies the blob's own bytes and the keys, and records ``input_consumed`` behind the copy."""
    self._check_packed_args(args, kwargs)
    batch, static = args[0], self._args[0]
    hdr, N, eigs = self.model._check_packed_train(batch)
    if (hdr.B, N, hdr.K, eigs, hdr.P) != self._packed_shape:
      raise ValueError('GraphedStep was captured for packed batches of (B, N, K, eigs, P) = %s, got %s'
                       % (self._packed_shape, (hdr.B, N, hdr.K, eigs, hdr.P)))
    if hdr.total > static['blob'].numel():
      raise ValueError('GraphedStep: a blob of %d bytes exceeds the captured capacity of %d bytes'
                       % (hdr.total, static['blob'].numel()))
    keys = [k for k in self._PACKED_KEYS if k in batch]
    if set(keys) != set(k for k in self._PACKED_KEYS if k in static):
      raise ValueError('GraphedStep was captured for a packed batch with keys %s, got %s'
                       % (sorted(k for k in self._PACKED_KEYS if k in static), sorted(keys)))
    for k in keys:
      src = batch[k]
      if not torch.is_tensor(src) or tuple(src.shape) != tuple(static[k].shape) or src.dtype != static[k].dtype:
        raise ValueError('GraphedStep was captured for %s %s %s' % (k, tuple(static[k].shape), static[k].dtype))
    static['blob'][:hdr.total].copy_(batch['blob'][:hdr.total], non_blocking=True)
    for k in keys:
      static[k].copy_(batch[k], non_blocking=True)
    self.input_consumed = torch.cuda.Event()               # this call's own: a loader keeps one per buffer
    self.input_consumed.record()

  def _body(self, zero=True):
    if zero:
      self.optimizer.zero_grad(set_to_none=True)
    if self.packed:
      score, label, self.status = self.model._train_packed(self._args[0], self._packed_shape[4])
      score, loss = self.model._finish(score, label)
    elif self.sparse:
      score, loss = self.model.forward_sparse_train(self._args[0], **self._kwargs)
    else:
      score, loss = self.model(*self._args, **self._kwargs)
    loss.backward()
    self.optimizer.step()
    return score, loss

  def __call__(self, *args, **kwargs):
    """Copy this batch into the captured buffers and replay.  Returns (score, loss): static device
    tensors that the next call overwrites."""
    if self.packed or self.sparse:
      if self.packed:
        self._copy_packed(args, kwargs)
      else:
        self._copy_records(args[0], kwargs)
      self.graph.replay()
      self.replays += 1
      return self.score, self.loss
    for dst, src in zip(self._args, args):
      if torch.is_tensor(dst):
        if dst.shape != src.shape:
          raise ValueError('GraphedStep was captured for %s, got %s' % (tuple(dst.shape), tuple(src.shape)))
        dst.copy_(src, non_blocking=True)
    for k, dst in self._kwargs.items():
      if torch.is_tensor(dst):
        dst.copy_(kwargs[k], non_blocking=True)
    self.graph.replay()
    self.replays += 1
    return self.score, self.loss
