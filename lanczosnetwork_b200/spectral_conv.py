"""Spectral graph-convolution forward built from the CUDA ops (shared by the three models).

One layer (reference: model/lanczos_net.py:157-182, model/ada_lanczos_net.py:321-347):

    msg = [ L0^k X  (k in short) ] ++ [ Q G_s Q^T X  (s in long) ] ++ [ L_e X  (e = 0..E) ]
    X'  = ReLU( cat(msg) W^T + b )

GPU mapping: the long-scale filters are applied in factored form Q (G_s (Q^T X)) -- the
N x N filter matrices V diag(f) V^T of lanczos_net.py:114-123 are never materialised -- and the
channel-innermost operator tensor L[B,N,N,E+1] is consumed in place through its element
stride (no strided-slice copies).  Messages are written straight into their column block of
the concatenated [B*N, C*D] buffer, which the wgmma 3xTF32 dense kernel then multiplies by W.
"""
import torch

from . import ops

__all__ = ['WeightCache', 'GraphContext', 'dense', 'graph_conv_layer', 'graph_conv_layer_unfused',
           'ritz_filter_coefficients']


class WeightCache(object):
  """tf32 hi/lo splits of nn.Linear weights, refreshed when the parameter changes.

  An entry is keyed on (name, device) and tagged with (storage pointer, in-place version) of its
  source tensors; it also HOLDS those tensors, so an address cannot be recycled for a different weight
  while its split is cached.  ``nn.DataParallel`` replicas share this object with the master and get
  freshly broadcast parameter tensors (version 0, recycled addresses) on every forward: for them the
  cache is bypassed (``bypass=True``) -- a stale hit would silently use old weights.  In-place edits
  through ``p.data`` do not bump ``_version``; call ``invalidate()`` (``model.invalidate_caches()``)
  after such an edit.  Mutations are serialised by a lock (one Python thread per device under
  DataParallel)."""

  def __init__(self):
    import threading
    self._store = {}
    self._lock = threading.Lock()
    self.bypass = False

  def _get(self, key, tag, build, sources):
    if self.bypass:
      return build()
    with self._lock:
      hit = self._store.get(key)
    if hit is None or hit[0] != tag:
      hit = (tag,) + tuple(build()) + (tuple(sources),)
      with self._lock:
        self._store[key] = hit
    return hit[1:-1]

  def invalidate(self):
    with self._lock:
      self._store.clear()

  def split(self, name, weight, pad_to=None):
    def build():
      w = weight.detach()
      if pad_to is not None and pad_to != w.shape[1]:
        w = torch.nn.functional.pad(w, (0, pad_to - w.shape[1]))   # zero input columns
      return ops.split_tf32(w)
    return self._get((name, weight.device.index), (weight.data_ptr(), weight._version, pad_to), build,
                     [weight])

  def split_stacked(self, name, weights, biases):
    """(hi, lo, bias) of torch.cat(weights, 0) / torch.cat(biases) -- the stacked form the
    grouped dense kernel consumes (one launch for the same MLP stage of every layer)."""
    dev = weights[0].device
    tag = tuple((w.data_ptr(), w._version) for w in list(weights) + list(biases))

    def build():
      hi, lo = ops.split_tf32(torch.cat([w.detach() for w in weights], dim=0))
      return hi, lo, torch.cat([b.detach() for b in biases], dim=0).contiguous()
    return self._get((name, dev.index), tag, build, list(weights) + list(biases))

  def split_mlp_chain(self, name, mlp_layers):
    """Stacked weights of the chain-fused filter MLP kernel: per layer the rows of stage 0
    (input columns zero-padded to the hidden width), stage 1, stage 2 and stage 3; returns
    (w_hi, w_lo, bias_all)."""
    ws = [w for layer in mlp_layers for (_, w, _) in layer]
    bs = [b for layer in mlp_layers for (_, _, b) in layer]
    tag = tuple((t.data_ptr(), t._version) for t in ws + bs)

    def build():
      hd = ws[1].shape[0]
      rows = []
      for layer in mlp_layers:
        w0 = layer[0][1].detach()
        rows.append(torch.nn.functional.pad(w0, (0, hd - w0.shape[1])))
        rows += [layer[1][1].detach(), layer[2][1].detach(), layer[3][1].detach()]
      hi, lo = ops.split_tf32(torch.cat(rows, dim=0).contiguous())
      return hi, lo, torch.cat([b.detach() for b in bs], dim=0).contiguous()
    return self._get((name, ws[0].device.index), tag, build, ws + bs)

  def split_conv_stack(self, name, weights, biases, kw):
    """Stacked convolution weights of consecutive layers for the one-kernel stack: rows
    [l*H, (l+1)*H) = layer l's filter weight, columns zero-padded to kw; returns
    (w_hi, w_lo, bias [L*H])."""
    tag = tuple((t.data_ptr(), t._version) for t in list(weights) + list(biases)) + (kw,)

    def build():
      rows = [torch.nn.functional.pad(w.detach(), (0, kw - w.shape[1])) for w in weights]
      hi, lo = ops.split_tf32(torch.cat(rows, dim=0).contiguous())
      return hi, lo, torch.cat([b.detach() for b in biases], dim=0).contiguous()
    return self._get((name, weights[0].device.index), tag, build, list(weights) + list(biases))

  def stacked(self, name, parts, split=False):
    """torch.cat(parts, 0) of per-module tensors (e.g. the per-head weights of GAT), rebuilt when any
    part changes; returns (hi, lo) of its tf32 split when ``split``, else a 1-tuple."""
    tag = tuple((t.data_ptr(), t._version) for t in parts) + (split,)

    def build():
      cat = torch.cat([t.detach() for t in parts], dim=0).contiguous()
      return ops.split_tf32(cat) if split else (cat,)
    return self._get((name, parts[0].device.index), tag, build, list(parts))

  def derived(self, name, sources, build):
    """Tensors ``build()`` computes from the parameters ``sources`` (e.g. a re-laid-out weight matrix
    and its tf32 split), rebuilt when any source changes; returns build()'s tuple."""
    tag = tuple((t.data_ptr(), t._version) for t in sources)
    return self._get((name, sources[0].device.index), tag, build, list(sources))

  def clear(self):
    self.invalidate()


def dense(x2d, weight, bias, relu, cache, name):
  """act(x2d @ weight^T + bias).  wgmma 3xTF32 kernel when rows are 16-byte multiples
  (x2d may carry zero-padded trailing columns beyond weight.shape[1]), otherwise the generic
  FFMA GEMM."""
  M, K = x2d.shape
  N = weight.shape[0]
  if K % 4 == 0:
    w_hi, w_lo = cache.split(name, weight, K)
    return ops.linear_tf32x3(x2d, w_hi, w_lo, bias, relu)
  assert K == weight.shape[1]
  out = torch.empty((M, N), device=x2d.device, dtype=torch.float32)
  w = weight.detach().contiguous()
  ops.bgemm(x2d, (0, 0, K, 1), w, (0, 0, 1, K), out, (0, 0, N, 1), 1, 1, M, N, K,
            bias=bias, relu=relu)
  return out


def ritz_filter_coefficients(D, powers, mlp_layers, cache, gext=None, table=None, ctas=0):
  """Per-layer multi-scale coefficients of the Ritz values (model/lanczos_net.py:109-113,
  146-149).  The MLP input does not depend on the layer state, so the power table is built once
  and every MLP stage runs for ALL layers in one launch: stage 0 as a dense layer with the
  layers' first weights stacked along the output dimension, stages 1-3 as block-diagonal
  (grouped) dense layers.  mlp_layers: list over layers of [(name, W, b) x 4] or None for the
  plain-power filter.  Returns (coeff [layers,B,K,S] or None, table [B,K,S])."""
  B, K = D.shape
  S = len(powers)
  if table is None:
    table = ops.ritz_power_table(D, powers)          # [B,K,S]
  if mlp_layers is None:
    return None, table
  nl = len(mlp_layers)
  flat = table.reshape(B * K, S)
  hd = mlp_layers[0][0][1].shape[0]
  if ops.ritz_filter_mlp_supported(S, hd):
    # all layers, all four stages in ONE persistent kernel, activations on chip; with the
    # extents of graph_prepare only the rows of non-zero Ritz vectors are evaluated
    w_hi, w_lo, bias_all = cache.split_mlp_chain('spectral_filter.chain', mlp_layers)
    rowmap = nrows = None
    if isinstance(gext, ops.GraphPrep):              # row list came with graph_prepare
      rowmap, nrows = gext.rowmap, gext.nrows
    elif gext is not None:
      rowmap, nrows = ops.ritz_rowmap(gext, K)
    coeff = ops.ritz_filter_mlp(flat, w_hi, w_lo, bias_all, nl, rowmap, nrows, ctas).reshape(nl, B, K, S)
    return coeff, table
  if S % 4 == 0 and hd % 4 == 0:
    h = flat
    for stage in range(4):
      ws = [mlp_layers[l][stage][1] for l in range(nl)]
      bs = [mlp_layers[l][stage][2] for l in range(nl)]
      w_hi, w_lo, bias = cache.split_stacked('spectral_filter.*.%d' % (2 * stage), ws, bs)
      if stage == 0:
        h = ops.linear_tf32x3(h, w_hi, w_lo, bias, True)               # shared input
      else:
        h = ops.linear_tf32x3_grouped(h, w_hi, w_lo, bias, nl, stage < 3)
    coeff = h.reshape(B, K, nl, S).permute(2, 0, 1, 3).contiguous()     # [layers,B,K,S]
    return coeff, table
  out = []
  for params in mlp_layers:
    h = flat
    for i, (name, w, b) in enumerate(params):
      h = dense(h, w, b, i < len(params) - 1, cache, name)
    out.append(h.reshape(B, K, S))
  return torch.stack(out, dim=0), table


class GraphContext(object):
  """Layer-invariant per-forward state: the operators, the Ritz / Lanczos vectors and (lazily)
  their compressed form for the fused kernel."""

  def __init__(self, L, Qv, binarize=False):
    self.L = L
    self.Qv = Qv
    self.binarize = binarize          # operators enter as their non-zero pattern (model/gcnfp.py:83)
    self._prep = None

  def prep(self, defer_tiles=False):
    """defer_tiles: the caller launches ops.tile_assign itself; otherwise tiles pending from a
    deferred prepare are assigned here, on the current stream."""
    if self._prep is None:
      self._prep = ops.graph_prepare(self.L, self.Qv, self.binarize, defer_tiles)
    elif getattr(self._prep, 'tiles_pending', False) and not defer_tiles:
      ops.tile_assign(self._prep, self.Qv.shape[2])
    return self._prep


def graph_conv_layer(state, ctx, coeff, dense_filter, short_dist, num_long, weight, bias, cache,
                     name, last=True, next_fused=False):
  """One spectral convolution layer: the fused wgmma kernel when the shape allows it
  (LanczosNet-style diagonal filters), otherwise the unfused ops below.

  The fused kernel may skip the constant rows of padded nodes only when the consumer of its
  output is another fused layer (which never reads them): an unfused layer multiplies every
  row, so 0 * uninitialised memory (NaN / Inf bit patterns) would leak into real rows."""
  L, Qv = ctx.L, ctx.Qv
  B, N, Din = state.shape
  if (num_long > 0 and Qv is not None and
      ops.fused_conv_supported(N, Din, Qv.shape[2], weight.shape[0], len(short_dist), dense_filter,
                               num_long, L.shape[3])):
    w_hi, w_lo = cache.split(name, weight)
    return ops.spectral_conv_fused(state, Qv, coeff, ctx.prep(), w_hi, w_lo, bias, True,
                                   write_pad=last or not next_fused)
  return graph_conv_layer_unfused(state, L, Qv, coeff, dense_filter, short_dist, num_long, weight,
                                  bias, cache, name)


def graph_conv_layer_unfused(state, L, Qv, coeff, dense_filter, short_dist, num_long, weight, bias,
                             cache, name):
  """One spectral convolution layer from the general-shape ops.

  state [B,N,Din]; L [B,N,N,E1] (channel innermost); Qv [B,N,K] Ritz / Lanczos vectors;
  coeff: [B,K,S] diagonal filter coefficients (LanczosNet) when dense_filter is False,
         [B,S,K,K] symmetric filter blocks (AdaLanczosNet) when True; None if num_long == 0.
  Returns [B,N,H]."""
  B, N, Din = state.shape
  E1 = L.shape[3]
  S = num_long
  n_short = len(short_dist)
  C = n_short + S + E1
  CD = (C * Din + 3) // 4 * 4          # row stride padded to 16 bytes for the tensor-core path
  dev = state.device
  if CD != C * Din:
    msg = torch.zeros((B, N, CD), device=dev, dtype=torch.float32)
  else:
    msg = torch.empty((B, N, CD), device=dev, dtype=torch.float32)
  if ops.graph_messages_supported(N, Qv.shape[2] if (S and Qv is not None) else 0, E1, S,
                                  max(short_dist) if n_short else 0):
    # small graphs: the whole message matrix in ONE launch (operators, filters on chip)
    ops.graph_messages(L, state, Qv if S else None, coeff if S else None, dense_filter, short_dist, msg)
    out = dense(msg.reshape(B * N, CD), weight, bias, True, cache, name)
    return out.reshape(B, N, -1)
  x_str = (N * Din, 0, Din, 1)
  col = 0
  # ---- short diffusion chain: walk <- L0 walk (lanczos_net.py:164-169) --------------------
  if n_short and ops.operator_chain_supported(N, max(short_dist)):
    # the whole walk in one launch (operator and walk on chip), selected steps -> column blocks
    steps = sorted(short_dist)
    sel = [steps.index(s) if s in steps else -1 for s in range(1, max(short_dist) + 1)]
    ops.operator_chain(L, state, max(short_dist), sel, msg, 0)
    col = n_short
  elif n_short:
    l0_str = (N * N * E1, 0, N * E1, E1)
    src, src_str, src_off = state, x_str, 0
    tmp = None
    for step in range(1, max(short_dist) + 1):
      if step in short_dist:
        dst, dst_str, dst_off = msg, (N * CD, 0, CD, 1), col * Din
        col += 1
      else:
        tmp = torch.empty((B, N, Din), device=dev, dtype=torch.float32)
        dst, dst_str, dst_off = tmp, x_str, 0
      ops.bgemm(L, l0_str, src, src_str, dst, dst_str, B, 1, N, Din, N, b_off=src_off,
                c_off=dst_off)
      src, src_off = dst, dst_off
      src_str = (dst_str[0], 0, dst_str[2], 1)
  # ---- long diffusion: Q G_s (Q^T X) ------------------------------------------------------
  if S:
    K = Qv.shape[2]
    U = torch.empty((B, K, Din), device=dev, dtype=torch.float32)
    # U = Q^T X : A[m=k][kk=n] = Q[n*K + k]
    ops.bgemm(Qv, (N * K, 0, 1, K), state, x_str, U, (K * Din, 0, Din, 1), B, 1, K, Din, N)
    if dense_filter:
      W = torch.empty((B, S, K, Din), device=dev, dtype=torch.float32)
      ops.bgemm(coeff, (S * K * K, K * K, K, 1), U, (K * Din, 0, Din, 1), W,
                (S * K * Din, K * Din, Din, 1), B, S, K, Din, K)
      ops.bgemm(Qv, (N * K, 0, K, 1), W, (S * K * Din, K * Din, Din, 1), msg,
                (N * CD, Din, CD, 1), B, S, N, Din, K, c_off=col * Din)
    else:
      ops.bgemm(Qv, (N * K, 0, K, 1), U, (K * Din, 0, Din, 1), msg, (N * CD, Din, CD, 1),
                B, S, N, Din, K, kscale=coeff, s_str=(K * S, 1, S), c_off=col * Din)
    col += S
  # ---- edge types: L_e X (lanczos_net.py:177-178) -----------------------------------------
  ops.bgemm(L, (N * N * E1, 1, N * E1, E1), state, x_str, msg, (N * CD, Din, CD, 1),
            B, E1, N, Din, N, c_off=col * Din)
  # ---- Linear + ReLU (lanczos_net.py:180-181) ---------------------------------------------
  out = dense(msg.reshape(B * N, CD), weight, bias, True, cache, name)
  return out.reshape(B, N, -1)
