"""Shared host-side scaffolding of the three drop-in modules.

Parameter containers, names and initialisation mirror the reference so its checkpoints load
unchanged (model/lanczos_net.py:15-93, utils/train_helper.py:14-32): ``embedding.weight``,
``filter.{i}.{weight,bias}``, ``spectral_filter.{l}.{0,2,4,6}.{weight,bias}``,
``att_func.0.{weight,bias}``.  The forward math lives in CUDA (lanczosnetwork_b200.ops).
"""
import collections
import os

import torch
import torch.nn as nn

from .. import _lib, ops
from .. import data as data_mod
from ..data import check_dist, packed_capacity
from ..spectral_conv import (GraphContext, WeightCache, graph_conv_layer,
                             ritz_filter_coefficients)


class Ragged(object):
  """A tensor whose leading dimension varies from batch to batch (bond lists, rows of real nodes).
  CUDA-graph replay keeps a static buffer of ``capacity`` rows and copies only the rows present; the
  consumer kernels read their extents from the pointer arrays that travel with the batch.  The
  default capacity rounds the row count up to a bucket so batches of similar size share a graph."""

  def __init__(self, tensor, capacity=None, bucket=4096):
    self.tensor = tensor
    rows = int(tensor.shape[0])
    self.capacity = int(capacity) if capacity is not None else max(bucket, -(-rows // bucket) * bucket)
    if rows > self.capacity:
      raise ValueError('Ragged: %d rows exceed the capacity %d' % (rows, self.capacity))

  @property
  def rows(self):
    return int(self.tensor.shape[0])

  def static_shape(self):
    return (self.capacity,) + tuple(self.tensor.shape[1:])


def _raw(t):
  return t.tensor if isinstance(t, Ragged) else t


# the bond-list records of one batch on the device (data.sparse_collate's layout), N = padding target,
# K = eigenpairs per graph of a batch without them (sparse_collate(..., eigs=False)), else None
SparseRecords = collections.namedtuple('SparseRecords', 'sizes node_ptr node_feat edge_ptr edges N K',
                                       defaults=(None,))


def _opt(obj, name, default):
  return getattr(obj, name) if hasattr(obj, name) else default


def _check_records_shape(N, E1):
  """N and E+1 of a records or packed batch within the limits of the records producers."""
  if not (1 <= N <= ops.MAX_N and 2 <= E1 <= ops.MAX_E1):
    raise ValueError('forward_sparse: N=%d, E+1=%d outside 1 <= N <= %d, 2 <= E+1 <= %d'
                     % (N, E1, ops.MAX_N, ops.MAX_E1))


def loss_function(name):
  """The loss module of the config's ``model.loss`` (model/lanczos_net.py:64-71 and the other models)."""
  if name == 'CrossEntropy':
    return torch.nn.CrossEntropyLoss()
  elif name == 'MSE':
    return torch.nn.MSELoss()
  elif name == 'L1':
    return torch.nn.L1Loss()
  raise ValueError("Non-supported loss function!")


def init_linears(modules):
  """Xavier-uniform weights and zero biases of the nn.Linear among ``modules``, in the order given (the
  reference's order, so a seed gives its initial weights); other modules are skipped."""
  for mod in modules:
    if isinstance(mod, nn.Linear):
      nn.init.xavier_uniform_(mod.weight.data)
      if mod.bias is not None:
        mod.bias.data.zero_()


def init_cell(cell):
  """The reference's GRU / RNN cell initialisation: Xavier on weight_hh, then weight_ih, zero biases."""
  nn.init.xavier_uniform_(cell.weight_hh.data)
  nn.init.xavier_uniform_(cell.weight_ih.data)
  if cell.bias:
    cell.bias_hh.data.zero_()
    cell.bias_ih.data.zero_()


class SpectralNetBase(nn.Module):
  """Common constructor pieces; subclasses define the embedding and the long-scale operator."""

  # True: the records' node_feat holds float feature rows [rows, input_dim] (SparseLanczosNetGeneral), so a
  # packed batch must carry rows of that width (header slot F = input_dim); False: int32 atom ids (F = 0)
  _feature_records = False

  def _setup_fields(self, config, num_edgetype):
    """The config fields every drop-in keeps; ``num_atom`` where the dataset has atom types."""
    m = config.model
    self.config = config
    self.input_dim = m.input_dim
    self.hidden_dim = m.hidden_dim
    self.output_dim = m.output_dim
    self.num_layer = m.num_layer
    self.dropout = _opt(m, 'dropout', 0.0)
    if hasattr(config.dataset, 'num_atom'):
      self.num_atom = config.dataset.num_atom
    self.num_edgetype = num_edgetype
    self._wcache = WeightCache()

  def _setup_common(self, config, num_edgetype, filter_mlp_in, filter_mlp_hidden):
    self._setup_fields(config, num_edgetype)
    m = config.model
    self.short_diffusion_dist = check_dist(m.short_diffusion_dist)
    self.long_diffusion_dist = check_dist(m.long_diffusion_dist)
    self.max_short_diffusion_dist = max(self.short_diffusion_dist) if self.short_diffusion_dist else None
    self.max_long_diffusion_dist = max(self.long_diffusion_dist) if self.long_diffusion_dist else None
    self.num_scale_short = len(self.short_diffusion_dist)
    self.num_scale_long = len(self.long_diffusion_dist)
    self.num_eig_vec = m.num_eig_vec
    self.spectral_filter_kind = m.spectral_filter_kind
    self._filter_mlp_dims = (filter_mlp_in, filter_mlp_hidden)

  def _build_layers(self):
    C = self.num_scale_short + self.num_scale_long + self.num_edgetype + 1
    dims = [self.input_dim] + list(self.hidden_dim) + [self.output_dim]
    self.filter = nn.ModuleList(
        [nn.Linear(dims[t] * C, dims[t + 1]) for t in range(self.num_layer)] +
        [nn.Linear(dims[-2], dims[-1])])
    return dims

  def _build_spectral_filter(self):
    if self.spectral_filter_kind == 'MLP' and self.num_scale_long > 0:
      n_in, hid = self._filter_mlp_dims
      self.spectral_filter = nn.ModuleList([
          nn.Sequential(nn.Linear(n_in, hid), nn.ReLU(), nn.Linear(hid, hid), nn.ReLU(),
                        nn.Linear(hid, hid), nn.ReLU(), nn.Linear(hid, n_in))
          for _ in range(self.num_layer)
      ])

  def _build_head(self, dims):
    self.att_func = nn.Sequential(nn.Linear(dims[-2], 1), nn.Sigmoid())
    self.loss_func = loss_function(self.config.model.loss)

  def _init_param(self):
    """Xavier-uniform weights, zero biases for filter / att_func / spectral_filter Linears
    (model/lanczos_net.py:74-93); the embedding keeps nn.Embedding's default N(0,1)."""
    groups = [self.filter, self.att_func]
    if hasattr(self, 'spectral_filter'):
      groups += list(self.spectral_filter)
    init_linears([mod for grp in groups for mod in grp])

  def _forward(self, inputs, label):
    """The forward of every drop-in: the training path under autograd (``_check_mode``), otherwise the
    fused inference path ``_forward_impl`` through the CUDA-graph cache; then the loss when labelled."""
    dev = self._device()
    if self._check_mode():
      score = self._train_impl(*[self._to(dev, t) for t in inputs])
    else:
      score = self._graph_forward(self._forward_impl, inputs)
    return self._finish(score, self._to(dev, label))

  # ------------------------------------------------------------------------------------------
  def _param_device(self):
    return self.filter[0].weight.device

  def _device(self):
    dev = self._param_device()
    if dev.type != 'cuda':
      raise RuntimeError(
          '%s runs on CUDA (sm_90a) only -- move the module with .cuda(); there is no CPU '
          'fallback (the CPU reference is the oracle).' % type(self).__name__)
    # DataParallel replicas share the master's WeightCache object: bypass it there (see WeightCache)
    if getattr(self, '_is_replica', False) and hasattr(self, '_wcache') and not self._wcache.bypass:
      self._wcache = type(self._wcache)()
      self._wcache.bypass = True
    return dev

  def invalidate_caches(self):
    """Drop the cached tf32 weight splits and the captured CUDA graphs (call after editing weights
    through ``p.data`` or any other route that does not bump the parameters' version counters)."""
    if hasattr(self, '_wcache'):
      self._wcache.invalidate()
    for name in ('_graphs', '_graphs_resident', '_resident_seen'):
      self.__dict__.pop(name, None)

  def graph_stats(self):
    """Counters of the CUDA-graph cache: captures (each costs a warm-up, two captures and two device
    synchronisations), replays, and live graphs -- a capture count that keeps growing means the input
    shapes thrash the cache (pad / bucket the batch shapes)."""
    st = self.__dict__.setdefault('_graph_stats', {'captures': 0, 'replays': 0})
    return dict(st, live=len(self.__dict__.get('_graphs', {})),
                live_resident=len(self.__dict__.get('_graphs_resident', {})))

  def _has_trainable_parameters(self):
    """nn.DataParallel replicas hold their parameter copies as plain attributes (``parameters()`` is
    empty there, the copies are listed in ``_former_parameters``): look at both."""
    for m in self.modules():
      for group in (m._parameters, getattr(m, '_former_parameters', None) or {}):
        for p in group.values():
          if p is not None and p.requires_grad:
            return True
    return False

  def _check_mode(self):
    """Returns True when this call has to be differentiable (autograd on, trainable parameters):
    the forward then runs the training path of lanczosnetwork_b200.train (unfused, every
    contraction and its adjoint in this library's kernels) instead of the fused inference kernels.
    Models without a training path raise."""
    if torch.is_grad_enabled() and self._has_trainable_parameters():
      if not hasattr(self, '_train_impl'):
        raise NotImplementedError(
            '%s has no training path in this build: call it under torch.no_grad() (as '
            'runner.test() / the validation loop do).' % type(self).__name__)
      return True
    if self.training and self.dropout > 0.0:
      raise NotImplementedError('dropout > 0 in training mode needs autograd enabled (the inference '
                                'kernels implement eval() semantics)')
    return False

  @staticmethod
  def _to(dev, t, dtype=None):
    if t is None:
      return None
    if t.device != dev:
      t = t.to(dev, non_blocking=True)
    if dtype is not None and t.dtype != dtype:
      t = t.to(dtype)
    return t

  # ------------------------------------------------------------------------------------------
  # Forward from a sparse batch (data.sparse_collate): the padded inputs are built on the device.
  SPARSE_KEYS = ('sizes', 'node_ptr', 'node_feat', 'edge_ptr', 'edges', 'N')

  def forward_sparse(self, batch, label=None):
    """Forward from a SPARSE batch (data.sparse_collate -> torch tensors, pinned host or device):
    per-molecule node ids and bond lists; ``D`` / ``V_rows``, when present, are read only by the models
    that consume eigenpairs.  The padded node ids, mask, ELL rows and whatever else the model reads are
    built on the device (lnb_graph_prepare_sparse and the model's own producers): the dense
    B x N x N x (E+1) tensor of the reference's collate never crosses PCIe.  Same scores as ``forward``
    on the collated batch, bit for bit.  Inference only (raises under autograd).  Returns score or
    (score, loss).

    A packed batch (data.pack_sparse / data.PackedMolecules.batch: one uint8 blob, with or without
    eigenpairs) is taken too: one copy of the blob, then lnb_records_unpack splits it into the records on
    the device, inside the same captured graph, and the model runs exactly as on those records."""
    if self._check_mode():
      raise NotImplementedError('forward_sparse is an inference path; train through forward() or, from '
                                'the same records, forward_sparse_train()')
    dev = self._device()
    inputs, impl, key = self._sparse_inputs(batch)
    score = self._graph_forward(impl, inputs, extra_key=key)
    return self._finish(score, self._to(dev, label))

  def forward_sparse_train(self, batch, label=None):
    """Differentiable forward from the same SPARSE batch as ``forward_sparse`` (data.sparse_collate
    records, pinned host or device): the training formulation of lanczosnetwork_b200.train with its
    operator products and adjoints over the ELL rows that lnb_graph_prepare_sparse builds
    (ops.ell_messages), so neither the padded operators nor their host collate exist.  It runs the
    training formulation whether or not autograd is on, applies the batch checks of ``forward_sparse``
    before any device work, and takes no packed batch.  Returns score or (score, loss)."""
    if not hasattr(self, '_train_records'):
      raise NotImplementedError('%s has no training entry from sparse batches; train it through forward() '
                                'on the collated batch' % type(self).__name__)
    if 'blob' in batch:
      raise NotImplementedError('%s.forward_sparse_train takes data.sparse_collate records, not packed '
                                'batches' % type(self).__name__)
    inputs, _, _ = self._sparse_inputs(batch)
    dev = self._device()
    raw = [self._to(dev, _raw(t)) for t in inputs]
    recs = SparseRecords(*raw[:5], N=int(batch['N']), K=int(batch['K']) if 'K' in batch else None)
    return self._finish(self._train_records(recs, *raw[5:]), self._to(dev, label))

  def _sparse_inputs(self, batch):
    """(inputs, impl, extra_key) of _graph_forward for a sparse batch: the bond-list records, whose
    device batch goes to the model's ``_forward_records`` hook."""
    if not hasattr(self, '_forward_records'):
      raise NotImplementedError('%s has no sparse-batch entry; call forward() on the collated batch'
                                % type(self).__name__)
    if 'blob' in batch:
      blob, unpack, key = self._packed_records(batch)
      return (blob,), lambda b_: self._forward_records(unpack(b_)), key
    N, B, E1 = self._check_sparse_batch(batch)
    self._check_runnable(N, E1)
    inputs = (batch['sizes'], batch['node_ptr'], Ragged(batch['node_feat'], B * N), batch['edge_ptr'],
              Ragged(batch['edges']))
    return inputs, lambda *a: self._forward_records(SparseRecords(*a, N=N)), ('records', N)

  def _check_sparse_batch(self, batch, feature_dim=None):
    """forward_sparse's checks of a records batch, before any device work: the keys, N and E+1 within the
    prepare kernel's limits, int32 pointers, uint8 [E, 4] bonds, and int32 atom ids -- or, with
    ``feature_dim``, float32 [rows, feature_dim] feature rows.  Returns (N, B, E1)."""
    missing = [k for k in self.SPARSE_KEYS if k not in batch]
    if missing:
      raise ValueError('forward_sparse: the batch lacks %s (data.sparse_collate records)' % ', '.join(missing))
    N, B = int(batch['N']), int(batch['sizes'].shape[0])
    E1 = self.num_edgetype + 1
    _check_records_shape(N, E1)
    for k in ('sizes', 'node_ptr', 'node_feat', 'edge_ptr'):
      if k == 'node_feat' and feature_dim is not None:
        nf = batch[k]
        if nf.dtype != torch.float32 or nf.dim() != 2 or nf.shape[1] != feature_dim:
          raise ValueError('forward_sparse: node_feat must be float32 feature rows [rows, %d]; got %s %s'
                           % (feature_dim, nf.dtype, tuple(nf.shape)))
      elif batch[k].dtype != torch.int32:
        raise ValueError('forward_sparse: %s must be int32; got %s' % (k, batch[k].dtype))
    if batch['edges'].dtype != torch.uint8 or batch['edges'].dim() != 2 or batch['edges'].shape[1] != 4:
      raise ValueError('forward_sparse: edges must be uint8 [E, 4]')
    return N, B, E1

  PACKED_KEYS = ('blob', 'B', 'N', 'K')

  def _packed_width(self):
    """The width F of the node rows this model reads from a packed batch: input_dim for float feature rows,
    0 for atom ids."""
    return int(self.input_dim) if self._feature_records else 0

  @staticmethod
  def _blob_width(batch):
    """The node-row width F a packed batch names: batch['F'], else its blob's header slot (a device blob with a
    small synchronous copy); None when neither can be read."""
    if 'F' in batch:
      return int(batch['F'])
    blob = batch.get('blob')
    if (not torch.is_tensor(blob) or blob.dtype != torch.uint8 or blob.dim() != 1 or blob.numel() < 64 or
        (blob.is_cuda and torch.cuda.is_current_stream_capturing())):
      return None
    return data_mod.read_packed_header(blob).F

  def _check_packed_width(self, F):
    """A packed batch's node-row width F against the model's: an atom-id blob given to a feature model raises
    NotImplementedError, a feature blob given to an atom-id model or one of another width ValueError."""
    want = self._packed_width()
    if F == want:
      return
    if want and not F:
      raise NotImplementedError('%s takes packed batches of float feature rows (F = %d), not packed batches of '
                                'atom ids' % (type(self).__name__, want))
    if not want:
      raise ValueError('forward_sparse: %s reads atom ids; the packed batch holds float feature rows (F = %d)'
                       % (type(self).__name__, F))
    raise ValueError('forward_sparse: the packed batch holds feature rows of width F = %d; %s reads input_dim = %d'
                     % (F, type(self).__name__, want))

  def _check_packed_batch(self, batch):
    """forward_sparse's checks of a packed batch (data.pack_sparse / data.PackedMolecules.batch), before any
    device work: the keys, a flat uint8 blob, N and E+1 within the prepare kernel's limits, and the blob's
    header -- magic, B and K against the batch's, the total size, node_ptr[B] <= B * N, the node-row width F
    against the model's -- which also says whether the blob carries eigenpairs.  A host blob is read in place.
    A device blob is read with two small synchronous copies unless the batch says both ``eigs`` and ``F``
    (pack_sparse and PackedMolecules.batch do; for an atom-id model a missing ``F`` means 0): then nothing is
    read on the host, both are trusted -- LanczosNet runs an eigenpair blob through
    lnb_graph_prepare_sparse_packed, which reads the Ritz rows, so ``eigs`` must be right -- and the header is
    checked by lnb_records_unpack on the device only; a batch that fails there gives the scores of empty
    graphs.  Returns (B, N, K, eigs, header): the data.PackHeader read, None when nothing was read."""
    if self._feature_records and self._blob_width(batch) == 0:
      self._check_packed_width(0)                # an atom-id blob is refused first, whatever else it lacks
    missing = [k for k in self.PACKED_KEYS if k not in batch]
    if missing:
      raise ValueError('forward_sparse: the packed batch lacks %s (data.pack_sparse)' % ', '.join(missing))
    blob = batch['blob']
    if not torch.is_tensor(blob) or blob.dtype != torch.uint8 or blob.dim() != 1 or blob.numel() < 64:
      raise ValueError('forward_sparse: blob must be a flat uint8 tensor of at least 64 bytes')
    B, N, K = int(batch['B']), int(batch['N']), int(batch['K'])
    E1 = self.num_edgetype + 1
    _check_records_shape(N, E1)
    if B < 1 or K < 1:
      raise ValueError('forward_sparse: packed batch with B=%d, K=%d' % (B, K))
    eigs = batch.get('eigs')
    F = batch.get('F', None if self._feature_records else 0)
    if F is not None:
      self._check_packed_width(int(F))
    if blob.is_cuda and eigs is not None and F is not None:
      return B, N, K, bool(eigs), None
    if blob.is_cuda and torch.cuda.is_current_stream_capturing():
      raise ValueError("forward_sparse: a device blob under stream capture needs batch['eigs'] and batch['F'] (its "
                       "header cannot be read on the host there)")

    hdr = data_mod.read_packed_header(blob)
    if hdr.magic != data_mod.PACK_MAGIC:
      raise ValueError('forward_sparse: blob magic %#x is not %#x (data.pack_sparse)' % (hdr.magic & 0xffffffff,
                                                                                         data_mod.PACK_MAGIC))
    if (hdr.B, hdr.K) != (B, K):
      raise ValueError('forward_sparse: blob header has B=%d, K=%d; the batch says B=%d, K=%d'
                       % (hdr.B, hdr.K, B, K))
    if 'F' in batch and hdr.F != int(batch['F']):
      raise ValueError("forward_sparse: batch['F'] is %d, the blob header says F=%d" % (int(batch['F']), hdr.F))
    self._check_packed_width(hdr.F)
    if not 64 <= hdr.total <= blob.numel():
      raise ValueError('forward_sparse: blob header total %d bytes outside [64, %d]' % (hdr.total, blob.numel()))
    if not (64 <= hdr.node_ptr and hdr.node_ptr % 16 == 0 and hdr.node_ptr + 4 * (B + 1) <= hdr.total):
      raise ValueError('forward_sparse: blob node_ptr offset %d outside the blob' % hdr.node_ptr)
    rows = blob[hdr.node_ptr + 4 * B:][:4].cpu().view(torch.int32).item()     # node_ptr[B], a second read
    if not 0 <= rows <= B * N:
      raise ValueError('forward_sparse: node_ptr[B]=%d node rows outside [0, B*N = %d]' % (rows, B * N))
    has = hdr.D != 0 or hdr.V_rows != 0
    if eigs is not None and bool(eigs) != has:
      raise ValueError("forward_sparse: batch['eigs'] is %s, the blob %s eigenpairs"
                       % (bool(eigs), 'carries' if has else 'has no'))
    return B, N, K, has, hdr

  def _packed_records(self, batch):
    """(blob input, unpack, graph-cache key) of a packed batch for a model with a records entry: the blob
    as ONE Ragged input whose capacity depends on (B, N, K) only, and ``unpack(device_blob)``, the
    SparseRecords that lnb_records_unpack writes from it into fixed-capacity buffers (node rows B * N, the
    bonds the blob's capacity can hold), so one captured graph serves every batch of the same shape."""
    B, N, K, eigs, _ = self._check_packed_batch(batch)
    self._check_runnable(N, self.num_edgetype + 1)
    blob = batch['blob']
    return (Ragged(blob, self._packed_capacity(B, N, K, eigs, blob.shape[0])),
            lambda b_: self._unpack(b_, B, N, K)[0], ('packed_records', B, N, K))

  def _packed_capacity(self, B, N, K, eigs, nbytes, label_dim=0):
    """data.packed_capacity of this model's packed batches (node rows of its width, its bond types)."""
    return packed_capacity(B, N, K, eigs, nbytes, label_dim, self._packed_width(), self.num_edgetype)

  def _takes_packed_training(self, batch):
    """True when ``train.GraphedStep(..., packed=True)`` trains this model from ``batch``: it has a training
    entry from records and its ``forward_sparse`` takes packed batches."""
    return hasattr(self, '_train_records') and hasattr(self, '_forward_records')

  def _check_packed_train(self, batch):
    """GraphedStep(packed=True)'s checks of a labelled packed batch, before any copy: those of
    ``forward_sparse`` with the header always read (a device blob with a small synchronous copy, even when the
    batch says ``eigs``: a training step must never run on a batch the device would refuse), and a label
    segment inside the blob.  Returns (header, N, eigs), the header a data.PackHeader."""
    B, N, K, eigs, hdr = self._check_packed_batch({k: v for k, v in batch.items() if k != 'eigs'})
    if 'eigs' in batch and bool(batch['eigs']) != eigs:
      raise ValueError("GraphedStep: batch['eigs'] is %s, the blob %s eigenpairs"
                       % (bool(batch['eigs']), 'carries' if eigs else 'has no'))
    if hdr.P < 1 or hdr.label < 64 or hdr.label % 16 or hdr.label + 4 * B * hdr.P > hdr.total:
      raise ValueError('GraphedStep: the packed batch carries no labels (label offset %d, P=%d): build it with '
                       'data.pack_sparse(..., label=True) or data.PackedMolecules(..., labels=True)'
                       % (hdr.label, hdr.P))
    return hdr, N, eigs

  def _train_packed(self, batch, P):
    """The training forward of a device blob with labels (the static batch of GraphedStep(packed=True)):
    lnb_records_unpack_labels into fixed-capacity records, then ``_train_records`` with whatever key the batch
    carries after the blob, as ``forward_sparse_train`` passes it.  Returns (score, label [B, P], status)."""
    inputs, _, _ = self._sparse_inputs(batch)
    B, N, K = int(batch['B']), int(batch['N']), int(batch['K'])
    recs, _, _, label, status = self._unpack(batch['blob'], B, N, K, P)
    return self._train_records(recs, *[_raw(t) for t in inputs[1:]]), label, status

  def _unpack(self, blob, B, N, K, P=0, eigs=False):
    """ops.records_unpack of a device blob into fixed-capacity records: B * N node rows, and as many bonds as
    the bytes past D's offset hold (the bonds lie behind it, with or without eigenpairs); P > 0 adds the labels.
    Returns (SparseRecords, D, V_rows[, label [B, P]], status), D and V_rows None without ``eigs``."""
    cap_edges = (blob.shape[0] - data_mod.packed_offsets(B, K).D) // 4
    out = ops.records_unpack(blob, B, K, B * N, cap_edges, eigs=eigs, label_dim=P, feature_dim=self._packed_width())
    return (SparseRecords(*out[:5], N=N, K=K),) + tuple(out[5:])

  def _check_runnable(self, N=None, E1=None):
    """Model-specific checks of a call, run before any launch (N, E1: those of a sparse batch)."""

  def _prepare_records(self, recs, binarize=False, want_dense=False):
    """lnb_graph_prepare_sparse on the records without Ritz vectors (the zero [rows, 4] block, as the
    padded path's zero [B, N, 4]): (GraphPrep, node_ids [B,N] int64, mask [B,N] uint8, V = zeros [B,N,4],
    dense L or None)."""
    V_rows = torch.zeros((recs.node_feat.shape[0], 4), device=recs.sizes.device, dtype=torch.float32)
    return ops.graph_prepare_sparse(recs.sizes, recs.node_ptr, recs.node_feat, recs.edge_ptr, recs.edges,
                                    V_rows, recs.N, self.num_edgetype + 1, binarize=binarize,
                                    want_dense=want_dense)

  # ------------------------------------------------------------------------------------------
  # CUDA-graph replay of the inference forward: the forward is ~15 short kernel launches issued
  # through ctypes; capturing them once per input signature removes the per-launch host cost
  # (CUDA streams and graphs instead of a tracing compiler).  Inputs are copied into static
  # buffers (H2D straight from pinned host memory, or D2D), the graph is replayed, the small
  # score tensor is cloned out.  Recaptured when shapes or any parameter version change.
  use_cuda_graph = os.environ.get('LNB_NO_GRAPH', '0') != '1'   # LNB_NO_GRAPH=1: eager (profiling)

  def _param_signature(self):
    return tuple((p.data_ptr(), p._version) for p in self.parameters())

  def _graph_forward(self, impl, inputs, extra_key=()):
    """impl(*device_tensors) -> score; inputs: tuple of tensors / Ragged / None (CPU or CUDA).

    Two graph slots with their own static buffers alternate, and the input copies run on a
    dedicated copy stream: the H2D (or D2D) transfer of call i+1 overlaps the replay of call i
    (the forward returns without synchronising), ordered by events only."""
    dev = self._device()
    eligible = (self.use_cuda_graph and not self.training and not torch.is_grad_enabled() and
                not getattr(self, '_is_replica', False) and
                not torch.cuda.is_current_stream_capturing())
    if not eligible:
      return impl(*[self._to(dev, _raw(t)) for t in inputs])
    key = (dev.index,) + tuple(extra_key) + tuple(
        None if t is None else ((t.static_shape(), t.tensor.dtype, 'ragged') if isinstance(t, Ragged)
                                else (tuple(t.shape), t.dtype)) for t in inputs)
    cache = self.__dict__.setdefault('_graphs', {})
    stats = self.__dict__.setdefault('_graph_stats', {'captures': 0, 'replays': 0})
    entry = cache.get(key)
    if entry is not None:
      cache[key] = cache.pop(key)               # LRU: most recently used last
    sig = self._param_signature()
    cur = torch.cuda.current_stream(dev)
    # Inputs already resident on this device: a graph bound to their addresses needs no copy at
    # all.  Such a graph is captured the second time the same buffers show up (data loaders /
    # serving loops that recycle a few device buffers); any live tensor found at a captured
    # address with the captured shape and dtype is read correctly, so no reference is kept.  The key
    # holds a Ragged input's own row count too: the captured forward reads the tensor it was given,
    # so a slice of another length at the same address is another graph.
    raw = [_raw(t) for t in inputs]
    if all(t is None or (t.is_cuda and t.device == dev and t.is_contiguous()) for t in raw):
      pkey = key + tuple(None if t is None else t.data_ptr() for t in raw) + tuple(
          t.rows for t in inputs if isinstance(t, Ragged))
      zc = self.__dict__.setdefault('_graphs_resident', {})
      hit = zc.get(pkey)
      if hit is not None and hit['sig'] == sig:
        zc[pkey] = zc.pop(pkey)
        stats['replays'] += 1
        hit['graph'].replay()
        _lib.note_graph_replay(hit['kernels'])
        return hit['out'].clone()
      seen = self.__dict__.setdefault('_resident_seen', {})
      if len(seen) > 256:
        seen.clear()
      seen[pkey] = seen.get(pkey, 0) + 1
      if seen[pkey] >= 2 and entry is not None and entry['sig'] == sig:   # caches are warm
        if len(zc) >= 16:
          zc.pop(next(iter(zc)))
        if '_resident_pool' not in self.__dict__:
          self._resident_pool = torch.cuda.graph_pool_handle()
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        n0 = int(_lib.load().lnb_launch_count())
        with torch.cuda.graph(graph, pool=self._resident_pool):
          out = impl(*raw)
        hit = {'graph': graph, 'out': out, 'sig': sig,
               'kernels': int(_lib.load().lnb_launch_count()) - n0}
        zc[pkey] = hit
        stats['captures'] += 1
        graph.replay()
        _lib.note_graph_replay(hit['kernels'])
        return out.clone()
    if entry is None or entry['sig'] != sig:
      slots = []
      for _ in range(2):
        static_in = [None if t is None else
                     (torch.zeros(t.static_shape(), dtype=t.tensor.dtype, device=dev)
                      if isinstance(t, Ragged) else torch.empty(t.shape, dtype=t.dtype, device=dev))
                     for t in inputs]
        for s_, t in zip(static_in, inputs):
          if isinstance(t, Ragged):
            s_[:t.rows].copy_(t.tensor, non_blocking=True)
          elif s_ is not None:
            s_.copy_(t, non_blocking=True)
        if not slots:
          side = torch.cuda.Stream(device=dev)
          side.wait_stream(cur)
          with torch.cuda.stream(side):
            impl(*static_in)                   # warm-up: fills the weight caches
          cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        n0 = int(_lib.load().lnb_launch_count())
        with torch.cuda.graph(graph):
          static_out = impl(*static_in)
        slots.append({'graph': graph, 'in': static_in, 'out': static_out,
                      'kernels': int(_lib.load().lnb_launch_count()) - n0,
                      'free': torch.cuda.Event(), 'ready': torch.cuda.Event()})
        slots[-1]['free'].record(cur)
      entry = {'sig': sig, 'slots': slots, 'next': 0, 'copy': torch.cuda.Stream(device=dev)}
      stats['captures'] += 1
      cache.pop(key, None)
      if len(cache) >= 8:                      # bound the number of live graphs: evict the LRU entry
        cache.pop(next(iter(cache)))
      cache[key] = entry
    slot = entry['slots'][entry['next']]
    entry['next'] ^= 1
    copy = entry['copy']
    copy.wait_event(slot['free'])              # the previous replay of this slot has consumed its inputs
    if any(t is not None and t.is_cuda for t in raw):
      copy.wait_stream(cur)                    # device inputs produced on the caller's stream
    with torch.cuda.stream(copy):
      for s_, t in zip(slot['in'], inputs):
        if isinstance(t, Ragged):
          s_[:t.rows].copy_(t.tensor, non_blocking=True)     # only the rows present cross PCIe
        elif s_ is not None:
          s_.copy_(t, non_blocking=True)
      slot['ready'].record(copy)
    cur.wait_event(slot['ready'])
    stats['replays'] += 1
    slot['graph'].replay()
    slot['free'].record(cur)
    _lib.note_graph_replay(slot['kernels'])
    return slot['out'].clone()

  def _filter_mlp_params(self):
    if not hasattr(self, 'spectral_filter'):
      return None
    out = []
    for l, seq in enumerate(self.spectral_filter):
      out.append([('spectral_filter.%d.%d' % (l, i), seq[i].weight, seq[i].bias)
                  for i in (0, 2, 4, 6)])
    return out

  def _ritz_conv_stack(self, state, node_ids, L, D, V, mask, prep=None, dims_hint=None):
    """Convolution stack + readout of the Ritz-pair models (LanczosNet, LanczosNetGeneral).
    ``prep`` (ops.GraphPrep built on the device by ops.graph_prepare_sparse) replaces the pass over
    the dense operators; ``L`` may then be None when every layer runs in the fused stack
    (``dims_hint`` = (N, E1) of the absent tensor).

    Consecutive layers the fused kernel supports run as ONE persistent launch (embedding gather
    in front when every layer qualifies, readout behind); a leading layer with an unsupported
    input width (e.g. LanczosNetGeneral's 10 features) runs through the unfused ops first."""
    S, nl = self.num_scale_long, self.num_layer
    if L is not None:
      N, K, E1 = L.shape[1], V.shape[2], L.shape[3]
    else:
      (N, E1), K = dims_hint, V.shape[2]
    din0 = self.embedding.weight.shape[1] if node_ids is not None else state.shape[2]
    dims = [din0] + list(self.hidden_dim)
    ok = [ops.fused_conv_supported(N, dims[t], K, dims[t + 1], len(self.short_diffusion_dist),
                                   False, S, E1) for t in range(nl)]
    H = dims[1]
    uniform = all(d == H for d in dims[1:])
    first = 0
    while first < nl and not ok[first]:
      first += 1
    stack_ok = uniform and first < nl and all(ok[first:]) and nl - first <= ops.CONV_MAX_LAYERS
    binarize = getattr(self, '_binarize_operators', False)
    if binarize and not (stack_ok and first == 0):
      L = (L != 0).to(L.dtype)          # shapes off the fused path read the dense operators
      binarize = False
    if L is None and not (stack_ok and first == 0):
      raise RuntimeError('sparse batches without the dense operators need every layer on the fused '
                         'stack kernel; call ops.graph_prepare_sparse(..., want_dense=True)')
    ctx = GraphContext(L, V, binarize)
    if prep is not None:
      ctx._prep = prep
    coeffs = table = None
    if S > 0:
      mlp = self._filter_mlp_params() if self.spectral_filter_kind == 'MLP' else None
      # the power table does not depend on graph_prepare: fork it onto a side stream so the
      # two run concurrently (also inside the captured graph)
      cur = torch.cuda.current_stream(D.device)
      side = self.__dict__.setdefault('_side_streams', {}).get(D.device.index)
      if side is None:
        side = self._side_streams[D.device.index] = torch.cuda.Stream(device=D.device)
      side.wait_stream(cur)
      with torch.cuda.stream(side):
        table = ops.ritz_power_table(D, self.long_diffusion_dist)
      table.record_stream(cur)
      gext = ctx.prep(defer_tiles=True) if (mlp is not None and stack_ok and first == 0) else None
      cur.wait_stream(side)
      ctas = 0
      if gext is not None and gext.tiles_pending:
        # the chain reads only the Ritz row list: the tile placement (one CTA) runs on the side
        # stream beside it and is joined before the stack.  The chain gets one SM fewer, so none of
        # its CTAs waits behind the placement's SM.
        side.wait_stream(cur)
        with torch.cuda.stream(side):
          ops.tile_assign(gext, K)
        ctas = torch.cuda.get_device_properties(D.device).multi_processor_count - 1
      coeffs, table = ritz_filter_coefficients(D, self.long_diffusion_dist, mlp, self._wcache, gext,
                                               table=table, ctas=ctas)
      cur.wait_stream(side)

    def layer_coeff(t):
      if S == 0:
        return None
      return coeffs[t] if coeffs is not None else table

    if node_ids is not None and not (stack_ok and first == 0):
      state = ops.embedding_rows(node_ids, self.embedding.weight)
    for t in range(first if stack_ok else nl):           # unfused / single-layer prefix
      state = graph_conv_layer(state, ctx, layer_coeff(t), False, self.short_diffusion_dist, S,
                               self.filter[t].weight, self.filter[t].bias, self._wcache,
                               'filter.%d' % t, last=(t == nl - 1),
                               next_fused=(t + 1 < nl and ok[t + 1]))
    if not stack_ok:
      return self._readout(state, mask)
    layers = list(range(first, nl))
    kw = (S + E1) * max(dims[t] for t in layers)
    w_hi, w_lo, bias = self._wcache.split_conv_stack(
        'filter.stack.%d' % first, [self.filter[t].weight for t in layers],
        [self.filter[t].bias for t in layers], kw)
    if S == 0:
      coeff, stride = None, 0
    elif coeffs is not None:
      coeff, stride = coeffs[first], coeffs.stride(0)
    else:
      coeff, stride = table, 0
    head, att = self.filter[nl], self.att_func[0]
    if head.weight.shape[0] > 48:                        # fused readout holds <= 48 outputs
      state, _ = ops.spectral_stack_forward(
          ctx.prep(), V, w_hi, w_lo, bias, [dims[t] for t in layers], H, S, coeff=coeff,
          coeff_stride=stride, X=None if (node_ids is not None and first == 0) else state,
          node_ids=node_ids if first == 0 else None,
          emb=self.embedding.weight if (node_ids is not None and first == 0) else None,
          want_state=True)
      return self._readout(state, mask)
    _, score = ops.spectral_stack_forward(
        ctx.prep(), V, w_hi, w_lo, bias, [dims[t] for t in layers], H, S, coeff=coeff,
        coeff_stride=stride, X=None if (node_ids is not None and first == 0) else state,
        node_ids=node_ids if first == 0 else None,
        emb=self.embedding.weight if (node_ids is not None and first == 0) else None,
        readout=(head.weight, head.bias, att.weight.reshape(-1), att.bias), mask=mask)
    return score

  def _sparse_stack_ok(self, N, E1, K, din0=None):
    """True when every layer of this model runs inside the one-launch stack kernel, so a sparse
    batch never needs the dense operator tensor.  ``din0``: the input width (default: the embedding's)."""
    S = self.num_scale_long
    if din0 is None:
      din0 = self.embedding.weight.shape[1]
    dims = [din0] + list(self.hidden_dim)
    ok = all(ops.fused_conv_supported(N, dims[t], K, dims[t + 1], len(self.short_diffusion_dist), False, S, E1)
             for t in range(self.num_layer))
    return ok and all(d == dims[1] for d in dims[1:]) and self.num_layer <= ops.CONV_MAX_LAYERS

  def _readout(self, state, mask):
    head = self.filter[self.num_layer]
    att = self.att_func[0]
    return ops.readout(state, head.weight, head.bias, att.weight.reshape(-1), att.bias, mask)

  def _finish(self, score, label):
    if label is not None:
      return score, self.loss_func(score, label)
    return score


class RitzRecords(object):
  """The entries from bond-list records of the Ritz-pair models, mixed in front of SpectralNetBase:
  ``forward_sparse`` / ``forward_sparse_train`` / ``GraphedStep(sparse=True)`` over records that carry the
  eigenpairs of the real nodes (``V_rows``, ``D``) or only K (``data.sparse_collate(..., eigs=False)``: one
  lnb_graph_eigs_sparse launch in front of the batch construction, inside the same CUDA graph -- no host
  eigh, no eigenvector bytes on the bus).  ``_feature_records`` is the one difference between the users:
  False, ``node_feat`` holds atom ids and the stack gathers the embedding (LanczosNet); True, it holds float
  feature rows [rows, input_dim] that the prepare kernel pads into X (SparseLanczosNetGeneral).  Packed
  batches (data.pack_sparse) hold the same node rows: atom ids, or feature rows of width F = input_dim."""

  def _sparse_inputs(self, batch):
    feat = self._feature_records
    if 'blob' in batch:
      # a packed batch (data.pack_sparse) crosses PCIe as ONE copy of exactly the bytes present
      B, N, K, eigs, _ = self._check_packed_batch(batch)
      inputs = (Ragged(batch['blob'], self._packed_capacity(B, N, K, eigs, batch['blob'].shape[0])),)
      if not eigs:
        # without eigenpairs: records_unpack, then the path of records without them
        return (inputs, lambda b_: self._forward_sparse_eigs_impl(N, K, *self._unpack(b_, B, N, K)[0][:5]),
                ('packed_eigs', B, N, K))
      return inputs, lambda b_: self._forward_packed_impl(B, N, K, b_), ('packed', B, N, K)
    if feat:
      self._check_ritz_records(batch)
    N, B = int(batch['N']), int(batch['sizes'].shape[0])
    if 'V_rows' not in batch and 'D' not in batch:
      K = int(batch['K'])
      inputs = (batch['sizes'], batch['node_ptr'], Ragged(batch['node_feat'], B * N), batch['edge_ptr'],
                Ragged(batch['edges']))
      return inputs, lambda *a: self._forward_sparse_eigs_impl(N, K, *a), ('sparse_eigs', N, K)
    inputs = (batch['sizes'], batch['node_ptr'], Ragged(batch['node_feat'], B * N), batch['edge_ptr'],
              Ragged(batch['edges']), Ragged(batch['V_rows'], B * N), batch['D'])
    return inputs, lambda *a: self._forward_sparse_impl(N, *a), ('sparse', N)

  def _check_ritz_records(self, batch):
    """The batch checks of feature records: those of every drop-in with float32 [rows, input_dim] feature
    rows, then either K alone or both eigenpair arrays."""
    _, B, _ = self._check_sparse_batch(batch, feature_dim=self.input_dim)
    if ('V_rows' in batch) != ('D' in batch):
      raise ValueError('forward_sparse: records carry both V_rows and D, or neither (then K)')
    if 'V_rows' not in batch:
      if 'K' not in batch:
        raise ValueError('forward_sparse: records without eigenpairs need K (data.sparse_collate(..., eigs=False))')
      return
    V_rows, D = batch['V_rows'], batch['D']
    if (V_rows.dtype != torch.float32 or V_rows.dim() != 2 or D.dtype != torch.float32 or
        tuple(D.shape) != (B, V_rows.shape[1])):
      raise ValueError('forward_sparse: V_rows must be float32 [rows, K] and D float32 [B, K]; got %s %s and %s %s'
                       % (V_rows.dtype, tuple(V_rows.shape), D.dtype, tuple(D.shape)))

  def _takes_packed_training(self, batch):
    """A feature model trains from blobs of feature rows only: given an atom-id blob (or no packed batch) it is
    outside GraphedStep(packed=True)'s list, which names it."""
    return not self._feature_records or bool(self._blob_width(batch))

  def _train_packed(self, batch, P):
    """A labelled blob with eigenpairs trains on its D and V_rows; one without gets them from
    lnb_graph_eigs_sparse, as records without them do."""
    recs, D, V_rows, label, status = self._unpack(batch['blob'], int(batch['B']), int(batch['N']),
                                                  int(batch['K']), P, eigs=bool(batch['eigs']))
    return self._train_records(recs, V_rows, D), label, status

  def _prepare_ritz_records(self, sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, N, **kw):
    """(GraphPrep, node ids or padded features X, mask, V, L or None) of the records."""
    prepare = ops.graph_prepare_sparse_features if self._feature_records else ops.graph_prepare_sparse
    return prepare(sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, N, self.num_edgetype + 1, **kw)

  def _forward_packed_impl(self, B, N, K, blob):
    """The forward of a device blob with eigenpairs: one lnb_graph_prepare_sparse(_features)_packed launch reads
    the segments in place, D at its fixed offset, and the tiles come with the blob."""
    E1 = self.num_edgetype + 1
    F = self._packed_width()
    dense = not self._sparse_stack_ok(N, E1, K, F or None)
    off_D = data_mod.packed_offsets(B, K).D
    D = blob[off_D:off_D + 4 * B * K].view(torch.float32).reshape(B, K)     # fixed address in the buffer
    prep, x, mask, V, L = ops.graph_prepare_sparse_packed(
        blob, B, N, E1, K, binarize=getattr(self, '_binarize_operators', False), want_dense=dense, feature_dim=F)
    return self._ritz_conv_stack(*self._ritz_inputs(x), L, D, V, mask, prep=prep, dims_hint=(N, E1))

  def _ritz_inputs(self, x):
    """(state, node_ids) of _ritz_conv_stack / ritz_stack_train for the prepare kernel's node output."""
    return (x, None) if self._feature_records else (None, x)

  def _forward_sparse_impl(self, N, sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, D):
    E1 = self.num_edgetype + 1
    K = V_rows.shape[1]
    dense = not self._sparse_stack_ok(N, E1, K, node_feat.shape[1] if self._feature_records else None)
    prep, x, mask, V, L = self._prepare_ritz_records(
        sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, N,
        binarize=getattr(self, '_binarize_operators', False), want_dense=dense, defer_tiles=True)
    return self._ritz_conv_stack(*self._ritz_inputs(x), L, D.float().contiguous(), V, mask, prep=prep,
                                 dims_hint=(N, E1))

  def _forward_sparse_eigs_impl(self, N, K, sizes, node_ptr, node_feat, edge_ptr, edges):
    # V_rows has node_feat's rows (the static capacity under graph replay); rows past node_ptr[B] are
    # written by nobody and read by nobody
    D, V_rows, _ = ops.graph_eigs_sparse(sizes, node_ptr, edge_ptr, edges, N, K,
                                         num_edgetype=self.num_edgetype, rows=node_feat.shape[0])
    return self._forward_sparse_impl(N, sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, D)

  def _train_records(self, recs, V_rows=None, D=None):
    # records without eigenpairs get them from lnb_graph_eigs_sparse, as data (no gradient flows to them)
    from ..train import ell_operator, ritz_stack_train
    if V_rows is None:
      D, V_rows, _ = ops.graph_eigs_sparse(recs.sizes, recs.node_ptr, recs.edge_ptr, recs.edges, recs.N, recs.K,
                                           num_edgetype=self.num_edgetype, rows=recs.node_feat.shape[0])
    prep, x, mask, V, _ = self._prepare_ritz_records(
        recs.sizes, recs.node_ptr, recs.node_feat, recs.edge_ptr, recs.edges, V_rows.float().contiguous(), recs.N)
    return ritz_stack_train(self, *self._ritz_inputs(x), ell_operator(prep), D, V, mask)
