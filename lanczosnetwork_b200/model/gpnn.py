"""Drop-in for the reference ``model.GPNN`` (model/gpnn.py:10-251): Graph Partition Neural Networks on the
bond channels.  Same constructor fields, parameter names, registration and initialisation order (so
``torch.manual_seed(s)`` gives the reference's initial weights and its checkpoints load by name), and the
same ``forward(node_feat, L, L_cluster, L_cut, label=None, mask=None)``.

A propagation step of the reference (model/gpnn.py:215-230) runs num_prop_cluster GRU steps of the
channel-0 messages over the cluster operator and num_prop_cut over the cut operator, both from the same
state, then ``state_func`` on [state | state_cluster | state_cut] and one GGNN step over the binarised L.
Here a step at the default counts (1 / 1) is eight launches:
  * ``msg_func[0]`` as two ``linear_tf32x3`` (the messages both partition chains start from);
  * ``lnb_gpnn_partition_update``: both chains in one 3xTF32 wgmma launch whose producer warps aggregate
    the messages over the VALUED partition operators (L4 Laplacians, row-normalised for ``avg``) and whose
    epilogue is the GRU cell; it writes the two results into column blocks 1 and 2 of the [B*N, 3H] input
    of ``state_func`` and copies the state into block 0, so the concatenation never runs as a pass;
  * ``state_func`` as two ``linear_tf32x3``;
  * the GGNN step of model.ggnn (stacked first message layers, grouped second layers, lnb_ggnn_update).
Unequal counts run the extra iterations of the longer chain as one-part launches.  With the embedding
gather, ``input_func``, two ``graph_prepare`` (one binarising L, one keeping the partition operators'
values) and the readout, the whole forward is captured as one CUDA graph.  The operators are read,
never modified.

Differences from the reference, on purpose:
  * the reference binarises the caller's ``L`` in place (``L[L != 0] = 1``, :158); this module leaves it
    unchanged (the GGNN step reads only its non-zero pattern); ``L_cluster`` and ``L_cut`` are used with
    their values, as in the reference;
  * ``update_func: MLP`` builds the same parameters as the reference, and the forward raises the
    reference's ``TypeError`` (nn.Sequential called with two arguments, :210) before touching the device;
  * the GRU gate pre-activations are one dot product over [messages | h] plus b_ih + b_hh;
  * ``L_cluster`` and ``L_cut`` may be left out (``None``, or both empty ``[B,0,0]`` tensors): the module
    then partitions every graph on the device (ops.spectral_partition, the collate's spectral clustering
    with ``num_partition`` clusters) inside its captured forward; on the training path the operators are
    constants, as the collate's are.
``update_func: RNN`` (relu RNNCell), shapes outside the kernels and ``input_dim % 4 != 0`` run the
training formulation of lanczosnetwork_b200.train under no_grad."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase, init_cell, init_linears, loss_function
from .ggnn import MSG_HIDDEN, cached_gates, embed_input, ggnn_step, ggnn_step_params
from .. import ops

__all__ = ['GPNN']

STATE_HIDDEN = 512                             # width of state_func, fixed in the reference (:68-72)


class GPNN(SpectralNetBase):

  def __init__(self, config):
    super(GPNN, self).__init__()
    m = config.model
    self._setup_fields(config, config.dataset.num_bond_type)
    self.num_prop = m.num_prop
    self.num_partition = m.num_partition
    self.num_prop_cluster = m.num_prop_cluster
    self.num_prop_cut = m.num_prop_cut
    self.aggregate_type = m.aggregate_type
    self.update_func_name = m.update_func
    assert self.num_layer == 1, "not implemented"
    assert self.aggregate_type in ['avg', 'sum'], 'not implemented'
    E1, D = self.num_edgetype + 1, self.hidden_dim

    self.embedding = nn.Embedding(self.num_atom, self.input_dim)
    if m.update_func == 'RNN':
      self.update_func = nn.RNNCell(input_size=D * E1, hidden_size=D, nonlinearity='relu')
      self.update_func_partition = nn.RNNCell(input_size=D, hidden_size=D, nonlinearity='relu')
    elif m.update_func == 'GRU':
      self.update_func = nn.GRUCell(input_size=D * E1, hidden_size=D)
      self.update_func_partition = nn.GRUCell(input_size=D, hidden_size=D)
    elif m.update_func == 'MLP':              # registered as in the reference; its forward raises
      self.update_func = nn.Sequential(nn.Linear(D * E1, D), nn.Tanh())
      self.update_func_partition = nn.Sequential(nn.Linear(D, D), nn.Tanh())
    self.state_func = nn.Sequential(nn.Linear(3 * D, STATE_HIDDEN), nn.ReLU(), nn.Linear(STATE_HIDDEN, D))
    if m.msg_func == 'MLP':
      self.msg_func = nn.ModuleList([
          nn.Sequential(nn.Linear(D, MSG_HIDDEN), nn.ReLU(), nn.Linear(MSG_HIDDEN, D)) for _ in range(E1)])
    else:
      self.msg_func = None
    self.att_func = nn.Sequential(nn.Linear(D, 1), nn.Sigmoid())
    self.input_func = nn.Sequential(nn.Linear(self.input_dim, D))
    self.output_func = nn.Sequential(nn.Linear(D, self.output_dim))
    self.loss_func = loss_function(m.loss)
    self._init_param()

  def _init_param(self):
    """The reference's order (model/gpnn.py:107-139): Xavier / zero bias for input_func, state_func,
    att_func and output_func (msg_func is a ModuleList, neither Sequential nor Linear, so it keeps PyTorch's
    default initialisation); then, per cell (update_func, update_func_partition), Xavier on weight_hh,
    weight_ih and zero biases (``if m.bias:`` is true).  The MLP update keeps PyTorch's default: the
    reference only re-initialises it when it is a Linear, and it is a Sequential."""
    init_linears([*self.input_func, *self.state_func, *self.att_func, *self.output_func])
    if self.update_func_name in ('GRU', 'RNN'):
      init_cell(self.update_func)
      init_cell(self.update_func_partition)

  def _param_device(self):
    return self.embedding.weight.device

  def forward(self, node_feat, L, L_cluster=None, L_cut=None, label=None, mask=None):
    """
      node_feat: long B x N (atom ids); L: float B x N x N x (E+1) operators (only their non-zero
      pattern is read; L is not modified); L_cluster, L_cut: float B x N x N partition operators (their
      values are read), or both None / empty (B x 0 x 0): partitioned on the device from channel 0 of L;
      label: B x P; mask: B x N (uint8 / bool / float).
      Returns score (B x P) or (score, loss).
    """
    self._check_runnable()
    absent = [t is None or t.numel() == 0 for t in (L_cluster, L_cut)]
    if any(absent):
      if not all(absent):
        raise ValueError('GPNN.forward: pass both L_cluster and L_cut, or neither (device partition)')
      L_cluster = L_cut = None
    return self._forward((node_feat, L, L_cluster, L_cut, mask), label)

  def _check_runnable(self, N=None, E1=None):
    """The reference's errors of the configs its forward cannot run, and (sparse batches, N given) the
    partition's envelope, before any launch."""
    if self.update_func_name == 'MLP':
      raise TypeError("forward() takes 2 positional arguments but 3 were given: update_func 'MLP' is an "
                      "nn.Sequential, which the reference calls with (messages, state) (model/gpnn.py:210)")
    if self.msg_func is None:
      raise UnboundLocalError("msg_func %r: the reference's propagation reads a message that is never "
                              "assigned (model/gpnn.py:193-200); only 'MLP' runs" % self.config.model.msg_func)
    if N is not None and not ops.spectral_partition_supported(N, self.num_partition):
      raise ValueError('GPNN.forward_sparse: N=%d, num_partition=%d outside the device partition\'s envelope'
                       % (N, self.num_partition))

  def _device_partition(self, L):
    """(L_cluster, L_cut) of the collate's spectral clustering, computed on the device."""
    _, L_cluster, L_cut, _ = ops.spectral_partition(L, self.num_partition)
    return L_cluster, L_cut

  def _train_impl(self, node_feat, L, L_cluster, L_cut, mask):
    from ..train import gpnn_train
    if L_cluster is None:
      with torch.no_grad():                    # constants, as the collate's operators are
        L_cluster, L_cut = self._device_partition(L)
    return gpnn_train(self, node_feat, L, L_cluster, L_cut, mask)

  def fused_supported(self, N, E1):
    """True when inference runs the kernel path (GRU update, the shapes of lnb_ggnn_update and
    lnb_gpnn_partition_update, an input width the dense kernel reads)."""
    return (self.update_func_name == 'GRU' and self.input_dim % 4 == 0 and
            self.update_func.weight_ih.shape[1] == E1 * self.hidden_dim and
            ops.ggnn_update_supported(N, self.hidden_dim, E1) and
            ops.gpnn_partition_update_supported(N, self.hidden_dim))

  def _partition_params(self):
    """Splits of msg_func[0], the partition gate matrix and state_func, once per parameter version."""
    cache = self._wcache
    msg = [(cache.split('msg_func.0.%d' % i, self.msg_func[0][i].weight), self.msg_func[0][i].bias) for i in (0, 2)]
    state = [(cache.split('state_func.%d' % i, self.state_func[i].weight), self.state_func[i].bias) for i in (0, 2)]
    return msg, cached_gates(cache, 'update_func_partition.gates', self.update_func_partition), state

  @staticmethod
  def _dense(x, layer, relu=False):
    (w_hi, w_lo), bias = layer
    return ops.linear_tf32x3(x, w_hi, w_lo, bias, relu=relu)

  def _partition(self, h, X, T, pprep, msg, gates, avg):
    """Both partition chains from the state h [B*N, H]; their results land in column blocks 1 (cluster)
    and 2 (cut) of X [B*N, 3H], the state in block 0.  Iteration j of a chain with c iterations writes to
    X when c - 1 - j is even and to the scratch T otherwise, so the last one lands in X and no launch
    reads the buffer it writes."""
    H = h.shape[1]
    counts = (self.num_prop_cluster, self.num_prop_cut)
    block = lambda buf, p: buf[:, (p + 1) * H:(p + 2) * H]
    cur = [h, h]
    shared = None
    for j in range(max(counts)):
      parts = []
      for p in (0, 1):
        if j >= counts[p]:
          parts.append(None)
          continue
        if j == 0:                      # both chains start from the same state: the same messages
          if shared is None:
            shared = self._dense(self._dense(h, msg[0], relu=True), msg[1])
          M = shared
        else:
          M = self._dense(self._dense(cur[p], msg[0], relu=True), msg[1])
        parts.append((M, cur[p], block(X if (counts[p] - 1 - j) % 2 == 0 else T, p)))
      ops.gpnn_partition_update(parts, pprep, gates[0], gates[1], gates[2], avg,
                                h_copy=X[:, :H] if j == 0 else None)
      cur = [pt[2] if pt is not None else c for pt, c in zip(parts, cur)]
    if max(counts) == 0:
      X[:, :H].copy_(h)
    for p in (0, 1):
      if counts[p] == 0:                # a chain without iterations is the state itself
        block(X, p).copy_(h)

  def _forward_impl(self, node_feat, L, L_cluster, L_cut, mask):
    B, N = node_feat.shape
    E1 = L.shape[3]
    if not self.fused_supported(N, E1):
      return self._train_impl(node_feat, L, L_cluster, L_cut, mask)   # RNN update / other shapes
    if L_cluster is None:
      L_cluster, L_cut = self._device_partition(L)
    # ELL rows of the 0/1 operators and of the valued partition operators; no Ritz vectors, one zero
    # block for both
    zeros = torch.zeros((B, N, 4), device=L.device, dtype=torch.float32)
    prep = ops.graph_prepare(L, zeros, binarize=True)
    pprep = ops.graph_prepare(torch.stack([L_cluster, L_cut], 3), zeros)
    return self._propagate(node_feat, prep, pprep, mask)

  def _forward_records(self, recs):
    # the partition's ELL rows come straight from lnb_spectral_partition_sparse
    fused = self.fused_supported(recs.N, self.num_edgetype + 1)
    prep, node_ids, mask, _, L = self._prepare_records(recs, binarize=True, want_dense=not fused)
    if not fused:
      return self._train_impl(node_ids, L, None, None, mask)
    _, _, pprep, _, _ = ops.spectral_partition_sparse(recs.sizes, recs.edge_ptr, recs.edges, recs.N,
                                                      self.num_partition, self.num_edgetype)
    return self._propagate(node_ids, prep, pprep, mask)

  def _train_records(self, recs):
    # the partition operators are constants, as on the padded path: their ELL rows straight from
    # lnb_spectral_partition_sparse
    from ..train import ell_operator, gpnn_train
    prep, node_ids, mask, _, _ = self._prepare_records(recs, binarize=True)
    _, _, pprep, _, _ = ops.spectral_partition_sparse(recs.sizes, recs.edge_ptr, recs.edges, recs.N,
                                                      self.num_partition, self.num_edgetype)
    return gpnn_train(self, node_ids, ell_operator(prep), ell_operator(pprep), None, mask)

  def _propagate(self, node_feat, prep, pprep, mask):
    """The fused inference forward from the binarised ELL rows of L and those of [L_cluster, L_cut]."""
    B, N = node_feat.shape
    H = self.hidden_dim
    h = embed_input(self, node_feat, self.embedding.weight)
    step = ggnn_step_params(self._wcache, self.msg_func, self.update_func)
    msg, gates, state = self._partition_params()
    X = torch.empty((B * N, 3 * H), device=h.device, dtype=torch.float32)
    T = torch.empty_like(X) if max(self.num_prop_cluster, self.num_prop_cut) > 1 else None
    spare = torch.empty_like(h)
    avg = self.aggregate_type == 'avg'
    for _ in range(self.num_prop):
      self._partition(h, X, T, pprep, msg, gates, avg)
      s = self._dense(self._dense(X, state[0], relu=True), state[1])
      h, spare = ggnn_step(s, prep, step, avg, out=spare), h
    head, att = self.output_func[0], self.att_func[0]
    return ops.readout(h.view(B, N, H), head.weight, head.bias, att.weight.reshape(-1), att.bias, mask)
