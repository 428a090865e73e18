"""GAT drop-in on the GPU: lnb_gat_attention across its envelope against fp64, the module against the
reference's outputs (tests/golden/gat_qm8.npz) and the fp64 oracle at the benchmark batch size, CUDA-graph
replay, weight updates and nn.DataParallel.  ``pytest -m gpu``."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import GAT
from oracle import gat_oracle

pytestmark = pytest.mark.gpu

FWD_ATOL = 2e-5
FWD_RTOL = 1e-4
SMALL = dict(num_layer=2, num_heads=[3, 3], hidden_dim=[8, 8], output_dim=5)


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _spec(cfg):
  return gat_oracle.make_spec(cfg.model.num_layer, cfg.model.num_heads, cfg.dataset.num_bond_type)


def _build(cfg, seed):
  mod = GAT(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()).eval(), params


# ------------------------------------------------------------------------------------------------
def attention_reference(Wh, bias, a1, a2, c1, c2, sb, last, dtype):
  """The formula of lnb_gat_attention in plain torch at ``dtype`` (all channels at once)."""
  B, N, _ = Wh.shape
  C, Fd = a1.shape
  E1 = bias.shape[3]
  W = Wh.to(dtype).view(B, N, C, Fd)
  s1 = torch.einsum('bncf,cf->bnc', W, a1.to(dtype)) + c1.to(dtype)
  s2 = torch.einsum('bncf,cf->bnc', W, a2.to(dtype)) + c2.to(dtype)
  chan = torch.arange(C, device=Wh.device) // (C // E1)
  e = F.leaky_relu(s1[:, :, None, :] + s2[:, None, :, :], 0.2) + bias.to(dtype)[..., chan]
  att = torch.softmax(e, dim=1)                                       # over the row index i
  h = torch.einsum('bikc,bkcf->bicf', att, W) + sb.to(dtype)
  return h.mean(dim=2) if last else F.elu(h).reshape(B, N, C * Fd)


def _attention_inputs(gen, B, N, Fd, heads, E1, kind):
  C = E1 * heads
  r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
  Wh = r(B, N, C * Fd)
  a1, a2 = r(C, Fd) / np.sqrt(Fd), r(C, Fd) / np.sqrt(Fd)
  c1, c2, sb = 0.1 * r(C), 0.1 * r(C), 0.1 * r(C, Fd)
  if kind == 'mask':                       # the collate's bias: -0.0 on edges and self-loops, -1e9 else
    adj = (torch.rand(B, N, N, E1, generator=gen) < 0.3).double()
    bias = torch.from_numpy(data.gat_bias((adj + adj.transpose(1, 2)).numpy()))
  else:                                    # arbitrary finite biases: the softmax works for real
    bias = (2.0 * r(B, N, N, E1)).float()
  f32 = [t.float().to(dev()) for t in (Wh, a1, a2, c1, c2, sb)]
  return [f32[0], bias.to(dev())] + f32[1:]


SWEEP = list(itertools.product([1, 2, 7, 26, 64, 128], [4, 16, 32, 64], [1, 3, 8], [1, 7]))


def test_attention_kernel_against_fp64_across_the_envelope():
  gen = torch.Generator().manual_seed(0)
  worst = 0.0
  for N, Fd, heads, E1 in SWEEP:
    for kind in ('mask', 'finite'):
      args = _attention_inputs(gen, 2, N, Fd, heads, E1, kind)
      for last in (False, True):
        got = ops.gat_attention(*args, last=last)
        r64 = attention_reference(*args, last, torch.float64)
        r32 = attention_reference(*args, last, torch.float32)
        scale = max(1.0, float(r64.abs().max()))
        e_ours = float((got.double() - r64).abs().max())
        e_orc = float((r32.double() - r64).abs().max())
        # 4x the fp32 oracle's own distance from fp64, floor 2e-6 of the output scale
        assert e_ours <= max(4 * e_orc, 2e-6 * scale), (N, Fd, heads, E1, kind, last, e_ours, e_orc)
        worst = max(worst, e_ours / scale)
        assert torch.equal(got, ops.gat_attention(*args, last=last))   # fixed order: bit-identical
  print('worst scaled error %.3g over %d shapes' % (worst, 4 * len(SWEEP)))


def test_attention_kernel_refuses_shapes_outside_the_envelope():
  gen = torch.Generator().manual_seed(1)
  for N, Fd, heads, E1 in ((129, 4, 1, 1), (8, 6, 1, 1), (8, 132, 1, 1), (8, 4, 1, 17), (8, 4, 33, 1)):
    args = _attention_inputs(gen, 1, N, Fd, heads, E1, 'finite')
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match='status -2'):
      ops.gat_attention(*args)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    assert not ops.gat_attention_supported(N, Fd, E1, heads)


# ------------------------------------------------------------------------------------------------
def test_model_matches_reference_golden():
  gg = load_golden('gat_qm8.npz')
  nf, L, mask = _t(gg['node_feat']).to(dev()), _t(gg['L']).to(dev()), _t(gg['node_mask']).to(dev())
  cases = [(configs.qm8_gat(), int(gg['weight_seed']), 'score', 'score_nomask'),
           (configs.qm8_gat(**SMALL), int(gg['weight_seed']) + 1, 'score_small', 'score_small_nomask')]
  for cfg, seed, k_mask, k_nomask in cases:
    mod, params = _build(cfg, seed)
    with torch.no_grad():
      if k_mask == 'score':
        score, loss = mod(nf, L, label=_t(gg['label']).to(dev()), mask=mask)
      else:
        score = mod(nf, L, mask=mask)
      nomask = mod(nf, L)
    for got, key, m in ((score, k_mask, gg['node_mask']), (nomask, k_nomask, None)):
      np.testing.assert_allclose(got.cpu().numpy(), gg[key], rtol=FWD_RTOL, atol=FWD_ATOL)
      s64 = gat_oracle.gat_forward(params, _spec(cfg), gg['node_feat'], gg['L'], m, dtype=torch.float64).numpy()
      e_ref = np.abs(gg[key] - s64).max()
      e_ours = np.abs(got.cpu().numpy() - s64).max()
      assert e_ours <= max(4 * e_ref, 5e-6), (key, e_ours, e_ref)
    if k_mask == 'score':
      assert abs(float(loss) - float(gg['loss'])) <= 1e-4 * abs(float(gg['loss']))


def test_bench_batch_against_fp64_oracle_graph_replay_and_updates():
  batch = data.synthetic_qm8_batch(1024, seed=5)
  cfg = configs.qm8_gat()
  mod, params = _build(cfg, 77)
  nf, mask = _t(batch['node_feat']).to(dev()), _t(batch['node_mask']).to(dev())
  L = _t(data.gat_bias(batch['L'])).to(dev())
  with torch.no_grad():
    mod.use_cuda_graph = False
    eager = mod(nf, L, mask=mask)
    mod.use_cuda_graph = True
    replays = [mod(nf, L, mask=mask) for _ in range(3)]
  assert all(torch.equal(eager, r) for r in replays)
  s64 = gat_oracle.gat_forward(params, _spec(cfg), batch['node_feat'], L, batch['node_mask'],
                               dtype=torch.float64, device=dev())
  s32 = gat_oracle.gat_forward(params, _spec(cfg), batch['node_feat'], L, batch['node_mask'], device=dev())
  e_ours = float((eager.double() - s64).abs().max())
  e_orc = float((s32.double() - s64).abs().max())
  np.testing.assert_allclose(eager.cpu().numpy(), s64.cpu().numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)
  assert e_ours <= max(4 * e_orc, 5e-6), (e_ours, e_orc)
  # an optimizer step updates the parameters in place: the captured graph is not reused stale
  opt = torch.optim.SGD(mod.parameters(), lr=0.5)
  for p in mod.parameters():
    p.grad = torch.full_like(p, 0.01)
  with torch.no_grad():
    opt.step()
    updated = mod(nf, L, mask=mask)
    mod.use_cuda_graph = False
    updated_eager = mod(nf, L, mask=mask)
  assert not torch.equal(updated, eager) and torch.equal(updated, updated_eager)
  new_params = {k: v.detach() for k, v in mod.state_dict().items()}
  u64 = gat_oracle.gat_forward(new_params, _spec(cfg), batch['node_feat'], L, batch['node_mask'],
                               dtype=torch.float64, device=dev())
  np.testing.assert_allclose(updated.cpu().numpy(), u64.cpu().numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)


def test_data_parallel_two_replicas_on_one_gpu():
  gg = load_golden('gat_qm8.npz')
  mod, _ = _build(configs.qm8_gat(), 3)
  nf, L, mask = _t(gg['node_feat']).to(dev()), _t(gg['L']).to(dev()), _t(gg['node_mask']).to(dev())
  label = _t(gg['label']).to(dev())
  with torch.no_grad():
    ref = mod(nf, L, mask=mask)
    dp = torch.nn.DataParallel(mod, device_ids=[0, 0]).eval()
    score, loss = dp(nf, L, label=label, mask=mask)
  assert loss.numel() == 2
  torch.testing.assert_close(score, ref, rtol=1e-5, atol=1e-6)
