"""Module-level parity: the drop-in nn.Modules against reference outputs (tests/golden) and
the CPU oracle, plus size-independent properties at the benchmark size.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden, oracle_spec
from lanczosnetwork_b200 import configs, data
from lanczosnetwork_b200.model import (AdaLanczosNet, ChebyNet, DCNN, GCN, GCNFP, LanczosNet,
                                       LanczosNetGeneral)
from oracle import lanczos_oracle as orc

pytestmark = pytest.mark.gpu

# Stated fp32 tolerance of the full 7-layer forward (scores are O(0.1..1)):
FWD_ATOL = 2e-5
FWD_RTOL = 1e-4


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _build(cls, cfg, seed):
  mod = cls(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()).eval(), params


def test_lanczosnet_matches_reference_golden():
  g = load_golden('lanczosnet_qm8.npz')
  mod, params = _build(LanczosNet, configs.qm8_lanczos_net(), int(g['weight_seed']))
  with torch.no_grad():
    score, loss = mod(_t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['D']).to(dev()),
                      _t(g['V']).to(dev()), label=_t(g['label']).to(dev()),
                      mask=_t(g['node_mask']).to(dev()))
  np.testing.assert_allclose(score.cpu().numpy(), g['score'], rtol=FWD_RTOL, atol=FWD_ATOL)
  assert abs(float(loss) - float(g['loss'])) <= 1e-4 * abs(float(g['loss']))
  # error budget: no further from the fp64 oracle than 4x the reference's own fp32 error
  spec = oracle_spec(mod, 'LanczosNet')
  s64 = orc.lanczos_net_forward(params, spec, g['node_feat'], g['L'], g['D'], g['V'],
                                g['node_mask'], dtype=torch.float64).numpy()
  e_ref = np.abs(g['score'] - s64).max()
  e_ours = np.abs(score.cpu().numpy() - s64).max()
  assert e_ours <= max(4 * e_ref, 5e-6), (e_ours, e_ref)


def test_lanczosnet_power_filter_matches_reference_golden():
  g = load_golden('lanczosnet_qm8.npz')
  cfg = configs.qm8_lanczos_net(spectral_filter_kind='power', num_layer=2, hidden_dim=[32, 32])
  mod, _ = _build(LanczosNet, cfg, int(g['weight_seed']) + 100)
  with torch.no_grad():
    score = mod(_t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['D']).to(dev()),
                _t(g['V']).to(dev()), mask=_t(g['node_mask']).to(dev()))
  np.testing.assert_allclose(score.cpu().numpy(), g['score_power'], rtol=FWD_RTOL, atol=FWD_ATOL)


def test_general_matches_reference_golden():
  g = load_golden('lanczosnet_general_synth.npz')
  mod, _ = _build(LanczosNetGeneral, configs.graph_lanczos_net(), int(g['weight_seed']))
  with torch.no_grad():
    score = mod(_t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['D']).to(dev()),
                _t(g['V']).to(dev()), mask=_t(g['node_mask']).to(dev()))
  np.testing.assert_allclose(score.cpu().numpy(), g['score'], rtol=FWD_RTOL, atol=FWD_ATOL)


def test_ada_matches_reference_golden():
  g = load_golden('ada_forward_small.npz')
  cfg = configs.qm8_ada_lanczos_net(num_layer=2, hidden_dim=[32, 32], num_eig_vec=8,
                                    long_diffusion_dist=[2, 5], short_diffusion_dist=[1, 3])
  mod, _ = _build(AdaLanczosNet, cfg, int(g['weight_seed']))
  torch.manual_seed(int(g['torch_seed']))     # the module draws q1 like the reference (CPU randn)
  with torch.no_grad():
    score = mod(_t(g['node_feat']).to(dev()), _t(g['L']).to(dev()),
                mask=_t(g['node_mask']).to(dev()))
  np.testing.assert_allclose(score.cpu().numpy(), g['score'], rtol=1e-3, atol=5e-5)


def test_lanczosnet_vs_oracle_batch256_and_properties():
  """Benchmark-shaped batch against the fp32 oracle, then size-independent properties:
  batch-permutation equivariance (bit-exact), invariance to extra zero padding."""
  batch = data.synthetic_qm8_batch(256, seed=99)
  mod, params = _build(LanczosNet, configs.qm8_lanczos_net(), 1234)
  spec = oracle_spec(mod, 'LanczosNet')
  args = [batch[k] for k in ('node_feat', 'L', 'D', 'V')]
  ref = orc.lanczos_net_forward(params, spec, *args, batch['node_mask']).numpy()
  dargs = [_t(a).to(dev()) for a in args]
  mask = _t(batch['node_mask']).to(dev())
  with torch.no_grad():
    out = mod(*dargs, mask=mask)
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=FWD_RTOL, atol=FWD_ATOL)
    perm = torch.randperm(256, generator=torch.Generator().manual_seed(1)).to(dev())
    outp = mod(*[a[perm] for a in dargs], mask=mask[perm])
    assert torch.equal(outp, out[perm])
    # pad every graph with 6 extra empty nodes: same scores
    B, N = dargs[0].shape
    nf = torch.zeros(B, N + 6, dtype=dargs[0].dtype, device=dev()); nf[:, :N] = dargs[0]
    Lp = torch.zeros(B, N + 6, N + 6, 7, device=dev()); Lp[:, :N, :N] = dargs[1]
    Vp = torch.zeros(B, N + 6, 20, device=dev()); Vp[:, :N] = dargs[3]
    mp = torch.zeros(B, N + 6, dtype=torch.uint8, device=dev()); mp[:, :N] = mask
    outpad = mod(nf, Lp, dargs[2], Vp, mask=mp)
    np.testing.assert_allclose(outpad.cpu().numpy(), out.cpu().numpy(), rtol=1e-5, atol=2e-6)


def test_dropin_surface_and_checkpoint_compat(tmp_path):
  """Same state_dict keys / shapes as the reference (keys recorded from the reference class),
  DataParallel wrapping, CPU inputs moved by the module, label -> (score, loss)."""
  g = load_golden('lanczosnet_qm8.npz')
  cfg = configs.qm8_lanczos_net()
  mod = LanczosNet(cfg)
  keys = list(mod.state_dict().keys())
  assert keys[:2] == ['filter.0.weight', 'filter.0.bias']
  assert 'embedding.weight' in keys and 'att_func.0.weight' in keys
  assert 'spectral_filter.6.6.bias' in keys and len(keys) == 16 + 1 + 56 + 2
  snap = {'model': deterministic_state_dict(mod, 5), 'optimizer': {}, 'step': 0}
  path = str(tmp_path / 'model_snapshot_best.pth')
  torch.save(snap, path)                                   # utils/train_helper.py:14-25 format
  mod.load_state_dict(torch.load(path)['model'])           # utils/train_helper.py:28-32
  wrapped = torch.nn.DataParallel(mod, device_ids=[0]).cuda().eval()   # runner/qm8_runner.py:291-292
  with torch.no_grad():
    score, loss = wrapped(_t(g['node_feat']).cuda(), _t(g['L']), _t(g['D']).cuda(),
                          _t(g['V']).cuda(), label=_t(g['label']).cuda(),
                          mask=_t(g['node_mask']).cuda())
  assert score.shape == (8, 16) and torch.isfinite(score).all() and loss.ndim == 0
  train_score = wrapped.module(_t(g['node_feat']).cuda(), _t(g['L']).cuda(), _t(g['D']).cuda(),
                               _t(g['V']).cuda(), mask=_t(g['node_mask']).cuda())
  assert train_score.requires_grad            # grad enabled -> the differentiable training path
  torch.testing.assert_close(train_score.detach(), score, rtol=1e-4, atol=2e-5)
  ada = AdaLanczosNet(configs.qm8_ada_lanczos_net(num_layer=1, hidden_dim=[32], num_eig_vec=8,
                                                  long_diffusion_dist=[2], short_diffusion_dist=[])).cuda()
  ada_score = ada(_t(g['node_feat']).cuda(), _t(g['L']).cuda(), mask=_t(g['node_mask']).cuda())
  assert ada_score.requires_grad and ada_score.shape == (8, 16)   # every drop-in has a training path
  with pytest.raises(RuntimeError):
    LanczosNet(cfg)(_t(g['node_feat']), _t(g['L']), _t(g['D']), _t(g['V']))   # CPU module: loud


def test_fused_lanczos_ritz_reproduces_low_rank_operator():
  """The north-star pipeline adjacency -> Lanczos -> QL -> Ritz pairs in one lnb_lanczos_ritz launch: for
  graphs with n_b <= K the Ritz decomposition reproduces the operator on the Krylov space."""
  from lanczosnetwork_b200 import ops
  rng = np.random.RandomState(4)
  sizes = [12, 9, 15, 7, 18, 20, 5, 11]
  N, K = 20, 20
  A = np.zeros((len(sizes), N, N), np.float32)
  mask = np.zeros((len(sizes), N), np.uint8)
  for b, n in enumerate(sizes):
    _, adjs = data.synthetic_molecule(rng, n)
    A[b, :n, :n] = data.get_laplacian(adjs.sum(axis=2))
    mask[b, :n] = 1
  q1 = rng.randn(len(sizes), N).astype(np.float32)
  lz = ops.lanczos_ritz(_t(A).to(dev()), _t(mask).to(dev()), _t(q1).to(dev()), K)
  theta, V, status = lz['theta'], lz['V'], lz['status']
  assert int(status.sum()) == 0
  o = orc.lanczos_tridiagonalise(_t(A).double(), _t(mask), _t(q1).double(), K)
  assert np.array_equal(lz['idx'].cpu().numpy(), o['idx'].numpy())
  th, S, Vo = orc.tridiag_ritz(o['alpha'].numpy(), o['beta'].numpy()[:, :K - 1], o['Q'].numpy())
  ours = np.einsum('bnk,bk,bmk->bnm', V.cpu().numpy().astype(np.float64),
                   theta.cpu().numpy().astype(np.float64), V.cpu().numpy().astype(np.float64))
  ref = np.einsum('bnk,bk,bmk->bnm', Vo, th, Vo)
  np.testing.assert_allclose(ours, ref, atol=5e-5)


def test_gcn_matches_reference_golden():
  """SURVEY 8(f3): model/gcn.py through the same one-launch stack kernel (no long scales)."""
  g, gg = load_golden('lanczosnet_qm8.npz'), load_golden('gcn_qm8.npz')
  mod, params = _build(GCN, configs.qm8_gcn(), int(gg['weight_seed']))
  nf, L = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev())
  with torch.no_grad():
    n0 = ops_launches()
    score, loss = mod(nf, L, label=_t(g['label']).to(dev()), mask=_t(g['node_mask']).to(dev()))
    nomask = mod(nf, L)
  np.testing.assert_allclose(score.cpu().numpy(), gg['score'], rtol=FWD_RTOL, atol=FWD_ATOL)
  np.testing.assert_allclose(nomask.cpu().numpy(), gg['score_nomask'], rtol=FWD_RTOL, atol=FWD_ATOL)
  assert abs(float(loss) - float(gg['loss'])) <= 1e-4 * abs(float(gg['loss']))
  spec = oracle_spec(mod, 'GCN')
  s64 = orc.gcn_forward(params, spec, g['node_feat'], g['L'], g['node_mask'], dtype=torch.float64).numpy()
  e_ref = np.abs(gg['score'] - s64).max()
  e_ours = np.abs(score.cpu().numpy() - s64).max()
  # unnormalised hidden states (no spectral part) are O(10): 3xTF32 leaves ~1e-5 of the 0.77 output
  # scale, inside FWD_ATOL; budget stated against the fp64 oracle
  assert e_ours <= max(4 * e_ref, 1.5e-5), (e_ours, e_ref)
  assert ops_launches() > n0
  # GCNFP: operators binarised inside lnb_graph_prepare; the caller's L stays untouched
  mod_fp, params_fp = _build(GCNFP, configs.qm8_gcn(name='GCNFP'), int(gg['weight_seed']) + 1)
  L_before = L.clone()
  with torch.no_grad():
    fp = mod_fp(nf, L, mask=_t(g['node_mask']).to(dev()))
  assert torch.equal(L, L_before)
  scale = float(np.abs(gg['score_fp']).max())
  np.testing.assert_allclose(fp.cpu().numpy(), gg['score_fp'], rtol=FWD_RTOL, atol=FWD_ATOL * max(1.0, scale))


def test_dcnn_matches_reference_golden():
  """SURVEY 8(f3): model/dcnn.py through the general-shape ops (30-step power chain per layer)."""
  g, gg = load_golden('lanczosnet_qm8.npz'), load_golden('gcn_qm8.npz')
  cfg = configs.qm8_dcnn()
  mod, params = _build(DCNN, cfg, int(gg['weight_seed']) + 2)
  nf, L, mask = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['node_mask']).to(dev())
  with torch.no_grad():
    mod.use_cuda_graph = False
    eager = mod(nf, L, mask=mask)
    mod.use_cuda_graph = True
    replay = [mod(nf, L, mask=mask) for _ in range(3)]
  np.testing.assert_allclose(eager.cpu().numpy(), gg['score_dcnn'], rtol=FWD_RTOL, atol=FWD_ATOL)
  assert all(torch.equal(eager, r) for r in replay)
  s64 = orc.dcnn_forward(params, cfg.model.diffusion_dist, cfg.dataset.num_bond_type,
                         cfg.model.num_layer, g['node_feat'], g['L'], g['node_mask'],
                         dtype=torch.float64).numpy()
  e_ref = np.abs(gg['score_dcnn'] - s64).max()
  e_ours = np.abs(eager.cpu().numpy() - s64).max()
  assert e_ours <= max(4 * e_ref, 1.5e-5), (e_ours, e_ref)


def test_cheby_net_matches_reference_golden():
  """SURVEY 8(f3): model/cheby_net.py; the recurrence runs as alpha / beta-addend batched GEMMs."""
  g, gg = load_golden('lanczosnet_qm8.npz'), load_golden('gcn_qm8.npz')
  cfg = configs.qm8_cheby_net()
  mod, params = _build(ChebyNet, cfg, int(gg['weight_seed']) + 3)
  nf, L, mask = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['node_mask']).to(dev())
  with torch.no_grad():
    mod.use_cuda_graph = False
    eager = mod(nf, L, mask=mask)
    mod.use_cuda_graph = True
    replay = [mod(nf, L, mask=mask) for _ in range(3)]
  np.testing.assert_allclose(eager.cpu().numpy(), gg['score_cheby'], rtol=FWD_RTOL, atol=FWD_ATOL)
  assert all(torch.equal(eager, r) for r in replay)
  s64 = orc.cheby_net_forward(params, cfg.model.polynomial_order, cfg.dataset.num_bond_type,
                              cfg.model.num_layer, g['node_feat'], g['L'], g['node_mask'],
                              dtype=torch.float64).numpy()
  e_ref = np.abs(gg['score_cheby'] - s64).max()
  e_ours = np.abs(eager.cpu().numpy() - s64).max()
  assert e_ours <= max(4 * e_ref, 1.5e-5), (e_ours, e_ref)


def test_sibling_models_large_graphs_use_the_per_step_path():
  """N > 32: the operator chain of DCNN / ChebyNet falls back to one batched GEMM per step."""
  rng = np.random.RandomState(3)
  B, N = 3, 40
  L = (rng.randn(B, N, N, 7) * (rng.rand(B, N, N, 7) < 0.1) / 4).astype(np.float32)
  nf = rng.randint(0, 70, size=(B, N))
  mask = (np.arange(N)[None, :] < np.array([40, 33, 17])[:, None]).astype(np.uint8)
  for cls, cfg, fwd in (
      (DCNN, configs.qm8_dcnn(num_layer=2, hidden_dim=[32, 32], diffusion_dist=[2, 5]),
       lambda p, c: orc.dcnn_forward(p, c.model.diffusion_dist, 6, 2, nf, L, mask)),
      (ChebyNet, configs.qm8_cheby_net(num_layer=2, hidden_dim=[32, 32], polynomial_order=4),
       lambda p, c: orc.cheby_net_forward(p, 4, 6, 2, nf, L, mask))):
    mod, params = _build(cls, cfg, 99)
    with torch.no_grad():
      out = mod(_t(nf).to(dev()), _t(L).to(dev()), mask=_t(mask).to(dev()))
    ref = fwd(params, cfg).numpy()
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=FWD_RTOL, atol=FWD_ATOL * max(1.0, np.abs(ref).max()))


def ops_mod():
  from lanczosnetwork_b200 import ops
  return ops


def ops_launches():
  from lanczosnetwork_b200 import ops
  return ops.launch_count()


def test_cuda_graph_replay_matches_eager_and_tracks_weight_updates():
  g = load_golden('lanczosnet_qm8.npz')
  mod, _ = _build(LanczosNet, configs.qm8_lanczos_net(), int(g['weight_seed']))
  args = [_t(g[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')]
  mask = _t(g['node_mask']).to(dev())
  with torch.no_grad():
    mod.use_cuda_graph = False
    eager = mod(*args, mask=mask)
    mod.use_cuda_graph = True
    first = mod(*args, mask=mask)          # capture (two static-buffer slots)
    replay = mod(*args, mask=mask)         # second sighting of these device buffers: zero-copy graph
    third = mod(*args, mask=mask)          # replay of the zero-copy graph
    assert torch.equal(eager, first) and torch.equal(eager, replay) and torch.equal(eager, third)
    assert len(mod._graphs_resident) == 1
    # new content in the same buffers is picked up by the address-bound graph
    saved = args[1].clone()
    args[1].mul_(0.5)
    changed = mod(*args, mask=mask)
    mod.use_cuda_graph = False
    assert torch.equal(changed, mod(*args, mask=mask)) and not torch.equal(changed, eager)
    mod.use_cuda_graph = True
    args[1].copy_(saved)
    # host (pinned) inputs go straight into the static buffers
    host = [_t(g[k]).pin_memory() for k in ('node_feat', 'L', 'D', 'V')]
    assert torch.equal(mod(*host, mask=_t(g['node_mask']).pin_memory()), eager)
    # an in-place weight update invalidates the captured graph (parameter version changes)
    mod.filter[7].bias.add_(1.0)
    shifted = mod(*args, mask=mask)
    assert not torch.equal(shifted, eager)
    mod.use_cuda_graph = False
    assert torch.equal(mod(*args, mask=mask), shifted)


def test_ada_full_qm8_config_vs_oracle():
  """AdaLanczosNet at the full QM8 config (K=20, 7 layers, 4096-wide learned filter, 351 M
  parameters) against the fp32 CPU oracle on a small batch, same start vector."""
  cfg = configs.qm8_ada_lanczos_net()
  mod = AdaLanczosNet(cfg)
  params = deterministic_state_dict(mod, 2024)
  mod.load_state_dict(params)
  mod = mod.to(dev()).eval()
  batch = data.synthetic_qm8_batch(6, seed=17)
  B, N = batch['node_feat'].shape
  torch.manual_seed(5)
  q1 = torch.randn(B, N, 1)
  spec = oracle_spec(mod, 'AdaLanczosNet')
  ref, aux = orc.ada_lanczos_net_forward(params, spec, batch['node_feat'], batch['L'],
                                         batch['node_mask'], q1[:, :, 0], return_aux=True)
  torch.manual_seed(5)
  mod.use_cuda_graph = False          # eager: last_lanczos then holds this call's tensors
  with torch.no_grad():
    out = mod(_t(batch['node_feat']).to(dev()), _t(batch['L']).to(dev()),
              mask=_t(batch['node_mask']).to(dev()))
    lz = mod.last_lanczos
    torch.manual_seed(5)
    mod.use_cuda_graph = True         # and the captured graph reproduces it bit for bit
    replay = [mod(_t(batch['node_feat']).to(dev()), _t(batch['L']).to(dev()),
                  mask=_t(batch['node_mask']).to(dev())) for _ in range(1)]
    mod.use_cuda_graph = False
  assert torch.equal(replay[0], out)
  assert np.array_equal(lz['idx'].cpu().numpy(), aux['idx'].numpy())
  # the learned Laplacian agrees with the oracle's to summation-order rounding ...
  from lanczosnetwork_b200 import ops
  state = ops.embedding_rows(_t(batch['node_feat']).to(dev()).long(), mod.embedding.weight)
  Le = ops.gaussian_laplacian(state, _t(batch['L']).to(dev()).float().contiguous()).cpu()
  # (entries of Le are <= 1; budget stated against the fp64 oracle: no further from it than 4x the
  # fp32 oracle's own distance, floor 2e-6 -- exp(-d2/sigma2) of 70-term fp32 sums carries ~1e-6
  # of summation-order noise on either side, which is why a direct fp32-vs-fp32 bound of 2e-5 was
  # host-CPU dependent and had been loosened to 1e-4 in round 1)
  adj = orc.adjacency_from_laplacian(_t(batch['L'])[..., 0].double())
  Le64 = orc.gaussian_kernel_laplacian(params['embedding.weight'].double()[_t(batch['node_feat']).long()], adj)
  e_ref = float((aux['Le'].double() - Le64).abs().max())
  e_ours = float((Le.double() - Le64).abs().max())
  assert e_ours <= max(4 * e_ref, 2e-6) and e_ours <= 2e-5, (e_ours, e_ref)
  # ... and the tridiagonalisation is compared on the SAME operator: Lanczos amplifies a 1e-5
  # operator perturbation to 1e-3 in the late coefficients, which made the end-to-end T
  # comparison depend on the host CPU's summation order in the oracle
  lz_ref = orc.lanczos_tridiagonalise(Le, _t(batch['node_mask']), q1[:, :, 0], spec['K'])
  np.testing.assert_allclose(lz['T'].cpu().numpy(), lz_ref['T'].numpy(), atol=5e-5)
  # final scores (O(0.16) here): rtol 5e-4 / atol 5e-5 against the fp32 oracle (round 1: 2e-3 / 2e-4) and a budget
  # against the fp64 oracle -- measured (tools/exp_ada_error.py): |ours - fp64| = 1.2e-6, fp32 oracle 1.4e-7
  np.testing.assert_allclose(out.cpu().numpy(), ref.numpy(), rtol=5e-4, atol=5e-5)
  ref64 = orc.ada_lanczos_net_forward(params, spec, batch['node_feat'], batch['L'], batch['node_mask'],
                                      q1[:, :, 0].double(), dtype=torch.float64).numpy()
  assert np.abs(out.cpu().numpy() - ref64).max() <= 2e-5


def test_lanczosnet_bench_shape_b1024_both_graph_paths():
  """The bench.py workload itself (B=1024 per step, rotating batches, ~140 packed tiles): every one
  of the 1024 x 16 scores of every rotating batch against the fp32 CPU oracle, through BOTH replay
  paths -- the double-buffered static-input graphs fed from pinned host memory (``e2e``) and the
  zero-copy address-bound graphs on resident inputs (``value``)."""
  mod, params = _build(LanczosNet, configs.qm8_lanczos_net(), 1234)
  spec = oracle_spec(mod, 'LanczosNet')
  keys = ('node_feat', 'L', 'D', 'V')
  nb = 3
  host = [data.synthetic_qm8_batch(1024, seed=1000 + i) for i in range(nb)]
  refs = [orc.lanczos_net_forward(params, spec, *[b[k] for k in keys], b['node_mask']).numpy()
          for b in host]
  pinned = [{k: _t(b[k]).pin_memory() for k in keys + ('node_mask',)} for b in host]
  resident = [{k: v.to(dev()) for k, v in p.items()} for p in pinned]
  with torch.no_grad():
    mod.use_cuda_graph = False
    eager = [mod(*[r[k] for k in keys], mask=r['node_mask']) for r in resident]
    mod.use_cuda_graph = True
    for i in range(nb):
      np.testing.assert_allclose(eager[i].cpu().numpy(), refs[i], rtol=FWD_RTOL, atol=FWD_ATOL)
    # pinned host inputs -> alternating static-buffer slots, two rounds
    for rnd in range(2):
      for i in range(nb):
        out = mod(*[pinned[i][k] for k in keys], mask=pinned[i]['node_mask'])
        assert torch.equal(out, eager[i]), (rnd, i)
    # resident inputs: first sighting static-buffer copy, second captures the zero-copy graph,
    # third and fourth replay it
    for rnd in range(4):
      for i in range(nb):
        out = mod(*[resident[i][k] for k in keys], mask=resident[i]['node_mask'])
        assert torch.equal(out, eager[i]), (rnd, i)
        np.testing.assert_allclose(out.cpu().numpy(), refs[i], rtol=FWD_RTOL, atol=FWD_ATOL)
    assert len(mod._graphs_resident) == nb
  prep_tiles = int(mod_tiles(resident[0]))
  assert 120 <= prep_tiles <= 148, prep_tiles      # packed tiles at the bench shape (256 unpacked 32-row slots)


def mod_tiles(r):
  from lanczosnetwork_b200 import ops
  return ops.graph_prepare(r['L'], r['V'])[4][0].item()


def test_non_uniform_hidden_dims_with_poisoned_allocator():
  """ADVICE r1: a fused layer followed by an unfused one (hidden_dim=[64,36,36]: 36 % 32 != 0) must
  write the constant rows of padded nodes, because the unfused layer multiplies every row: recycled
  allocator memory full of NaNs must not reach the scores."""
  g = load_golden('lanczosnet_qm8.npz')
  cfg = configs.qm8_lanczos_net(num_layer=3, hidden_dim=[64, 36, 36])
  mod, params = _build(LanczosNet, cfg, 321)
  spec = oracle_spec(mod, 'LanczosNet')
  ref = orc.lanczos_net_forward(params, spec, g['node_feat'], g['L'], g['D'], g['V'], g['node_mask']).numpy()
  args = [_t(g[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')]
  mask = _t(g['node_mask']).to(dev())
  mod.use_cuda_graph = False
  with torch.no_grad():
    for _ in range(3):
      junk = [torch.full((n,), float('nan'), device=dev()) for n in (8 * 26 * 64, 8 * 26 * 36, 8 * 26 * 128, 1 << 20)]
      del junk                                   # blocks go back to the caching allocator, NaN-filled
      out = mod(*args, mask=mask)
      assert torch.isfinite(out).all()
      np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=FWD_RTOL, atol=FWD_ATOL)


def test_dcnn_unsorted_diffusion_dist_matches_general_path():
  """ADVICE r1: the one-launch operator chain (N <= 32) emits the scales in ascending step order like
  the reference loop (dcnn.py:88-92) for an unsorted config list."""
  g = load_golden('lanczosnet_qm8.npz')
  cfg = configs.qm8_dcnn(num_layer=2, hidden_dim=[32, 32], diffusion_dist=[5, 2])
  mod, params = _build(DCNN, cfg, 17)
  ref = orc.dcnn_forward(params, sorted(cfg.model.diffusion_dist), cfg.dataset.num_bond_type, 2,
                         g['node_feat'], g['L'], g['node_mask']).numpy()
  with torch.no_grad():
    out = mod(_t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), mask=_t(g['node_mask']).to(dev()))
  np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=FWD_RTOL, atol=FWD_ATOL * max(1.0, np.abs(ref).max()))


def test_online_ritz_provider_feeds_lanczosnet():
  """SURVEY 8(f4): adjacency operator -> fused Lanczos+QL kernel -> (D, V) -> LanczosNet.forward.
  For molecules with n_b <= K and (generically) simple spectra the Ritz decomposition equals the
  eigh one as an operator, V theta V^T = V_e D V_e^T, and the scores agree to fp32 rounding of the
  spectral filters; graphs with repeated eigenvalues return fewer pairs (documented model-input
  change) and are only required to give finite scores and exact Ritz values."""
  from lanczosnetwork_b200 import provider
  batch = data.synthetic_qm8_batch(128, seed=21, max_nodes=18)
  t = {k: _t(batch[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V', 'node_mask')}
  th, V, info = provider.online_ritz_pairs(t['L'], t['node_mask'], 20,
                                           generator=torch.Generator(device=dev()).manual_seed(3))
  assert int((info['status'] & 1).sum()) == 0
  n_b = batch['node_mask'].sum(axis=1)
  idx = info['idx'].cpu().numpy()
  assert np.all(idx <= n_b)
  A = batch['L'][..., 0].astype(np.float64)
  th_n, V_n = th.cpu().numpy().astype(np.float64), V.cpu().numpy().astype(np.float64)
  # well-conditioned graphs whose Krylov space is the whole space: exact decomposition (a beta near
  # the 1e-4 acceptance threshold costs orthogonality like eps / beta, see the kernel-level test)
  out = ops_mod().lanczos_ritz(t['L'][..., 0].contiguous(), t['node_mask'], torch.randn(
      128, t['L'].shape[1], device=dev(), generator=torch.Generator(device=dev()).manual_seed(3)), 20,
      want_ritz=False, proper=True)
  beta = out['beta'].cpu().numpy()
  bmin = np.array([beta[b, :max(idx[b] - 1, 1)].min() if idx[b] > 1 else 1.0 for b in range(len(idx))])
  full = (idx == n_b) & (bmin > 1e-2)
  assert full.mean() > 0.4
  rec = np.einsum('bnk,bk,bmk->bnm', V_n, th_n, V_n)
  np.testing.assert_allclose(rec[full], A[full], atol=5e-5)
  for b in np.flatnonzero(full):         # every Ritz value is an eigenvalue of its operator
    lam = np.linalg.eigvalsh(A[b, :n_b[b], :n_b[b]])
    for v in th_n[b, :idx[b]]:
      assert np.abs(lam - v).min() < 5e-5
  mod, _ = _build(LanczosNet, configs.qm8_lanczos_net(), 1234)
  with torch.no_grad():
    s_e = mod(t['node_feat'], t['L'], t['D'], t['V'], mask=t['node_mask'])
    s_r = mod(t['node_feat'], t['L'], th, V, mask=t['node_mask'])
  assert torch.isfinite(s_r).all()
  fb = torch.from_numpy(full).to(dev())
  np.testing.assert_allclose(s_r[fb].cpu().numpy(), s_e[fb].cpu().numpy(), rtol=2e-3, atol=2e-4)


def _sparse_tensors(sp, device=None, pin=False):
  out = {}
  for k, v in sp.items():
    if isinstance(v, np.ndarray):
      t = torch.from_numpy(v)
      if pin:
        t = t.pin_memory()
      out[k] = t.to(device) if device is not None else t
    else:
      out[k] = v
  return out


def test_graph_prepare_sparse_is_bit_identical_to_collate_plus_prepare():
  """SURVEY 8(f2): GPU-side batch construction.  From bond lists + node ids + Ritz rows the device
  builds (a) the reference's padded tensors -- node_feat, node_mask, V and, on request, the dense
  L4 operators of every channel -- bit for bit what data.collate (itself bit-exact vs the reference
  loader, tests/test_host_logic.py) produces on the host, and (b) every output of lnb_graph_prepare
  run on that dense tensor: ELL values / indices / row maxima, extents, tile table, Ritz row list."""
  from lanczosnetwork_b200 import ops
  rng = np.random.RandomState(5)
  samples = data.synthetic_qm8_samples(200, seed=77)
  # hand-made corner cases: single atom, two atoms doubly bonded in two channels (multiplicity 2 in the
  # simple graph), a duplicate bond record, an isolated atom next to a bonded pair
  def mol(n, bonds):
    adjs = np.zeros((n, n, 6))
    for u, v, c in bonds:
      adjs[u, v, c] = adjs[v, u, c] = 1.0
    return data.prepare_graph(adjs, rng.randint(0, 70, size=n), label=rng.randn(1, 16))
  samples += [mol(1, []), mol(2, [(0, 1, 0), (0, 1, 3)]), mol(3, [(0, 1, 2)]), mol(5, [(0, 4, 5), (1, 2, 5), (2, 3, 0)])]
  dup = mol(4, [(0, 1, 1), (1, 2, 1)])
  dup['edges'] = np.concatenate([dup['edges'], dup['edges'][:1]], axis=0)      # same bond listed twice
  samples.append(dup)
  dense = data.collate(samples, 20)
  sp = _sparse_tensors(data.sparse_collate(samples, 20), dev())
  B, N = dense['node_feat'].shape
  prep_s, ids, mask, V, L = ops.graph_prepare_sparse(sp['sizes'], sp['node_ptr'], sp['node_feat'],
                                                     sp['edge_ptr'], sp['edges'], sp['V_rows'], N, 7,
                                                     want_dense=True)
  assert torch.equal(ids.cpu(), _t(dense['node_feat']))
  assert torch.equal(mask.cpu(), _t(dense['node_mask']))
  assert torch.equal(V.cpu(), _t(dense['V']))
  assert torch.equal(L.cpu(), _t(dense['L']))                 # values: identical bits, not 1 ulp
  prep_d = ops.graph_prepare(_t(dense['L']).to(dev()), _t(dense['V']).to(dev()))
  assert torch.equal(prep_s[2], prep_d[2]) and torch.equal(prep_s[3], prep_d[3])       # ell_max, gext
  T = int(prep_d[4][0])
  assert torch.equal(prep_s[4][:T + 2], prep_d[4][:T + 2])                              # tile table
  nr = int(prep_d.nrows)
  assert int(prep_s.nrows) == nr and torch.equal(prep_s.rowmap[:nr], prep_d.rowmap[:nr])
  emax = prep_d[2].cpu().numpy()
  vs, vd = prep_s[0].cpu().numpy(), prep_d[0].cpu().numpy()
  js, jd = prep_s[1].cpu().numpy(), prep_d[1].cpu().numpy()
  for b in range(B):
    for e in range(7):
      m = emax[b, e]
      assert np.array_equal(vs[b, e, :m], vd[b, e, :m]) and np.array_equal(js[b, e, :m], jd[b, e, :m])
  # packed batch: one buffer, tile table and Ritz-row offsets computed on the HOST with the same rule
  spn = data.sparse_collate(samples, 20)
  pk = data.pack_sparse(spn)
  prep_p, ids_p, mask_p, V_p, L_p = ops.graph_prepare_sparse_packed(_t(pk['blob']).to(dev()), B, N, 7, 20,
                                                                    want_dense=True)
  assert torch.equal(ids_p, ids) and torch.equal(mask_p, mask) and torch.equal(V_p, V) and torch.equal(L_p, L)
  assert torch.equal(prep_p[2], prep_d[2]) and torch.equal(prep_p[3], prep_d[3])
  assert torch.equal(prep_p[4][:T + 2], prep_d[4][:T + 2])                       # host tiles == device tiles
  assert int(prep_p.nrows) == nr and torch.equal(prep_p.rowmap[:nr], prep_d.rowmap[:nr])
  vp, jp = prep_p[0].cpu().numpy(), prep_p[1].cpu().numpy()
  for b in range(0, B, 7):
    for e in range(7):
      m = emax[b, e]
      assert np.array_equal(vp[b, e, :m], vd[b, e, :m]) and np.array_equal(jp[b, e, :m], jd[b, e, :m])
  # GCNFP's binarisation flag
  pb_s = ops.graph_prepare_sparse(sp['sizes'], sp['node_ptr'], sp['node_feat'], sp['edge_ptr'],
                                  sp['edges'], sp['V_rows'], N, 7, binarize=True)[0]
  pb_d = ops.graph_prepare(_t(dense['L']).to(dev()), _t(dense['V']).to(dev()), True)
  for b in range(0, B, 17):
    for e in range(7):
      m = emax[b, e]
      assert torch.equal(pb_s[0][b, e, :m], pb_d[0][b, e, :m])


def test_forward_sparse_equals_forward_on_the_collated_batch():
  """LanczosNet.forward_sparse (device-side batch construction, no dense operators anywhere) returns
  the same bits as forward on the reference's padded batch: eager, CUDA-graph replay from pinned host
  records (ragged copies), zero-copy replay on resident records; H2D payload < 1/10 of the dense one."""
  samples = data.synthetic_qm8_samples(300, seed=5)
  dense = data.collate(samples, 20)
  spn = data.sparse_collate(samples, 20)
  mod, params = _build(LanczosNet, configs.qm8_lanczos_net(), 1234)
  spec = oracle_spec(mod, 'LanczosNet')
  ref = orc.lanczos_net_forward(params, spec, dense['node_feat'], dense['L'], dense['D'], dense['V'],
                                dense['node_mask']).numpy()
  args = [_t(dense[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')]
  with torch.no_grad():
    mod.use_cuda_graph = False
    want = mod(*args, mask=_t(dense['node_mask']).to(dev()))
    eager = mod.forward_sparse(_sparse_tensors(spn, dev()))
    assert torch.equal(eager, want)
    np.testing.assert_allclose(eager.cpu().numpy(), ref, rtol=FWD_RTOL, atol=FWD_ATOL)
    mod.use_cuda_graph = True
    host = _sparse_tensors(spn, pin=True)
    for _ in range(3):
      assert torch.equal(mod.forward_sparse(host), want)
    # a second batch of the same B with different sizes goes through the same static buffers
    samples2 = data.synthetic_qm8_samples(300, seed=6)
    d2 = data.collate(samples2, 20)
    want2 = mod(*[_t(d2[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')], mask=_t(d2['node_mask']).to(dev()))
    assert torch.equal(mod.forward_sparse(_sparse_tensors(data.sparse_collate(samples2, 20), pin=True)), want2)
    assert torch.equal(mod.forward_sparse(host), want)
    res = _sparse_tensors(spn, dev())
    for _ in range(3):
      assert torch.equal(mod.forward_sparse(res), want)
    score, loss = mod.forward_sparse(host, label=_t(dense['label']).to(dev()))
    assert torch.equal(score, want) and loss.ndim == 0
    # packed batches: the same records as ONE buffer (one H2D copy per step)
    pk = data.pack_sparse(spn)
    pk2 = data.pack_sparse(data.sparse_collate(samples2, 20))
    hp = dict(pk, blob=_t(pk['blob']).pin_memory())
    hp2 = dict(pk2, blob=_t(pk2['blob']).pin_memory())
    for _ in range(2):
      assert torch.equal(mod.forward_sparse(hp), want)
      assert torch.equal(mod.forward_sparse(hp2), want2)
    rp = dict(pk, blob=_t(pk['blob']).to(dev()))
    for _ in range(3):
      assert torch.equal(mod.forward_sparse(rp), want)
    mod.use_cuda_graph = False
    assert torch.equal(mod.forward_sparse(rp), want)
    mod.use_cuda_graph = True
    assert pk['blob'].nbytes < 1.1 * sum(spn[k].nbytes for k in ('sizes', 'node_ptr', 'node_feat', 'edge_ptr', 'edges', 'V_rows', 'D')) + 512
  h2d_sparse = sum(v.nbytes for v in spn.values() if isinstance(v, np.ndarray) and v.dtype != np.float64) - spn['label'].nbytes
  h2d_dense = sum(dense[k].nbytes for k in ('node_feat', 'L', 'D', 'V', 'node_mask'))
  assert h2d_sparse * 10 < h2d_dense, (h2d_sparse, h2d_dense)


def test_invalidate_caches_after_data_edit_and_graph_stats():
  """An in-place edit through ``p.data`` bumps no version counter: cached tf32 splits and captured
  graphs keep the old weights until ``invalidate_caches()`` (ADVICE r1); the graph cache reports its
  captures / replays so shape thrash is visible."""
  g = load_golden('lanczosnet_qm8.npz')
  mod, _ = _build(LanczosNet, configs.qm8_lanczos_net(), 77)
  args = [_t(g[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')]
  mask = _t(g['node_mask']).to(dev())
  with torch.no_grad():
    a = mod(*args, mask=mask)
    b = mod(*args, mask=mask)
    c = mod(*args, mask=mask)
    st = mod.graph_stats()
    assert st['captures'] == 2 and st['replays'] >= 2 and torch.equal(a, b) and torch.equal(a, c)
    mod.filter[3].weight.data.mul_(0.5)              # silent edit
    mod.invalidate_caches()
    d = mod(*args, mask=mask)
    assert not torch.equal(d, a)
    mod.use_cuda_graph = False
    assert torch.equal(mod(*args, mask=mask), d)


def test_graph_prepare_sparse_random_multigraphs():
  """GPU-side batch construction on adversarial inputs: random multigraphs (several bond types between
  the same pair, self loops, duplicate records, isolated nodes, single-node graphs), N up to 96 and 1
  to 15 bond types -- dense operators bit-identical to the host mirror of the reference's L4
  (utils/data_helper.py:92-116,155-156) and ELL / extents identical to lnb_graph_prepare on them."""
  from lanczosnetwork_b200 import ops
  rng = np.random.RandomState(123)
  for N, E, B in ((40, 3, 24), (96, 1, 9), (17, 15, 31), (128, 2, 4)):
    samples = []
    for b in range(B):
      n = int(rng.randint(1, N + 1)) if b else N
      adjs = np.zeros((n, n, E))
      ne = int(rng.randint(0, 3 * n + 1))
      recs = []
      for _ in range(ne):
        u, v, c = int(rng.randint(n)), int(rng.randint(n)), int(rng.randint(E))
        adjs[u, v, c] = adjs[v, u, c] = 1.0
        recs.append((min(u, v), max(u, v), c))
      rec = data.prepare_graph(adjs, rng.randint(0, 70, size=n), label=rng.randn(1, 4))
      if recs and b % 3 == 0:                      # ship the raw records, duplicates and order included
        rec['edges'] = np.array(recs + recs[:2], np.uint8).reshape(-1, 3)
      samples.append(rec)
    dense = data.collate(samples, 12)
    sp = _sparse_tensors(data.sparse_collate(samples, 12), dev())
    prep_s, ids, mask, V, L = ops.graph_prepare_sparse(sp['sizes'], sp['node_ptr'], sp['node_feat'],
                                                       sp['edge_ptr'], sp['edges'], sp['V_rows'], N, E + 1,
                                                       want_dense=True)
    assert torch.equal(L.cpu(), _t(dense['L'])), (N, E)
    assert torch.equal(mask.cpu(), _t(dense['node_mask'])) and torch.equal(V.cpu(), _t(dense['V']))
    prep_d = ops.graph_prepare(_t(dense['L']).to(dev()), _t(dense['V']).to(dev()))
    assert torch.equal(prep_s[2], prep_d[2]) and torch.equal(prep_s[3], prep_d[3])
    T = int(prep_d[4][0])
    assert torch.equal(prep_s[4][:T + 2], prep_d[4][:T + 2])
    emax = prep_d[2].cpu().numpy()
    vs, vd = prep_s[0].cpu().numpy(), prep_d[0].cpu().numpy()
    js, jd = prep_s[1].cpu().numpy(), prep_d[1].cpu().numpy()
    for b in range(B):
      for e in range(E + 1):
        m = emax[b, e]
        assert np.array_equal(vs[b, e, :m], vd[b, e, :m]) and np.array_equal(js[b, e, :m], jd[b, e, :m])
    pk = data.pack_sparse(data.sparse_collate(samples, 12))
    prep_p = ops.graph_prepare_sparse_packed(_t(pk['blob']).to(dev()), B, N, E + 1, 12)[0]
    assert torch.equal(prep_p[4][:T + 2], prep_d[4][:T + 2]) and torch.equal(prep_p[3], prep_d[3])
