"""The convolution-stack kernel's two-deep rings and the Z it keeps in the A ring, against fp64.

Step 0 of a layer leaves Z (Ritz rows x H) in the A ring; the consumers read it back for V Z before
the edge step's first MMA, and only then may the producers write that step's first k-block.  The
cases below fill the ring with Z (128 Ritz rows x H = 128), run enough tiles that every CTA moves
to a second tile (ring phases, W prefetch and the readout scratch in the A ring cross tiles), and
cover Din0 != H, H < 128, K = 32 and S = 0.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from test_gpu_conv_envelope import STACK_FLOOR_PER_LAYER, _check, _graphs, _weights, stack_ref

pytestmark = pytest.mark.gpu

CASES = [
    # name, N, graph size (None: random), dins, H, S, K, E1, P
    ('ztot128-rtot128', 32, 32, [64, 128, 128], 128, 8, 32, 3, 16),
    ('din0-ne-h', 26, None, [96, 64, 64], 64, 5, 32, 7, 12),
    ('s0', 32, 32, [128, 96, 96], 96, 0, 32, 7, 8),
]


@pytest.mark.parametrize('name,N,size,dins,H,S,K,E1,P', CASES, ids=[c[0] for c in CASES])
def test_stack_kept_z_and_rings_across_tiles(name, N, size, dins, H, S, K, E1, P):
  from lanczosnetwork_b200 import ops
  from lanczosnetwork_b200 import spectral_conv as sc
  d = torch.device('cuda:0')
  sms = torch.cuda.get_device_properties(d).multi_processor_count
  nl = len(dins)
  B = 8 * sms + 8
  seed = 4242 + H + S
  L, V, _ = _graphs(B, N, K, E1, seed, sizes=None if size is None else [size] * B, empty=(5,))
  g = torch.Generator().manual_seed(seed)
  Ws, bs = [], []
  for din in dins:
    (w,), (b,) = _weights(g, H, (S + E1) * din)
    Ws.append(w)
    bs.append(b)
  X0 = torch.randn(B, N, dins[0], generator=g)
  coeffs = torch.randn(nl, B, K, S, generator=g) if S else None
  ro = [torch.randn(P, H, generator=g) / np.sqrt(H), torch.randn(P, generator=g),
        torch.randn(H, generator=g) / np.sqrt(H), torch.randn(1, generator=g)]
  mask = (torch.arange(N)[None, :] < torch.randint(1, N + 1, (B, 1), generator=g)).to(torch.uint8)
  for din in dins:
    assert ops.fused_conv_supported(N, din, K, H, 0, False, S, E1)
  Lg, Vg, Xg, mg = L.to(d), V.to(d), X0.to(d), mask.to(d)
  Wg, bg = [w.to(d) for w in Ws], [b.to(d) for b in bs]
  cg = coeffs.to(d) if S else None
  rog = [t.to(d) for t in ro]
  w_hi, w_lo, ball = sc.WeightCache().split_conv_stack('t', Wg, bg, (S + E1) * max(dins))
  prep = ops.graph_prepare(Lg, Vg)
  gext, tiles = prep[3].cpu(), prep[4].cpu()
  T = int(tiles[B + 2])                        # tiles the kernel runs (the schedule)
  assert T > sms, T                            # at least one CTA runs a second tile
  if size == 32:                               # four graphs per tile: 128 node rows, 128 Ritz rows
    assert int(gext[:4, 0].sum()) == 128 and int(gext[:4, 1].sum()) == 128
  st, score = ops.spectral_stack_forward(prep, Vg, w_hi, w_lo, ball, dins, H, S, X=Xg, coeff=cg,
                                         coeff_stride=cg.stride(0) if S else 0, want_state=True,
                                         readout=rog, mask=mg)
  # repeated launches are bit-identical
  st2, score2 = ops.spectral_stack_forward(prep, Vg, w_hi, w_lo, ball, dins, H, S, X=Xg, coeff=cg,
                                           coeff_stride=cg.stride(0) if S else 0, want_state=True,
                                           readout=rog, mask=mg)
  assert torch.equal(st, st2) and torch.equal(score, score2)
  st64, sc64 = stack_ref(Xg.double(), Lg.double(), Vg.double(), None if cg is None else cg.double(),
                         [w.double() for w in Wg], [b.double() for b in bg], [t.double() for t in rog], mg)
  torch.backends.cuda.matmul.allow_tf32 = False
  st32, sc32 = stack_ref(Xg, Lg, Vg, cg, Wg, bg, rog, mg)
  _check(st, st64, st32, STACK_FLOOR_PER_LAYER * nl, name + ' state')
  _check(score, sc64, sc32, STACK_FLOOR_PER_LAYER * nl, name + ' score')
