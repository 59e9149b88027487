"""The radial-MLP hidden-layer kernels (nequip_b200/csrc/nqb_mlp.cu: batches of 32 edges per warp with prefetched
basis values, float2 arithmetic, four-edge gradient reduction) against the fp64 restatement of
``silu(emb @ W1 a1)`` and its gradient (nequip/nn/mlp.py:262-268), including edge counts that are not multiples of
32 or 4."""
import math

import pytest
import torch

from nequip_b200 import ops

pytestmark = pytest.mark.gpu


def _run(emb, w1s, gh):
    E = emb.shape[0]
    h = torch.full((E, 128), float("nan"), device="cuda")
    gemb = torch.full((E, 8), float("nan"), device="cuda")
    ops.mlp_hidden_fwd(emb, w1s, h)
    ops.mlp_hidden_bwd(emb, w1s, gh, gemb)
    torch.cuda.synchronize()
    return h, gemb


@pytest.mark.parametrize("E", [1, 3, 4, 5, 31, 32, 33, 63, 100, 257, 4099, 50001])
def test_hidden_layer_matches_fp64(E):
    g = torch.Generator().manual_seed(E)
    emb = (torch.rand(E, 8, generator=g) * 2 - 0.7).cuda()
    w1s = ((torch.rand(8, 128, generator=g) * 2 - 1) * math.sqrt(3) / math.sqrt(8)).cuda()
    gh = torch.randn(E, 128, generator=g).cuda()
    h, gemb = _run(emb, w1s, gh)
    e64 = emb.double().requires_grad_(True)
    h64 = torch.nn.functional.silu(e64 @ w1s.double())
    (g64,) = torch.autograd.grad(h64, e64, gh.double())
    hs, gs = float(h64.abs().max()), float(g64.abs().max())
    assert torch.isfinite(h).all() and torch.isfinite(gemb).all()  # every element written (buffers start as NaN)
    assert float((h.double() - h64).abs().max()) <= 1e-6 * hs
    assert float((gemb.double() - g64).abs().max()) <= 3e-6 * gs


def test_hidden_extreme_preactivations():
    """|p| up to ~100: ex2.approx overflows to inf for very negative p and rcp(inf) = 0 must give silu = -0, not NaN."""
    emb = torch.tensor([[40.0] * 8, [-40.0] * 8, [0.0] * 8, [1e-3] * 8], device="cuda")
    w1s = torch.full((8, 128), 0.35, device="cuda")
    gh = torch.ones(4, 128, device="cuda")
    h, gemb = _run(emb, w1s, gh)
    e64 = emb.double().requires_grad_(True)
    h64 = torch.nn.functional.silu(e64 @ w1s.double())
    (g64,) = torch.autograd.grad(h64, e64, gh.double())
    assert torch.isfinite(h).all() and torch.isfinite(gemb).all()
    assert float((h.double() - h64).abs().max()) <= 1e-6 * float(h64.abs().max())
    assert float((gemb.double() - g64).abs().max()) <= 3e-6 * float(g64.abs().max())
