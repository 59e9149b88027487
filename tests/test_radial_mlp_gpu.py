"""GPU parity of the radial MLP on the product path (CUDA-core hidden layer k_hidden_fwd/bwd + grouped
wgmma 3xTF32 GEMM, nequip_b200/nn/dense.py RadialMLPGemm) against the fp64 restatement of
ScalarMLPFunction (nequip/nn/mlp.py:80-195, 262-268)."""
import math

import pytest
import torch

from nequip_b200.nn import dense
from nequip_b200.nn.model import ScalarLinearLayer

pytestmark = pytest.mark.gpu


def _ref(emb, W1, a1, W2, a2):
    h = torch.nn.functional.silu(emb.double() @ (W1.double() * a1))
    return h @ (W2.double() * a2)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("E,W", [(1, 32), (127, 96), (128, 192), (1000, 864), (4099, 1728), (20000, 2176)])
def test_radial_mlp_forward_backward(E, W):
    g = torch.Generator().manual_seed(E + W)
    emb = (torch.rand(E, 8, generator=g) * 2 - 0.7)
    W1 = (torch.rand(8, 128, generator=g) * 2 - 1) * math.sqrt(3)
    W2 = (torch.rand(128, W, generator=g) * 2 - 1) * math.sqrt(3)
    a1, a2 = 1.0 / math.sqrt(8), math.sqrt(2) / math.sqrt(128)
    gw = torch.randn(E, W, generator=g)
    emb_r = emb.clone().double().requires_grad_(True)
    ref = _ref(emb_r, W1, a1, W2, a2)
    (gref,) = torch.autograd.grad(ref, emb_r, gw.double())

    l1, l2 = ScalarLinearLayer(8, 128, a1).cuda(), ScalarLinearLayer(128, W, a2).cuda()
    with torch.no_grad():
        l1.weight.copy_(W1)
        l2.weight.copy_(W2)
    mlp = dense.RadialMLPGemm(l1, l2, "cuda")
    emb_k = emb.cuda().requires_grad_(True)
    out = mlp(emb_k)
    torch.cuda.synchronize()
    err = (out.detach().cpu().double() - ref.detach()).abs().max().item()
    scale = ref.detach().abs().max().item()
    assert err <= 2e-6 * scale + 1e-6, (err, scale)
    (gk,) = torch.autograd.grad(out, emb_k, gw.cuda())
    torch.cuda.synchronize()
    gerr = (gk.cpu().double() - gref).abs().max().item()
    gscale = gref.abs().max().item()
    # segmented accumulation (K = W up to 2176 in 320-wide segments): fp32-GEMM class error
    assert gerr <= 5e-6 * gscale + 1e-6, (gerr, gscale)
