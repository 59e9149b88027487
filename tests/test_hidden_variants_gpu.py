"""The two generations of the radial-MLP hidden-layer kernels (nequip_b200/csrc/nqb_mlp.cu: v1 = one edge per warp
iteration, v2 = batches of 32 edges with prefetched basis values, float2 arithmetic, four-edge gradient
reduction) against each other and against the fp64 restatement of ``silu(emb @ W1 a1)`` and its gradient
(nequip/nn/mlp.py:262-268), including edge counts that are not multiples of 32 or 4."""
import math

import pytest
import torch

from nequip_b200 import ops

pytestmark = pytest.mark.gpu


def _run(variant, emb, w1s, gh):
    prev = ops.mlp_hidden_variant(variant)
    try:
        E = emb.shape[0]
        h = torch.full((E, 128), float("nan"), device="cuda")
        gemb = torch.full((E, 8), float("nan"), device="cuda")
        ops.mlp_hidden_fwd(emb, w1s, h, None)
        ops.mlp_hidden_bwd(emb, w1s, gh, gemb)
        torch.cuda.synchronize()
        return h, gemb
    finally:
        ops.mlp_hidden_variant(prev)


@pytest.mark.parametrize("E", [1, 3, 4, 5, 31, 32, 33, 63, 100, 257, 4099, 50001])
def test_hidden_v2_matches_v1_and_fp64(E):
    g = torch.Generator().manual_seed(E)
    emb = (torch.rand(E, 8, generator=g) * 2 - 0.7).cuda()
    w1s = ((torch.rand(8, 128, generator=g) * 2 - 1) * math.sqrt(3) / math.sqrt(8)).cuda()
    gh = torch.randn(E, 128, generator=g).cuda()
    h1, g1 = _run(1, emb, w1s, gh)
    h2, g2 = _run(2, emb, w1s, gh)
    e64 = emb.double().requires_grad_(True)
    h64 = torch.nn.functional.silu(e64 @ w1s.double())
    (g64,) = torch.autograd.grad(h64, e64, gh.double())
    hs, gs = float(h64.abs().max()), float(g64.abs().max())
    assert torch.isfinite(h2).all() and torch.isfinite(g2).all()  # every element written (buffers start as NaN)
    assert float((h2.double() - h64).abs().max()) <= 1e-6 * hs
    assert float((g2.double() - g64).abs().max()) <= 3e-6 * gs
    assert float((h2 - h1).abs().max()) <= 5e-7 * hs
    assert float((g2 - g1).abs().max()) <= 2e-6 * gs


def test_hidden_extreme_preactivations():
    """|p| up to ~100: ex2.approx overflows to inf for very negative p and rcp(inf) = 0 must give silu = -0, not NaN."""
    emb = torch.tensor([[40.0] * 8, [-40.0] * 8, [0.0] * 8, [1e-3] * 8], device="cuda")
    w1s = torch.full((8, 128), 0.35, device="cuda")
    gh = torch.ones(4, 128, device="cuda")
    h2, g2 = _run(2, emb, w1s, gh)
    e64 = emb.double().requires_grad_(True)
    h64 = torch.nn.functional.silu(e64 @ w1s.double())
    (g64,) = torch.autograd.grad(h64, e64, gh.double())
    assert torch.isfinite(h2).all() and torch.isfinite(g2).all()
    assert float((h2.double() - h64).abs().max()) <= 1e-6 * float(h64.abs().max())
    assert float((g2.double() - g64).abs().max()) <= 3e-6 * float(g64.abs().max())


@pytest.mark.timeout(120)
def test_hidden_variant_timing_is_reported():
    """Not a pass/fail criterion: prints the isolated times of both generations at the bench frame's edge count."""
    E = 588616
    g = torch.Generator().manual_seed(0)
    emb = torch.rand(E, 8, generator=g).cuda()
    w1s = ((torch.rand(8, 128, generator=g) * 2 - 1) * 0.6).cuda()
    gh = torch.randn(E, 128, generator=g).cuda()
    h, gemb = torch.empty(E, 128, device="cuda"), torch.empty(E, 8, device="cuda")
    flush = torch.empty(64 * 1024 * 1024, device="cuda")  # 256 MB > L2

    def t(fn):
        for _ in range(3):
            fn()
        ms = []
        for _ in range(10):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]

    prev = ops.mlp_hidden_variant(0)
    try:
        for v in (1, 2):
            ops.mlp_hidden_variant(v)
            tf = t(lambda: ops.mlp_hidden_fwd(emb, w1s, h, None))
            tb = t(lambda: ops.mlp_hidden_bwd(emb, w1s, gh, gemb))
            print(f"hidden variant {v}: fwd {tf * 1e3:.1f} us  bwd {tb * 1e3:.1f} us  (E = {E}, L2 flushed)")
    finally:
        ops.mlp_hidden_variant(prev)
