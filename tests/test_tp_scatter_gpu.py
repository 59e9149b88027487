"""GPU parity of the fused TP+scatter kernels against the CPU oracle.

Modelled on the reference's own kernel test
(tests/unit/nn/test_tp_scatter_kernel.py:34-179): same irreps grid,
same N=8 / E=15 random graph, forward plus gradients w.r.t. x, edge_attr and
edge_weight, atol = rtol = 1e-5 (float32) / 1e-10 (float64).  The "base
implementation" it is compared with is oracle.tp (the e3nn formulation restated
on the CPU in float64) instead of e3nn itself.
"""
import pytest
import torch

from nequip_b200 import known_signatures as ks
from nequip_b200 import ops
from nequip_b200.codegen import GenOptions
from nequip_b200.irreps import Irreps
from nequip_b200.nn import B200TensorProductScatter
from oracle import tp as otp

pytestmark = pytest.mark.gpu

NUM_NODES = 8
NUM_EDGES = 15
TOL = {torch.float32: 1e-5, torch.float64: 1e-10}


def _ir_str(irr):
    return "+".join(f"{m}x{ir.l}{'e' if ir.p == 1 else 'o'}" for m, ir in Irreps(irr))


def _oracle(sig, x, y, w, dst, src):
    ins = [(a, b, c, "uvu", True) for a, b, c in sig.instructions]
    return otp.tp_scatter(
        x, y, w, dst, src, _ir_str(sig.irreps_in1), _ir_str(sig.irreps_in2), _ir_str(sig.irreps_out), ins
    )


def _run_case(sig, dtype, N, E, seed=0, sort_edges=False, dst_hi=None, scale_check=True, layout="mul_ir"):
    dev = "cuda"
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, sig.d_in, generator=g, dtype=torch.float64)
    y = torch.randn(E, sig.s_dim, generator=g, dtype=torch.float64)
    w = torch.randn(E, sig.weight_numel, generator=g, dtype=torch.float64)
    src = torch.randint(0, N, (E,), generator=g)
    dst = torch.randint(0, dst_hi or N, (E,), generator=g)
    if sort_edges:
        dst, order = torch.sort(dst, stable=True)
        src = src[order]
    gout = torch.randn(N, sig.d_out, generator=g, dtype=torch.float64)

    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        mod = B200TensorProductScatter(
            sig.irreps_in1, sig.irreps_in2, sig.irreps_out, [(a, b, c, "uvu", True) for a, b, c in sig.instructions],
            layout=layout,
        )
    finally:
        torch.set_default_dtype(prev)
    from nequip_b200.irreps import ir_mul_to_mul_ir, mul_ir_to_ir_mul

    # ir_mul: node features are channel-contiguous; the output layout is defined over irreps_mid.simplify()
    to_k = (lambda t, irr: mul_ir_to_ir_mul(t, irr)) if layout == "ir_mul" else (lambda t, irr: t)
    from_k = (lambda t, irr: ir_mul_to_mul_ir(t, irr)) if layout == "ir_mul" else (lambda t, irr: t)
    out_irr = sig.irreps_out.simplify()

    # oracle (float64, CPU)
    xo, yo, wo = (t.clone().requires_grad_(True) for t in (x, y, w))
    out_o = _oracle(sig, xo, yo, wo, dst, src)
    gxo, gyo, gwo = torch.autograd.grad(out_o, [xo, yo, wo], gout)

    # kernel
    xk = to_k(x, sig.irreps_in1).to(dev, dtype).requires_grad_(True)
    yk, wk = (t.to(dev, dtype).requires_grad_(True) for t in (y, w))
    out_k = mod(xk, yk, wk, dst.to(dev), src.to(dev))
    assert out_k.shape == (N, sig.d_out) and out_k.dtype == dtype
    tol = TOL[dtype]
    torch.testing.assert_close(from_k(out_k.detach().cpu().double(), out_irr), out_o.detach(), atol=tol, rtol=tol)
    gout_k = to_k(gout, out_irr).to(dev, dtype)
    for name, inp, ref in (("x", xk, gxo), ("edge_attr", yk, gyo), ("edge_weight", wk, gwo)):
        (gk,) = torch.autograd.grad(out_k, inp, gout_k, retain_graph=True)
        if name == "x":
            gk = from_k(gk.cpu(), sig.irreps_in1)
        # gradients of sums over E*paths terms: scale tolerance like assert_close does (atol + rtol*|ref|)
        torch.testing.assert_close(gk.cpu().double(), ref, atol=tol * (10 if dtype == torch.float32 else 1), rtol=tol,
                                   msg=lambda m: f"grad wrt {name}: {m}")


_GRID = ks.reference_test_grid()


@pytest.mark.parametrize("layout", ["mul_ir", "ir_mul"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("idx", range(len(_GRID)))
def test_reference_grid(idx, dtype, layout):
    _run_case(_GRID[idx], dtype, NUM_NODES, NUM_EDGES, seed=idx, layout=layout)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("cfg", [(2, 32, 4), (2, 64, 4), (1, 32, 4), (3, 32, 5)], ids=lambda c: f"l{c[0]}f{c[1]}")
def test_model_layer_shapes(cfg, dtype):
    """Every interaction layer of the BASELINE.json model families, on a small sorted graph."""
    lmax, nf, nl = cfg
    for li, sig in enumerate(ks.nequip_layer_signatures(lmax, nf, nl)):
        _run_case(sig, dtype, N=23, E=301, seed=100 + li, sort_edges=True)
        _run_case(sig, dtype, N=23, E=301, seed=100 + li, sort_edges=True, layout="ir_mul")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_edge_cases(dtype):
    sig = ks.nequip_layer_signatures(2, 32, 4)[1]
    # unsorted destinations, many isolated nodes (dst only hits the first 3 rows)
    _run_case(sig, dtype, N=40, E=97, seed=7, dst_hi=3)
    # single node, single edge (self loop)
    _run_case(sig, dtype, N=1, E=1, seed=8)
    # one edge only, two nodes
    _run_case(sig, dtype, N=2, E=1, seed=9)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_empty_graph(dtype):
    sig = ks.nequip_layer_signatures(2, 32, 4)[1]
    mod = B200TensorProductScatter(
        sig.irreps_in1, sig.irreps_in2, sig.irreps_out, [(a, b, c, "uvu", True) for a, b, c in sig.instructions]
    )
    mod.model_dtype = dtype
    x = torch.randn(5, sig.d_in, device="cuda", dtype=dtype, requires_grad=True)
    y = torch.zeros(0, sig.s_dim, device="cuda", dtype=dtype)
    w = torch.zeros(0, sig.weight_numel, device="cuda", dtype=dtype)
    idx = torch.zeros(0, dtype=torch.long, device="cuda")
    out = mod(x, y, w, idx, idx)
    assert out.shape == (5, sig.d_out) and float(out.abs().max()) == 0.0
    (gx,) = torch.autograd.grad(out.sum(), x)
    assert float(gx.abs().max()) == 0.0


def test_deterministic_forward():
    """The forward uses no atomics: bitwise identical across repeated launches."""
    sig = ks.nequip_layer_signatures(2, 32, 4)[2]
    mod = B200TensorProductScatter(
        sig.irreps_in1, sig.irreps_in2, sig.irreps_out, [(a, b, c, "uvu", True) for a, b, c in sig.instructions]
    )
    mod.model_dtype = torch.float32
    g = torch.Generator().manual_seed(3)
    N, E = 64, 3000
    x = torch.randn(N, sig.d_in, generator=g).cuda()
    y = torch.randn(E, sig.s_dim, generator=g).cuda()
    w = torch.randn(E, sig.weight_numel, generator=g).cuda()
    src = torch.randint(0, N, (E,), generator=g).cuda()
    dst = torch.randint(0, N, (E,), generator=g).cuda()
    a = mod(x, y, w, dst, src)
    b = mod(x, y, w, dst, src)
    assert torch.equal(a, b)


def test_cpu_tensors_rejected():
    sig = ks.nequip_layer_signatures(2, 32, 4)[0]
    mod = B200TensorProductScatter(
        sig.irreps_in1, sig.irreps_in2, sig.irreps_out, [(a, b, c, "uvu", True) for a, b, c in sig.instructions]
    )
    x = torch.randn(3, sig.d_in)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        mod(x, torch.randn(2, sig.s_dim), torch.randn(2, sig.weight_numel), torch.tensor([0, 1]), torch.tensor([1, 2]))


@pytest.mark.parametrize("layout", ["mul_ir", "ir_mul"])
def test_deterministic_backward_is_bitwise_repeatable_and_matches_default(layout):
    """ops.set_deterministic(True): grad_x via per-edge rows + source-sorted segmented sum, grad_Y via one slice per
    writer -- bitwise identical from run to run, and equal (to rounding) to the default red.global.add path."""
    from nequip_b200 import known_signatures as ks

    sig = ks.nequip_layer_signatures(2, 32, 4)[2]
    plan = ops.get_plan(sig.irreps_in1, sig.irreps_in2, sig.irreps_out, sig.instructions, GenOptions(layout=layout))
    g = torch.Generator().manual_seed(3)
    N, E = 300, 9000
    x = torch.randn(N, sig.d_in, generator=g).cuda()
    y = torch.randn(E, sig.s_dim, generator=g).cuda()
    w = torch.randn(E, sig.weight_numel, generator=g).cuda()
    dst = torch.sort(torch.randint(0, N, (E,), generator=g)).values.cuda()
    src = torch.randint(0, N, (E,), generator=g).cuda()
    go = torch.randn(N, sig.d_out, generator=g).cuda()
    csr = ops.build_csr(dst, N)
    ref = ops.tp_scatter_bwd_raw(plan, x, y, w, src, csr, go, force_deterministic=False)
    runs = [ops.tp_scatter_bwd_raw(plan, x, y, w, src, csr, go, force_deterministic=True) for _ in range(3)]
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert torch.equal(a, b)
    for a, b in zip(runs[0], ref):
        scale = float(b.abs().max())
        assert float((a - b).abs().max()) <= 2e-5 * scale
    # the default path is generally NOT bitwise repeatable for grad_x (atomic order); it must still agree to rounding
    again = ops.tp_scatter_bwd_raw(plan, x, y, w, src, csr, go, force_deterministic=False)
    assert float((again[0] - ref[0]).abs().max()) <= 2e-5 * float(ref[0].abs().max())
