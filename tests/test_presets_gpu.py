"""GPU: degree-4 harmonics, the TP kernels of every preset layer and the S/M/L/XL models end to end, against the CPU
oracle (oracle.sh / oracle.tp and the per-degree-width restatement in preset_oracle)."""
import math
import warnings

import pytest
import torch

import preset_oracle as po
from nequip_b200 import data as D
from nequip_b200 import known_signatures as ks
from nequip_b200 import ops
from nequip_b200.codegen import GenOptions
from nequip_b200.graph import GraphedEnergyForces
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel
from oracle import sh as osh
from test_tp_scatter_gpu import _run_case

pytestmark = pytest.mark.gpu

PRESETS = ["S", "M", "L", "XL"]


# ------------------------------------------------------------------ l_max = 4 harmonics and edge embedding
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_sh_lmax4_forward_backward(dtype):
    g = torch.Generator().manual_seed(4)
    vec = torch.randn(257, 3, generator=g, dtype=torch.float64) * 2.0
    gy = torch.randn(257, 25, generator=g, dtype=torch.float64)
    v_o = vec.clone().requires_grad_(True)
    y_o = osh.spherical_harmonics(4, v_o)
    (gv_o,) = torch.autograd.grad(y_o, v_o, gy)
    v_k = vec.cuda().requires_grad_(True)
    y_k = ops.spherical_harmonics(v_k, 4, out_dtype=dtype)
    assert y_k.shape == (257, 25) and y_k.dtype == dtype
    tol = 1e-6 if dtype == torch.float32 else 1e-12
    torch.testing.assert_close(y_k.detach().cpu().double(), y_o.detach(), atol=tol, rtol=tol)
    (gv_k,) = torch.autograd.grad(y_k, v_k, gy.cuda().to(dtype))
    torch.testing.assert_close(gv_k.cpu(), gv_o, atol=10 * tol, rtol=10 * tol)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_edge_embed_lmax4(dtype):
    sysd = D.make_system("li3po4", 6, r_max=5.0, seed=1)
    pos, ei, cell, shift = sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"]
    lmax, nb, r_max, p = 4, 8, 5.0, 6.0
    E = ei.shape[1]
    g = torch.Generator().manual_seed(6)
    gy = torch.randn(E, 25, generator=g, dtype=torch.float64)
    gemb = torch.randn(E, nb, generator=g, dtype=torch.float64)
    p_o = pos.clone().requires_grad_(True)
    vec_o, y_o, emb_o = omodel.edge_embed(p_o, ei, cell, shift, lmax, nb, r_max, p, dtype)
    (gp_o,) = torch.autograd.grad([y_o, emb_o], [p_o], [gy.to(dtype), gemb.to(dtype)])
    p_k = pos.cuda().requires_grad_(True)
    vec_k, y_k, emb_k = ops.edge_embed(p_k, ei.cuda(), shift.cuda(), cell.cuda(), lmax=lmax, num_bessel=nb,
                                       r_max=r_max, poly_p=p, prefactor=2 * math.pi / r_max**2, out_dtype=dtype)
    tol = 2e-6 if dtype == torch.float32 else 1e-12
    torch.testing.assert_close(y_k.detach().cpu().double(), y_o.detach().double(), atol=tol, rtol=tol)
    torch.testing.assert_close(emb_k.detach().cpu().double(), emb_o.detach().double(), atol=tol, rtol=tol)
    (gp_k,) = torch.autograd.grad([y_k, emb_k], [p_k], [gy.cuda().to(dtype), gemb.cuda().to(dtype)])
    scale = float(gp_o.abs().max())
    torch.testing.assert_close(gp_k.cpu(), gp_o, atol=(2e-5 if dtype == torch.float32 else 1e-10) * scale, rtol=1e-5)
    # the edge-vector (ML-IAP) entry point: same harmonics, gradient w.r.t. the vectors
    v_o = vec_o.detach().clone().requires_grad_(True)
    y2_o = osh.spherical_harmonics(lmax, v_o).to(dtype)
    (gv_o,) = torch.autograd.grad(y2_o, v_o, gy.to(dtype))
    v_k = vec_o.detach().cuda().requires_grad_(True)
    y2_k, _emb2 = ops.edge_embed_from_vectors(v_k, lmax=lmax, num_bessel=nb, r_max=r_max, poly_p=p,
                                              prefactor=2 * math.pi / r_max**2, out_dtype=dtype)
    torch.testing.assert_close(y2_k.detach().cpu().double(), y2_o.detach().double(), atol=tol, rtol=tol)
    (gv_k,) = torch.autograd.grad(y2_k, v_k, gy.cuda().to(dtype))
    torch.testing.assert_close(gv_k.cpu(), gv_o.double(), atol=(2e-5 if dtype == torch.float32 else 1e-10)
                               * float(gv_o.abs().max()), rtol=1e-5)


# ------------------------------------------------------------------ TP kernels of the preset layers
def _distinct_layer_sigs(name):
    seen, out = set(), []
    for li, s in enumerate(ks.preset_layer_signatures(name)):
        if s.canonical() not in seen:
            seen.add(s.canonical())
            out.append((li, s))
    return out


@pytest.mark.parametrize("layout", ["mul_ir", "ir_mul"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", PRESETS)
def test_preset_layer_tp_matches_oracle(name, dtype, layout):
    """Forward and the gradients w.r.t. x, edge_attr and edge_weight of every distinct layer signature."""
    for li, sig in _distinct_layer_sigs(name):
        _run_case(sig, dtype, N=23, E=301, seed=200 + li, sort_edges=True, layout=layout)
        _run_case(sig, dtype, N=40, E=97, seed=300 + li, dst_hi=3, layout=layout)  # unsorted, isolated nodes
        _run_high_degree(sig, dtype, layout, seed=400 + li)


def _run_high_degree(sig, dtype, layout, seed, N=6, E=700):
    """~350 edges into each of two nodes: the ring kernels stage edge ids in several passes of RING_CAP = 256.  Every
    output element sums ~350 products, so float32 rounding grows with the node degree; as in the model-level checks the
    tolerance is relative to the largest element of each compared tensor (1e-5 in float32, 1e-10 in float64)."""
    from nequip_b200.irreps import ir_mul_to_mul_ir, mul_ir_to_ir_mul
    from nequip_b200.nn import B200TensorProductScatter
    from test_tp_scatter_gpu import _oracle

    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, sig.d_in, generator=g, dtype=torch.float64)
    y = torch.randn(E, sig.s_dim, generator=g, dtype=torch.float64)
    w = torch.randn(E, sig.weight_numel, generator=g, dtype=torch.float64)
    src = torch.randint(0, N, (E,), generator=g)
    dst = torch.randint(0, 2, (E,), generator=g)
    gout = torch.randn(N, sig.d_out, generator=g, dtype=torch.float64)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        mod = B200TensorProductScatter(sig.irreps_in1, sig.irreps_in2, sig.irreps_out,
                                       [(a, b, c, "uvu", True) for a, b, c in sig.instructions], layout=layout)
    finally:
        torch.set_default_dtype(prev)
    ir = layout == "ir_mul"
    out_irr = sig.irreps_out.simplify()
    xo, yo, wo = (t.clone().requires_grad_(True) for t in (x, y, w))
    out_o = _oracle(sig, xo, yo, wo, dst, src)
    refs = [out_o.detach()] + list(torch.autograd.grad(out_o, [xo, yo, wo], gout))
    xk = (mul_ir_to_ir_mul(x, sig.irreps_in1) if ir else x).to("cuda", dtype).requires_grad_(True)
    yk, wk = (t.to("cuda", dtype).requires_grad_(True) for t in (y, w))
    out_k = mod(xk, yk, wk, dst.cuda(), src.cuda())
    gouts = (mul_ir_to_ir_mul(gout, out_irr) if ir else gout).to("cuda", dtype)
    gxk, gyk, gwk = torch.autograd.grad(out_k, [xk, yk, wk], gouts)
    got = [out_k.detach().cpu().double(), gxk.cpu().double(), gyk.cpu().double(), gwk.cpu().double()]
    if ir:
        got[0] = ir_mul_to_mul_ir(got[0], out_irr)
        got[1] = ir_mul_to_mul_ir(got[1], sig.irreps_in1)
    tol = 1e-5 if dtype == torch.float32 else 1e-10
    for name, a, b in zip(("out", "grad_x", "grad_edge_attr", "grad_edge_weight"), got, refs):
        err = float((a - b).abs().max()) / float(b.abs().max())
        assert err <= tol, (name, err)


@pytest.mark.parametrize("layout", ["mul_ir", "ir_mul"])
@pytest.mark.parametrize("name", ["M", "XL"])
def test_deterministic_backward_mixed_multiplicities(name, layout):
    """One grad_Y slice per work item: bitwise repeatable, and equal to rounding to the atomic path."""
    sig = ks.preset_layer_signatures(name)[1]
    plan = ops.get_plan(sig.irreps_in1, sig.irreps_in2, sig.irreps_out, sig.instructions, GenOptions(layout=layout))
    g = torch.Generator().manual_seed(11)
    N, E = 300, 6000
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
        assert float((a - b).abs().max()) <= 2e-5 * float(b.abs().max())


# ------------------------------------------------------------------ models end to end
def _frozen_preset(name, meta, dtype=torch.float32, **kw):
    m = NequIPEnergyModel.from_preset(name, r_max=5.0, type_names=meta["type_names"],
                                      avg_num_neighbors=meta["avg_num_neighbors"], model_dtype=dtype,
                                      strict_fast_path=(dtype == torch.float32), **kw).cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


# atoms per side of the Li3PO4-like box: the CPU oracle of XL (6 layers, 320 + 96 + 64 + 32 + 32 channels) is the slow part
SIDE = {"S": 6, "M": 5, "L": 4, "XL": 4}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", PRESETS)
def test_preset_energy_forces_f32_match_oracle(name):
    """Frozen weights with strict_fast_path: the wgmma dense blocks and float2 TP kernels, 1e-5 relative."""
    sysd = D.make_system("li3po4", SIDE[name], r_max=5.0, seed=3)
    meta = sysd.pop("_meta")
    model = _frozen_preset(name, meta)
    out = model(D.to_device(sysd, "cuda"))
    torch.cuda.synchronize()
    assert all(l.conv._tc_cache is not None and l.conv._tc_cache[1] is not None for l in model.layers)
    e_ref, ea_ref, f_ref = po.energy_and_forces(model.state_dict(), model.config, sysd, torch.float32, tp_chunk=20000)
    ferr = float((out["forces"].cpu() - f_ref).abs().max()) / float(f_ref.abs().max())
    eerr = abs(float(out["total_energy"]) - float(e_ref)) / float(ea_ref.abs().sum())
    print(f"{name} f32: N={sysd['pos'].shape[0]} max|dF|/max|F| = {ferr:.2e}, |dE|/sum|E_i| = {eerr:.2e}")
    assert ferr <= 1e-5 and eerr <= 1e-5


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["M", "XL"])
def test_preset_energy_forces_f64_match_oracle(name):
    sysd = D.make_system("li3po4", 4, r_max=5.0, seed=4)
    meta = sysd.pop("_meta")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # float64 runs the torch dense blocks, by design
        model = _frozen_preset(name, meta, torch.float64)
        out = model(D.to_device(sysd, "cuda"))
    e_ref, ea_ref, f_ref = po.energy_and_forces(model.state_dict(), model.config, sysd, torch.float64, tp_chunk=20000)
    assert abs(float(out["total_energy"]) - float(e_ref)) <= 1e-9 * float(ea_ref.abs().sum())
    assert float((out["forces"].cpu() - f_ref).abs().max()) <= 1e-9 * float(f_ref.abs().max())


def _small_lmax4(meta, dtype):
    """An l_max = 4 model with per-degree widths that keeps the CPU oracle quick."""
    return _frozen_preset("XL", meta, dtype, num_layers=3, num_features=[32, 16, 16, 8, 8], type_embed_num_features=8)


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-9), (torch.float32, 1e-5)])
def test_lmax4_stress_and_virial_match_oracle(dtype, tol):
    sysd = D.make_system("li3po4", 4, r_max=5.0, seed=5)
    meta = sysd.pop("_meta")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = _small_lmax4(meta, dtype)
        out = model(D.to_device(sysd, "cuda"), compute_stress=True)
    e_ref, f_ref, s_ref, v_ref = po.energy_forces_stress(model.state_dict(), model.config, sysd, dtype)
    assert float((out["stress"].cpu() - s_ref).abs().max()) <= tol * float(s_ref.abs().max())
    assert float((out["virial"].cpu() - v_ref).abs().max()) <= tol * float(v_ref.abs().max())
    assert float((out["forces"].cpu() - f_ref).abs().max()) <= tol * float(f_ref.abs().max())


def test_lmax4_edge_force_branch_matches_oracle():
    sysd = D.make_system("li3po4", 4, r_max=5.0, seed=6)
    meta = sysd.pop("_meta")
    model = _small_lmax4(meta, torch.float32)
    vec = omodel.edge_vectors(sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"])
    d = {k: v for k, v in sysd.items() if k not in ("cell", "edge_cell_shift")}
    d["edge_vectors"] = vec
    out = model(D.to_device(d, "cuda"))
    e_ref, g_ref = po.edge_forces(model.state_dict(), model.config, d, torch.float32)
    assert float((out["edge_forces"].cpu() - g_ref).abs().max()) <= 1e-5 * float(g_ref.abs().max())
    assert abs(float(out["total_energy"]) - float(e_ref)) <= 1e-5 * float(out["atomic_energy"].abs().sum())


def test_preset_graph_replay_equals_eager():
    sysd = D.make_system("li3po4", 6, r_max=5.0, seed=7)
    meta = sysd.pop("_meta")
    model = _frozen_preset("M", meta)
    dev = D.to_device(sysd, "cuda")
    eager = model(dev)
    e, f = eager["total_energy"].clone(), eager["forces"].clone()
    graphed = GraphedEnergyForces(model, dev)
    out = graphed(dev)
    graphed.check_sorted()
    # same kernels, same order; only atomics (red.global.add) may reorder
    assert abs(float(out["total_energy"]) - float(e)) <= 1e-9 * abs(float(e)) + 1e-9
    assert float((out["forces"] - f).abs().max()) <= 2e-6 * float(f.abs().max())
