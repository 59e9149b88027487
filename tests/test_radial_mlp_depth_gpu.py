"""Radial MLPs of any depth and width on the project's kernels: the SiLU epilogue of the grouped GEMM
(nqb_gemm_grouped_act), RadialMLPGemm against the float64 restatement of ScalarMLPFunction
(nequip/nn/mlp.py:80-195, 262-268), whole models under strict_fast_path against the oracle, and the graphed MD step."""
import math

import pytest
import torch

import kernel_contracts as kc
from kernel_contracts import Guarded, assert_elementwise
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn import dense
from nequip_b200.nn.model import NequIPEnergyModel, ScalarLinearLayer
from oracle import model as omodel

pytestmark = pytest.mark.gpu

F32 = torch.float32


def _silu(v):
    return v * torch.sigmoid(v)


def _dsilu(p):
    s = torch.sigmoid(p)
    return s * (1 + p * (1 - s))


# ---------------------------------------------------------------------------------------------------------------
# the activation epilogue
# ---------------------------------------------------------------------------------------------------------------
# (M, K, N, a_off, lda, c_off, ldc): M around the 128-row tile and 0, N below one tile and across two, K resident
# and streamed, offsets and strides
EPI_SHAPES = [
    (1, 8, 4, 0, 8, 0, 4), (127, 8, 64, 0, 8, 0, 64), (129, 64, 128, 0, 64, 0, 128), (300, 36, 132, 8, 56, 12, 164),
    (kc.BIG_M, 128, 128, 0, 128, 0, 128), (1000, 324, 260, 4, 332, 8, 276), (0, 8, 64, 0, 8, 0, 64),
]


def _epilogue_case(mode, M, K, N, a_off, lda, c_off, ldc, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g) / math.sqrt(K) * 2.0
    scale = 0.8
    Afull = torch.full((M, lda), float("nan"))
    Afull[:, a_off:a_off + K] = A
    ga = Guarded(M, lda, F32, body=Afull)
    gc = Guarded(M, ldc, F32)
    v = A.double() @ B.double() * scale
    bv = kc.gemm_bound(A, B, scale)
    if mode == "silu_grad":
        P = torch.randn(M, N, generator=g) * 3.0
        body = kc.poison_value(F32).expand(M, ldc).clone()
        body[:, c_off:c_off + N] = P
        gx = Guarded(M, ldc, F32, body=body)
    else:
        gx = Guarded(M, ldc, F32)
    gg = ops.GroupedGemm([ops.GemmProblem(a_off, lda, c_off, ldc, B, scale=scale, act=mode)], "cuda")
    gg.run(ga.view, gc.view, M, aux=gx.view if mode != "silu" else None)
    torch.cuda.synchronize()
    ga.check_guards("A")
    gc.check_guards("C")
    gx.check_guards("aux")
    C, X = gc.view.cpu(), gx.view.cpu()
    # nothing outside columns [c_off, c_off + N) of either matrix is touched
    for T, what in ((C, "C"), (X, "aux")):
        assert bool(kc.is_poison(T[:, :c_off]).all()) and bool(kc.is_poison(T[:, c_off + N:]).all()), what
    Cs = C[:, c_off:c_off + N]
    if mode == "silu_grad":
        p = P.double()
        ref = v * _dsilu(p)
        # silu' is at most 1.1; the SFU sigmoid (ex2 / rcp approx) adds a few fp32 ulps per factor
        bound = 1.1 * bv + 2e-6 * v.abs() * (1 + p.abs()) + 2.0 ** -22 * ref.abs()
        assert_elementwise(Cs, ref, bound, f"silu_grad {(M, K, N)}")
        assert torch.equal(X[:, c_off:c_off + N].view(torch.int32), P.view(torch.int32)), "aux is an input here"
        return
    ref = _silu(v)
    bound = 1.1 * bv + 2e-6 * ref.abs() + 1e-30
    assert_elementwise(Cs, ref, bound, f"{mode} {(M, K, N)}")
    if mode == "silu_save":
        assert_elementwise(X[:, c_off:c_off + N], v, bv + 2.0 ** -23 * v.abs(), f"saved pre-activation {(M, K, N)}")
    else:
        assert bool(kc.is_poison(X).all()), "silu without save wrote aux"


@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode", ["silu", "silu_save", "silu_grad"])
@pytest.mark.parametrize("shape", EPI_SHAPES, ids=lambda s: "M%d_K%d_N%d" % s[:3])
def test_activation_epilogue_write_contract(mode, shape):
    """C (and aux with silu_save) fully written in rows < M, columns < N; with silu_grad aux is read only; guards
    intact; values within the GEMM bound carried through the activation."""
    M, K, N, a_off, lda, c_off, ldc = shape
    _epilogue_case(mode, M, K, N, a_off, lda, c_off, ldc, seed=M * 3 + K + N)


def test_activation_launch_needs_aux_and_keeps_plain_launches_plain():
    g = torch.Generator().manual_seed(2)
    B = torch.randn(8, 64, generator=g)
    a = torch.randn(10, 8, generator=g).cuda()
    c = torch.empty(10, 64, device="cuda")
    for mode in ("silu_save", "silu_grad"):
        gg = ops.GroupedGemm([ops.GemmProblem(0, 8, 0, 64, B, act=mode)], "cuda")
        with pytest.raises(ValueError, match="need aux"):
            gg.run(a, c, 10)
        # the C entry point: a null aux is an error, and nothing is launched
        n0 = _capi.launch_count()
        rc = _capi.lib().nqb_gemm_grouped_act(ops._ptr(gg.descs), gg.ndesc, gg.ntiles_total, None, 0, ops._ptr(a),
                                              ops._ptr(gg.prepared), ops._ptr(c), None, 0, 10, None, ops._stream())
        assert rc != 0 and b"aux_base is null" in _capi.lib().nqb_last_error()
        assert _capi.launch_count() == n0
    plain = ops.GroupedGemm([ops.GemmProblem(0, 8, 0, 64, B)], "cuda")
    with pytest.raises(ValueError, match="no problem sets an activation"):
        plain.run(a, c, 10, aux=torch.empty_like(c))


# ---------------------------------------------------------------------------------------------------------------
# RadialMLPGemm, any depth and width
# ---------------------------------------------------------------------------------------------------------------
def _mlp_layers(depth, width, W, seed, nb=8):
    g = torch.Generator().manual_seed(seed)
    dims = [nb] + [width] * depth + [W]
    lins = []
    for i, (a, b) in enumerate(zip(dims, dims[1:])):
        lin = ScalarLinearLayer(a, b, (1.0 if i == 0 else math.sqrt(2)) / math.sqrt(a))
        with torch.no_grad():
            lin.weight.copy_((torch.rand(a, b, generator=g) * 2 - 1) * math.sqrt(3))
        lins.append(lin.cuda().requires_grad_(False))
    return lins


def _mlp_ref(emb, lins):
    x = emb.double()
    for i, lin in enumerate(lins):
        x = x @ (lin.weight.double().cpu() * float(lin.alpha))
        if i + 1 < len(lins):
            x = _silu(x)
    return x


@pytest.mark.timeout(600)
@pytest.mark.parametrize("E", [1, 127, 4099, 20000])
@pytest.mark.parametrize("width", [8, 64, 128])
@pytest.mark.parametrize("depth", [1, 2, 3])
def test_radial_mlp_any_depth_matches_fp64(depth, width, E):
    W = 96
    lins = _mlp_layers(depth, width, W, seed=depth * 1000 + width + E)
    g = torch.Generator().manual_seed(E)
    emb = torch.rand(E, 8, generator=g) * 2 - 0.7
    gw = torch.randn(E, W, generator=g)
    emb_r = emb.clone().double().requires_grad_(True)
    ref = _mlp_ref(emb_r, lins)
    (gref,) = torch.autograd.grad(ref, emb_r, gw.double())
    mlp = dense.RadialMLPGemm(lins[0], lins[-1], "cuda", middle=lins[1:-1])
    emb_k = emb.cuda().requires_grad_(True)
    out = mlp(emb_k)
    (gk,) = torch.autograd.grad(out, emb_k, gw.cuda())
    torch.cuda.synchronize()
    err = (out.detach().cpu().double() - ref.detach()).abs().max().item()
    scale = ref.detach().abs().max().item()
    assert err <= 4e-6 * scale + 1e-6, (err, scale)
    gerr = (gk.cpu().double() - gref).abs().max().item()
    gscale = gref.abs().max().item()
    assert gerr <= 1e-5 * gscale + 1e-6, (gerr, gscale)
    # without a gradient: the "silu" launches, no pre-activations, the same values
    with torch.no_grad():
        out2 = mlp(emb_k)
    assert torch.equal(out2, out.detach())


# ---------------------------------------------------------------------------------------------------------------
# whole models under strict_fast_path
# ---------------------------------------------------------------------------------------------------------------
MODELS = {
    # the reference tutorial (configs/tutorial.yaml: radial 2 x 64)
    "tutorial_l1": ("water", 6, dict(l_max=1, num_layers=4, num_features=32, radial_mlp_depth=2, radial_mlp_width=64)),
    # the Li3PO4 frame's model family with a radial 3 x 128 MLP
    "li3po4_l2_r3x128": ("li3po4", 6, dict(l_max=2, num_layers=4, num_features=64, radial_mlp_depth=3,
                                            radial_mlp_width=128)),
    # the reference's unit-test shape (radial 1 x 8)
    "ref_test_r1x8": ("water", 5, dict(l_max=1, num_layers=3, num_features=32, radial_mlp_depth=1, radial_mlp_width=8)),
}


def _model(name, seed=0):
    kind, n_side, cfg = MODELS[name]
    sysd = D.make_system(kind, n_side, r_max=5.0, seed=seed)
    meta = sysd.pop("_meta")
    model = NequIPEnergyModel(r_max=5.0, type_names=meta["type_names"], parity=True,
                              avg_num_neighbors=meta["avg_num_neighbors"], strict_fast_path=True, **cfg).cuda()
    for p in model.parameters():
        p.requires_grad_(False)
    return model, sysd


def _assert_oracle(out, ref, what):
    e_ref, ea_ref, f_ref = ref
    e, f = out["total_energy"].cpu(), out["forces"].cpu()
    assert abs(float(e) - float(e_ref)) <= 1e-5 * float(ea_ref.abs().sum()), (what, float(e), float(e_ref))
    fscale = float(f_ref.abs().max())
    assert float((f - f_ref).abs().max()) <= 1e-5 * fscale, (what, float((f - f_ref).abs().max()) / fscale)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", list(MODELS))
def test_model_any_radial_depth_strict_fast_path_matches_oracle(name):
    model, sysd = _model(name)
    dev = D.to_device(sysd, "cuda")
    ref = omodel.energy_and_forces(model.state_dict(), model.config, sysd, torch.float32)
    n0 = _capi.launch_count()
    out = model(dev)
    torch.cuda.synchronize()
    assert all(l.conv._tc_cache is not None and l.conv._tc_cache[1] is not None for l in model.layers)
    assert all(l.conv._tc_cache[1]["mlp"] is not None for l in model.layers), "radial MLP not on the GEMM path"
    assert _capi.launch_count() - n0 >= 4 * len(model.layers)
    _assert_oracle(out, ref, "auto")
    # both sides of the per-layer fused / unfused choice, whichever the timing picked
    fusable = [l.conv for l in model.layers if l.conv._tc_cache[1]["fused"] is not None]
    for mode in (True, False):
        for conv in fusable:
            conv.use_fused_radial_tp = mode
        _assert_oracle(model(dev), ref, f"use_fused_radial_tp={mode}")
    # energy only: the "silu" launches without saved pre-activations
    e_only = model(dev, compute_forces=False)["total_energy"]
    assert abs(float(e_only) - float(ref[0])) <= 1e-5 * float(ref[1].abs().sum())


@pytest.mark.timeout(900)
def test_graphed_md_step_tutorial_model():
    model, sysd = _model("tutorial_l1")
    dev = D.to_device(sysd, "cuda")
    pos0 = dev["pos"].clone()
    g = GraphedMDStep(model, dev)
    for t in range(12):
        pos = D.oscillating_positions(pos0, t, period=50, seed=5)
        out = {k: v.clone() for k, v in g(pos).items()}
        nl = ops.neighbor_list(pos, dev["cell"], True, 5.0)
        ref = model(dict(dev, pos=pos, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))
        assert int(out["num_edges"]) == nl["edge_index"].shape[1]
        e_ref = float(ref["total_energy"])
        assert abs(float(out["total_energy"]) - e_ref) <= 1e-9 * abs(e_ref) + 1e-6, (t, float(out["total_energy"]), e_ref)
        fs = float(ref["forces"].abs().max())
        assert float((out["forces"] - ref["forces"]).abs().max()) <= 2e-6 * fs, t
    n0 = _capi.launch_count()
    g(D.oscillating_positions(pos0, 3, period=50, seed=5))
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0, "a replay launched nequip_b200 kernels eagerly"
