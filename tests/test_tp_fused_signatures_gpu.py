"""The fused radial-MLP -> TP -> scatter forward kernel (``nqb_tp_fused_fwd``, DESIGN section 4.7) against float64 on
every signature of tests/test_tp_fused_signatures.py, and the models whose eligible layers only ``"auto"`` used to
reach, with the choice made explicit.

Kernel cases: hidden widths K = 8, 40 and 128 (zero-padded K in the resident W2^T tile, and the full tile).
  * a small graph whose node degrees cross the 64-edge tile (0, 1, 63, 64, 65, 129, 150, isolated nodes first, in the
    middle and last), against the CPU float64 oracle (``oracle.tp``) with ``w = h @ (W2 alpha2)`` in float64;
  * a 3001-node graph, so that every CTA owns a range of several nodes, against the float64 device kernels
    (``ops.tp_scatter``, themselves checked against the oracle in test_tp_scatter_gpu.py).
``out`` and the side output ``w_out`` are written into poisoned, guarded buffers (tests/kernel_contracts.py) and
checked element by element: ``w_out`` under the 3xTF32 GEMM bound, ``out`` to 3e-6 of max |ref| (dropping one path or
taking a neighbouring weight column is an error of the order of max |ref|).  Isolated nodes must be exactly 0, and
``out`` must not depend on whether ``w_out`` is written.
"""
import math

import pytest
import torch

import kernel_contracts as kc
import preset_oracle as po
from kernel_contracts import Guarded, assert_elementwise
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.codegen import TPGenerator, TPSignature
from nequip_b200.graph import GraphedMDStep
from nequip_b200.irreps import mul_ir_to_ir_mul
from nequip_b200.nn import dense
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel
from test_tp_fused_signatures import CASES, IR_MUL
from test_tp_scatter_gpu import _oracle

pytestmark = pytest.mark.gpu

F32, F64 = torch.float32, torch.float64
P = ops._ptr
KS = [8, 40, 128]
SMALL_DEGS = [0, 1, 63, 64, 0, 65, 129, 150, 2, 0]
OUT_TOL = 3e-6


def _large_degs(seed):
    """3001 nodes of degree 0..5, with a few nodes of 64, 65 and 150 edges."""
    g = torch.Generator().manual_seed(seed)
    degs = torch.randint(0, 6, (3001,), generator=g)
    degs[[0, 1000, 1500, 2000, 3000]] = torch.tensor([0, 64, 150, 65, 0])
    return degs.tolist()


def _run_fused(sig, K, degs, seed):
    """One graph through nqb_tp_fused_fwd on guarded buffers, with and without w_out.  Returns the plan, the float64
    inputs x (mul_ir) and y, dst, src, the kernel's out (ir_mul) and the float64 edge weights h @ (W2 alpha2)."""
    plan = ops.get_plan(sig.irreps_in1, sig.irreps_in2, sig.irreps_out, sig.instructions, IR_MUL)
    g = torch.Generator().manual_seed(seed)
    W2 = (torch.rand(K, sig.weight_numel, generator=g) * 2 - 1) * math.sqrt(3)
    a2 = math.sqrt(2) / math.sqrt(K)
    fw = ops.FusedTPWeights(plan, W2.cuda(), a2, "cuda")
    N = len(degs)
    dst = torch.repeat_interleave(torch.arange(N), torch.tensor(degs))
    E = dst.numel()
    src = torch.randint(0, N, (E,), generator=g)
    x = torch.randn(N, sig.d_in, generator=g, dtype=F64)
    y = torch.randn(E, sig.s_dim, generator=g, dtype=F64)
    h = torch.randn(E, K, generator=g).float()
    gx = Guarded(N, sig.d_in, F32, body=mul_ir_to_ir_mul(x, sig.irreps_in1))
    gy = Guarded(E, sig.s_dim, F32, body=y)
    gh = Guarded(E, K, F32, ld=K + 4, body=h)
    row_ptr = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(torch.tensor(degs), 0)])
    grp = Guarded(N + 1, 1, torch.int64, body=row_ptr.view(-1, 1))
    gsrc = Guarded(E, 1, torch.int64, body=src.view(-1, 1))
    gout, gwo, gout2 = Guarded(N, sig.d_out, F32), Guarded(E, sig.weight_numel, F32), Guarded(N, sig.d_out, F32)
    for o, wo in ((gout, P(gwo.view)), (gout2, 0)):
        _capi.check(_capi.lib().nqb_tp_fused_fwd(plan.handle, P(gx.view), P(gy.view), P(gh.view), gh.ld, K,
                                                 P(fw.prepared), P(grp.view), P(gsrc.view), N, E, P(o.view), wo,
                                                 P(fw.cta0_dev), int(fw.nctas), ops._stream()))
    torch.cuda.synchronize()
    for nm, b in (("x", gx), ("y", gy), ("h", gh), ("row_ptr", grp), ("src", gsrc), ("out", gout), ("w_out", gwo),
                  ("out without w_out", gout2)):
        b.check_guards(nm)
    bits = [o.view.contiguous().view(torch.int32) for o in (gout, gout2)]
    assert torch.equal(*bits), "out depends on whether w_out is written"
    iso = torch.tensor(degs) == 0
    assert bool((gout.view[iso.cuda()] == 0).all()), "an isolated node is not exactly 0"
    W2s = (W2.double() * a2).cuda()
    hd = h.cuda()
    w_ref = hd.double() @ W2s
    assert_elementwise(gwo.view, w_ref, 2 * kc.gemm_bound(hd, W2s, ref=w_ref), "w_out")
    return plan, x, y, dst, src, gout.view, w_ref


def _assert_out(out, ref, what):
    assert_elementwise(out, ref, OUT_TOL * max(float(ref.abs().max()), 1e-30), what)
    return float((out.double().cpu() - ref.cpu()).abs().max()) / float(ref.abs().max())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_fused_small_graph_matches_oracle(case, K):
    sig = case.sig
    plan, x, y, dst, src, out, w_ref = _run_fused(sig, K, SMALL_DEGS, seed=K)
    ref = _oracle(sig, x, y, w_ref.cpu(), dst, src)
    err = _assert_out(out, mul_ir_to_ir_mul(ref, sig.irreps_out.simplify()), "out")
    print(f"{case.name} K={K} small: max|err|/max|ref| = {err:.2e}")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_fused_large_graph_matches_f64_kernels(case, K):
    sig = case.sig
    plan, x, y, dst, src, out, w_ref = _run_fused(sig, K, _large_degs(K), seed=1000 + K)
    xd = mul_ir_to_ir_mul(x, sig.irreps_in1).cuda()
    ref = ops.tp_scatter(plan, xd, y.cuda(), w_ref, dst.cuda(), src.cuda(), csr=ops.build_csr(dst.cuda(), xd.shape[0]))
    err = _assert_out(out, ref, "out")
    print(f"{case.name} K={K} large: max|err|/max|ref| = {err:.2e}")


# ------------------------------------------------------------------ models with the choice made explicit
MODELS = [
    # (name, system, constructor arguments or None for a preset): the models whose eligible layers no other test forces
    ("l1_f128", "li3po4", dict(l_max=1, num_layers=4, num_features=128)),
    ("l2_f128", "li3po4", dict(l_max=2, num_layers=4, num_features=128)),
    ("l2_f64_noparity", "water", dict(l_max=2, num_layers=4, num_features=64, parity=False)),
    ("S", "li3po4", None),
    ("M", "li3po4", None),
    ("L", "li3po4", None),
]
R_MAX = 5.0


def _model(name, mk, meta):
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
              strict_fast_path=True)
    m = (NequIPEnergyModel(radial_mlp_depth=1, radial_mlp_width=128, **kw, **mk) if mk
         else NequIPEnergyModel.from_preset(name, **kw)).cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _eligible(model):
    return [TPGenerator(TPSignature(l.conv.feature_irreps_in, l.conv.irreps_edge_attr, l.conv.irreps_mid,
                                    l.conv.instructions), IR_MUL).fused_layout() is not None for l in model.layers]


def _set_mode(model, modes):
    for l, m in zip(model.layers, modes):
        l.conv.use_fused_radial_tp = m


@pytest.fixture
def fused_calls(monkeypatch):
    """ids of the FusedRadialTP blocks whose kernel ran (returned a result) since the fixture was set up."""
    ran = set()
    orig = dense.FusedRadialTP.__call__

    def call(self, *a, **k):
        r = orig(self, *a, **k)
        if r is not None:
            ran.add(id(self))
        return r

    monkeypatch.setattr(dense.FusedRadialTP, "__call__", call)
    return ran


def _ran_on(model, ran):
    blocks = [l.conv._tc_cache[1] if l.conv._tc_cache is not None else None for l in model.layers]
    return [b is not None and b["fused"] is not None and id(b["fused"]) in ran for b in blocks]


def _outputs(model, dev):
    out = model(dev)
    torch.cuda.synchronize()
    return {k: out[k].detach().clone() for k in ("total_energy", "atomic_energy", "forces")}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name,kind,mk", MODELS, ids=[m[0] for m in MODELS])
def test_model_fused_forced_matches_oracle_unfused_and_auto(name, kind, mk, fused_calls):
    sysd = D.make_system(kind, 4, r_max=R_MAX, seed=2)
    meta = sysd.pop("_meta")
    model = _model(name, mk, meta)
    dev = D.to_device(sysd, "cuda")
    eligible = _eligible(model)
    assert any(eligible)
    nl = len(model.layers)

    _set_mode(model, [True] * nl)
    fused = _outputs(model, dev)
    assert _ran_on(model, fused_calls) == eligible, "the fused kernel did not run on every eligible layer"
    fused_calls.clear()
    _set_mode(model, [False] * nl)
    unfused = _outputs(model, dev)
    assert not any(_ran_on(model, fused_calls))

    if mk:
        e_ref, ea_ref, f_ref = omodel.energy_and_forces(model.state_dict(), model.config, sysd, torch.float32)
    else:
        e_ref, ea_ref, f_ref = po.energy_and_forces(model.state_dict(), model.config, sysd, torch.float32)
    fs, es = float(f_ref.abs().max()), float(ea_ref.abs().sum())
    for what, o in (("fused", fused), ("unfused", unfused)):
        assert abs(float(o["total_energy"]) - float(e_ref)) <= 1e-5 * es, what
        ferr = float((o["forces"].cpu() - f_ref).abs().max()) / fs
        assert ferr <= 1e-5, (what, ferr)
    assert float((fused["forces"] - unfused["forces"]).abs().max()) <= 2e-6 * float(unfused["forces"].abs().max())
    assert abs(float(fused["total_energy"]) - float(unfused["total_energy"])) <= 2e-6 * float(
        unfused["atomic_energy"].abs().sum())

    # "auto": times both paths once per eligible layer and keeps one; its result is that forced path's, bit for bit
    # (forward and energies; the forces only up to the float64 atomics of the edge-embedding backward)
    prev = ops.deterministic()
    ops.set_deterministic(True)
    try:
        _set_mode(model, ["auto"] * nl)
        auto = _outputs(model, dev)
        choice = [l.conv._fused_choice for l in model.layers]
        timing = [getattr(l.conv, "fused_timing_ms", None) for l in model.layers]
        _set_mode(model, [bool(c) for c in choice])
        forced = _outputs(model, dev)
    finally:
        ops.set_deterministic(prev)
    assert [c is not None for c in choice] == eligible
    assert torch.equal(auto["total_energy"], forced["total_energy"])
    assert torch.equal(auto["atomic_energy"], forced["atomic_energy"])
    assert float((auto["forces"] - forced["forces"]).abs().max()) <= 1e-12 * fs
    print(f"{name}: N={sysd['pos'].shape[0]} E={sysd['edge_index'].shape[1]} auto chose "
          + ", ".join(f"layer {i}: {'fused' if c else 'unfused'} ({t['fused']:.3f} vs {t['unfused']:.3f} ms)"
                      for i, (c, t) in enumerate(zip(choice, timing)) if c is not None))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name,kind,mk", MODELS, ids=[m[0] for m in MODELS])
def test_graphed_md_step_with_fused_kernel_matches_eager(name, kind, mk, fused_calls):
    sysd = D.make_system(kind, 4, r_max=R_MAX, seed=5)
    meta = sysd.pop("_meta")
    model = _model(name, mk, meta)
    dev = D.to_device(sysd, "cuda")
    _set_mode(model, [True] * len(model.layers))
    g = GraphedMDStep(model, dev)
    assert _ran_on(model, fused_calls) == _eligible(model), "the fused kernel did not run on every eligible layer"
    for t in (1, 7):
        pos = D.oscillating_positions(dev["pos"], t, period=50, seed=3)
        out = {k: v.clone() for k, v in g(pos).items()}
        nl = ops.neighbor_list(pos, dev["cell"], True, R_MAX)
        ref = model(dict(dev, pos=pos, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))
        assert int(out["num_edges"]) == nl["edge_index"].shape[1]
        e_ref = float(ref["total_energy"])
        torch.testing.assert_close(out["total_energy"], ref["total_energy"], rtol=1e-12, atol=1e-9 * abs(e_ref))
        fs = float(ref["forces"].abs().max())
        assert float((out["forces"] - ref["forces"]).abs().max()) <= 2e-6 * fs, t
