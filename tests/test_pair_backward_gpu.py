"""The radial MLP's backward on the slots of the reverse-edge pair map (nqb_gemm_grouped_pair_sum +
nqb_mlp_hidden_bwd_rows): the gathered-sum GEMM against float64, both kernels' write contracts, and whole models
against the float64 oracle and against the same model with a map without pairs."""
import math

import pytest
import torch

from kernel_contracts import assert_elementwise, gemm_bound, guarded, is_poison
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.nn import dense
from nequip_b200.nn.model import NequIPEnergyModel, ScalarLinearLayer
from oracle import model as omodel

pytestmark = pytest.mark.gpu

R_MAX = 5.0


def _mlp(W, seed=0):
    g = torch.Generator().manual_seed(seed)
    l1, l2 = ScalarLinearLayer(8, 128, 1 / math.sqrt(8)).cuda(), ScalarLinearLayer(128, W, 1 / math.sqrt(128)).cuda()
    with torch.no_grad():
        l1.weight.copy_(torch.randn(8, 128, generator=g))
        l2.weight.copy_(torch.randn(128, W, generator=g))
    return dense.RadialMLPGemm(l1, l2, "cuda"), l2


def _slots(E, U, seed):
    """U slots covering rows of [0, E): slot u = (r[u], r[U + u]) for u < E - U, (r[u], -1) after; rows >= U are -7."""
    g = torch.Generator().manual_seed(seed)
    r = torch.randperm(E, generator=g)
    rows = torch.full((E, 2), -7, dtype=torch.int64)
    rows[:U, 0] = r[:U]
    rows[:U, 1] = -1
    npair = min(U, E - U)
    rows[:npair, 1] = r[U:U + npair]
    return rows.cuda()


# ---------------------------------------------------------------------------------------------------------------
# the gathered-sum GEMM and the slot hidden-layer backward
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("W", [192, 960, 1728])
@pytest.mark.parametrize("U", ["zero", "odd", "half", "capacity"])
def test_pair_sum_gemm_and_slot_hidden_bwd(W, U):
    E = 3001
    # half: every slot has a partner; odd: U not a multiple of 128 with 2U < E, so some rows are in no slot;
    # capacity: U = E, every partner is -1
    U = {"zero": 0, "odd": 1111, "half": (E + 1) // 2, "capacity": E}[U]
    mlp, l2 = _mlp(W, seed=W)
    g = torch.Generator().manual_seed(U + W)
    gw = torch.randn(E, W, generator=g).cuda()
    emb = (torch.rand(E, 8, generator=g) * 2 - 0.7).cuda()
    rows = _slots(E, U, U + 1)
    count = torch.tensor([U], dtype=torch.int64, device="cuda")

    gh, ck_gh = guarded(E, 128, torch.float32)
    mlp.bwd.run_pair_sum(gw, gh, (rows, count))
    torch.cuda.synchronize()
    ck_gh("grad_h")
    assert bool(is_poison(gh[U:]).all()), "rows >= count written"
    if U:
        rep, par = rows[:U, 0], rows[:U, 1]
        a = gw[rep].double() + torch.where((par >= 0).unsqueeze(1), gw[par.clamp(min=0)].double(), 0.0)
        B = l2.weight.detach().t().double()  # grad_h = gw_slot @ (W2 a2)^T
        ref = a @ B * float(l2.alpha)
        assert not bool(is_poison(gh[:U]).any())
        assert_elementwise(gh[:U].double(), ref, gemm_bound(a, B, float(l2.alpha), ref=ref), f"grad_h W={W} U={U}")

    # slot backward of the hidden layer: representative rows = the per-edge kernel on the slot's grad_h, partner rows
    # exactly 0, every row of a covering map written, nothing else
    gemb, ck_ge = guarded(E, 8, torch.float32)
    ops.mlp_hidden_bwd_rows(emb, mlp.w1s, gh, (rows, count), gemb)
    torch.cuda.synchronize()
    ck_ge("grad_emb")
    listed = torch.cat([rows[:U, 0], rows[:U, 1][rows[:U, 1] >= 0]])
    written = ~is_poison(gemb).all(1)
    mask = torch.zeros(E, dtype=torch.bool, device="cuda")
    mask[listed] = True
    assert torch.equal(written, mask)
    if U:
        assert not bool(is_poison(gemb[listed]).any())
        ref_rep = torch.empty((U, 8), device="cuda")
        ops.mlp_hidden_bwd(emb[rows[:U, 0]].contiguous(), mlp.w1s, gh[:U].contiguous(), ref_rep)
        torch.cuda.synchronize()
        assert torch.equal(gemb[rows[:U, 0]], ref_rep)
        par = rows[:U, 1][rows[:U, 1] >= 0]
        assert bool((gemb[par] == 0).all()) and not bool(torch.signbit(gemb[par]).any())


def test_pair_sum_rejects_non_plain_problems():
    l2 = ScalarLinearLayer(128, 64, 1.0).cuda()
    gg = ops.GroupedGemm([ops.GemmProblem(0, 128, 0, 64, l2.weight.detach(), act="silu")], "cuda")
    rows = torch.zeros((4, 2), dtype=torch.int64, device="cuda")
    count = torch.ones(1, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        gg.run_pair_sum(torch.zeros(4, 128, device="cuda"), torch.zeros(4, 64, device="cuda"), (rows, count))


def test_grad_emb_slot_sum_equals_per_edge_sum():
    """Summed per slot, the slot backward's grad_emb equals the per-edge backward's on a real pair map."""
    sysd = D.make_system("li3po4", 6, r_max=R_MAX, seed=2)
    d = D.to_device(sysd, "cuda")
    ei = d["edge_index"]
    _v, _y, emb = ops.edge_embed(d["pos"], ei, d["edge_cell_shift"], d["cell"], lmax=2, num_bessel=8, r_max=R_MAX,
                                 prefactor=2 * math.pi / R_MAX ** 2)
    pairs = ops.edge_pairs(ei, d["edge_cell_shift"], emb, ops.build_csr(ei[0], d["pos"].shape[0]))
    E = ei.shape[1]
    U = int(pairs[1].item())
    assert 2 * U == E
    mlp, _ = _mlp(960, seed=7)
    gw = torch.randn(E, 960, generator=torch.Generator().manual_seed(1)).cuda()
    slot = mlp.grad_emb(emb, gw, (), pairs)
    edge = mlp.grad_emb(emb, gw, ())
    rep, par = pairs[0][:U, 0], pairs[0][:U, 1]
    assert bool((slot[par] == 0).all())
    want = edge[rep].double() + edge[par].double()
    err = float((slot[rep].double() - want).abs().max()) / float(want.abs().max())
    assert err <= 2e-6, err


# ---------------------------------------------------------------------------------------------------------------
# whole models
# ---------------------------------------------------------------------------------------------------------------
def _count_calls(monkeypatch):
    calls = {"gemm": 0, "hidden": 0}
    real_gemm, real_hidden = ops.GroupedGemm.run_pair_sum, ops.mlp_hidden_bwd_rows

    def gemm(self, *a):
        calls["gemm"] += 1
        return real_gemm(self, *a)

    def hidden(*a):
        calls["hidden"] += 1
        return real_hidden(*a)

    monkeypatch.setattr(ops.GroupedGemm, "run_pair_sum", gemm)
    monkeypatch.setattr(ops, "mlp_hidden_bwd_rows", hidden)
    return calls


def _no_pairs(edge_index, shift, emb, csr):
    E = edge_index.shape[1]
    ar = torch.arange(E, dtype=torch.int64, device=emb.device)
    return torch.stack([ar, torch.full_like(ar, -1)], 1).contiguous(), torch.full((1,), E, dtype=torch.int64,
                                                                                     device=emb.device)


def _model(n_side=5, seed=1, **kw):
    sysd = D.make_system("li3po4", n_side, r_max=R_MAX, seed=seed)
    meta = sysd.pop("_meta")
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], l_max=2, num_layers=4, num_features=64,
                              parity=True, avg_num_neighbors=meta["avg_num_neighbors"], strict_fast_path=True,
                              **kw).cuda()
    for p in model.parameters():
        p.requires_grad_(False)
    for layer in model.layers:  # the unfused radial MLP on every layer, whatever the one-off timing would pick
        layer.conv.use_fused_radial_tp = False
    return model, sysd


def _close(a, b, keys=("forces", "stress", "virial"), rel=2e-6):
    """Energies bitwise equal, ``keys`` within rel * max|b| (each key that ``a`` holds)."""
    for k in ("total_energy", "atomic_energy"):
        if k in a:
            assert torch.equal(a[k], b[k]), k
    assert any(k in a for k in keys)
    for k in keys:
        if k in a:
            scale = float(b[k].abs().max())
            err = float((a[k] - b[k]).abs().max())
            assert err <= rel * scale + 1e-12, (k, err / scale)


@pytest.mark.timeout(900)
def test_bench_family_model_matches_oracle_and_no_pairs(monkeypatch):
    model, sysd = _model()
    dev = D.to_device(sysd, "cuda")
    calls = _count_calls(monkeypatch)
    out = {k: v.clone() for k, v in model(dev, compute_stress=True).items() if torch.is_tensor(v)}
    assert calls["gemm"] == 4 and calls["hidden"] == 4, calls  # one slot backward per layer
    e_ref, f_ref, s_ref, v_ref = omodel.energy_forces_stress(model.state_dict(), model.config, sysd, torch.float32)
    escale = float(out["atomic_energy"].abs().sum())
    assert abs(float(out["total_energy"]) - float(e_ref)) <= 1e-5 * escale
    for k, ref in (("forces", f_ref), ("stress", s_ref), ("virial", v_ref)):
        err = float((out[k].cpu() - ref).abs().max()) / float(ref.abs().max())
        assert err <= 1e-5, (k, err)
    monkeypatch.setattr(ops, "edge_pairs", _no_pairs)
    base = {k: v.clone() for k, v in model(dev, compute_stress=True).items() if torch.is_tensor(v)}
    _close(out, base)


@pytest.mark.timeout(600)
def test_edge_vectors_and_asymmetric_cutoffs_keep_the_per_edge_backward(monkeypatch):
    model, sysd = _model(n_side=4)
    dev = D.to_device(sysd, "cuda")
    calls = _count_calls(monkeypatch)
    vec = ops.edge_embed(dev["pos"], dev["edge_index"], dev["edge_cell_shift"], dev["cell"], lmax=0, num_bessel=8,
                         r_max=R_MAX)[0]
    d2 = {k: v for k, v in dev.items() if k not in ("edge_cell_shift", "cell")}
    d2["edge_vectors"] = vec.clone()
    out = model(d2)
    assert "edge_forces" in out
    assert calls == {"gemm": 0, "hidden": 0}, calls
    names = model.config["type_names"]
    asym = {names[0]: {names[1]: 4.0}, names[1]: {names[0]: 3.5}}
    m2, s2 = _model(n_side=4, per_edge_type_cutoff=asym)
    m2(D.to_device(s2, "cuda"))
    assert calls == {"gemm": 0, "hidden": 0}, calls
    sym = {names[0]: {names[1]: 4.0}, names[1]: {names[0]: 4.0}}
    m3, s3 = _model(n_side=4, per_edge_type_cutoff=sym)
    m3(D.to_device(s3, "cuda"))
    assert calls == {"gemm": 4, "hidden": 4}, calls


@pytest.mark.timeout(600)
def test_deterministic_mode_repeats():
    """The slot backward has no atomics: its grad_emb is bitwise repeatable.  In deterministic mode the whole model's
    energy is bitwise repeatable and its forces agree to the float64 atomic-order noise of the position gradient (the
    edge-embedding backward accumulates dE/dpos with float64 atomics, as in the per-edge backward)."""
    model, sysd = _model()
    dev = D.to_device(sysd, "cuda")
    ei = dev["edge_index"]
    _v, _y, emb = ops.edge_embed(dev["pos"], ei, dev["edge_cell_shift"], dev["cell"], lmax=2, num_bessel=8,
                                 r_max=R_MAX, prefactor=2 * math.pi / R_MAX ** 2)
    pairs = ops.edge_pairs(ei, dev["edge_cell_shift"], emb, ops.build_csr(ei[0], dev["pos"].shape[0]))
    ops.set_deterministic(True)
    try:
        a = {k: v.clone() for k, v in model(dev).items() if torch.is_tensor(v)}
        b = {k: v.clone() for k, v in model(dev).items() if torch.is_tensor(v)}
    finally:
        ops.set_deterministic(False)
    assert torch.equal(a["total_energy"], b["total_energy"])
    assert float((a["forces"] - b["forces"]).abs().max()) <= 1e-12 * float(a["forces"].abs().max())
    mlp = model.layers[2].conv._tc_cache[1]["mlp"]  # prepared by the calls above
    gw = torch.randn(ei.shape[1], mlp.W, generator=torch.Generator().manual_seed(4)).cuda()
    assert torch.equal(mlp.grad_emb(emb, gw, (), pairs), mlp.grad_emb(emb, gw, (), pairs))


@pytest.mark.timeout(900)
def test_graphed_steps_use_the_slot_backward(monkeypatch):
    from nequip_b200.graph import GraphedEnergyForces, GraphedMDStep

    model, sysd = _model()
    dev = D.to_device(sysd, "cuda")
    eager = model(dev)
    calls = _count_calls(monkeypatch)
    ga = GraphedEnergyForces(model, dev)
    out = ga.replay()
    assert calls["gemm"] >= 4 and calls["hidden"] >= 4
    _close(out, eager, keys=("forces",), rel=1e-6)
    del ga
    # padded capacity (null edges get slots of their own), a re-capture, a fixed and a variable cell
    pos1 = D.oscillating_positions(dev["pos"], 7, seed=3)
    for variable in (False, True):
        outs = []
        for fn in (ops.edge_pairs, _no_pairs):
            with monkeypatch.context() as m:
                m.setattr(ops, "edge_pairs", fn)
                e0 = int(dev["edge_index"].shape[1])
                g = GraphedMDStep(model, dev, capacity=e0 // 2, **(dict(variable_cell=True) if variable else {}))
                args = (pos1, dev["cell"] * 1.01) if variable else (pos1,)
                o1 = {k: v.clone() for k, v in g(*args).items()}
                assert g.recaptures == 1
                outs.append(o1)
                del g
        _close(outs[0], outs[1], keys=("forces", "stress", "virial") if variable else ("forces",))
