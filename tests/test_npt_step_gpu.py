"""Variable-cell neighbour list (nqb_nl_*_dp, ops.NeighborListPlan(variable_cell=True)) and the graphed NPT step
(graph.GraphedMDStep(variable_cell=True)): one plan follows a sequence of cells with the exact lists of
ops.neighbor_list, and one graph follows a trajectory whose cell changes every step, stress and virial included."""
import math

import numpy as np
import pytest
import torch

from cell_frames import cell_frame
from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel

pytestmark = pytest.mark.gpu

R_MAX = 5.0


def _cell_sequence(cell0):
    """cell0, +-3 % isotropic, sheared to triclinic, shrunk below 2 r_max (several images of a neighbour), cell0."""
    shear = np.array([[1.0, 0.0, 0.0], [0.22, 1.0, 0.0], [-0.12, 0.08, 1.0]])
    small = cell0 * (8.2 / np.linalg.norm(cell0, axis=1).max()) @ shear
    return [("cell0", cell0), ("expanded", cell0 * 1.03), ("compressed", cell0 * 0.97),
            ("triclinic", cell0 @ shear), ("small", small), ("back", cell0)]


def _guarded_dp_list(plan, pos, capacity):
    """The three _dp kernels and nqb_nl_pad of ``plan`` (after its set_cell), every output in a guarded, poisoned
    buffer; returns numpy copies after checking that no sentinel word was touched and every element was written."""
    N = pos.shape[0]
    s = dict(plan._s)
    outs = {"wpos": guarded(N, 3, torch.float64), "base": guarded(N, 3, torch.int32),
            "binid": guarded(1, N, torch.int64), "cidx": guarded(N, 3, torch.int32),
            "counts": guarded(1, N, torch.int64)}
    for k, (t, _ck) in outs.items():
        s[k] = t.view(-1) if k in ("binid", "counts") else t
    ops._nl_rows(pos, plan._a, s, plan._params_dev)
    ei, ck_ei = guarded(2, capacity, torch.int64)
    sh, ck_sh = guarded(capacity, 3, torch.float64)
    rp, ck_rp = guarded(1, N + 1, torch.int64)
    ne, ck_ne = guarded(1, 1, torch.int64)
    of, ck_of = guarded(1, 1, torch.int32)
    L, st = _capi.lib(), torch.cuda.current_stream().cuda_stream
    _capi.check(L.nqb_nl_pad(N, capacity, s["row_ptr"].data_ptr(), rp.data_ptr(), ne.data_ptr(), of.data_ptr(), st))
    _capi.check(L.nqb_nl_fill_capacity_dp(N, capacity, plan._params_dev.data_ptr(), s["wpos"].data_ptr(),
                                          s["cidx"].data_ptr(), s["base"].data_ptr(), s["order"].data_ptr(),
                                          s["bin_start"].data_ptr(), rp.data_ptr(), of.data_ptr(), ei.data_ptr(),
                                          sh.data_ptr(), st))
    torch.cuda.synchronize()
    checks = [(ck, k) for k, (_t, ck) in outs.items()] + [
        (ck_ei, "edge_index"), (ck_sh, "shifts"), (ck_rp, "row_ptr_pad"), (ck_ne, "num_edges"), (ck_of, "overflow")]
    for ck, what in checks:
        ck(what)
    written = [(t, k) for k, (t, _ck) in outs.items()] + [
        (ei, "edge_index"), (sh, "shifts"), (rp, "row_ptr_pad"), (ne, "num_edges"), (of, "overflow")]
    for t, what in written:
        assert not bool(is_poison(t).any()), f"{what}: {int(is_poison(t).sum())} elements never written"
    return ei.cpu().numpy(), sh.cpu().numpy(), rp.view(-1).cpu().numpy(), int(ne.item()), int(of.item())


def _assert_rows_match(ei, sh, rp, ex, pad_shift, cell, what):
    ei_x, sh_x, rp_x = (ex["edge_index"].cpu().numpy(), ex["edge_cell_shift"].cpu().numpy(),
                        ex["row_ptr"].cpu().numpy())
    N = rp.shape[0] - 1
    pads = np.diff(rp) - np.diff(rp_x)
    assert pads.min() >= 0, what
    for i in range(N):
        b, n, bx, nx = rp[i], rp[i + 1] - rp[i], rp_x[i], rp_x[i + 1] - rp_x[i]
        np.testing.assert_array_equal(ei[:, b:b + nx], ei_x[:, bx:bx + nx], err_msg=f"{what} row {i}")
        np.testing.assert_array_equal(sh[b:b + nx], sh_x[bx:bx + nx], err_msg=f"{what} row {i}")
        assert np.all(ei[:, b + nx:b + n] == i), f"{what} row {i}"
        assert np.all(sh[b + nx:b + n] == pad_shift), f"{what} row {i}"
    # every null edge (i, i, shift) is at least r_max + |a_d| long in THIS cell
    null = np.ones(ei.shape[1], dtype=bool)
    for i in range(N):
        null[rp[i]:rp[i] + (rp_x[i + 1] - rp_x[i])] = False
    assert null.sum() == ei.shape[1] - ei_x.shape[1]
    lengths = np.linalg.norm(sh[null] @ cell, axis=1)
    assert lengths.min() >= R_MAX + np.linalg.norm(cell, axis=1).max(), (what, lengths.min())


def test_one_plan_follows_a_sequence_of_cells():
    frac, cell0 = D.jittered_lattice(6, D.PRESETS["li3po4"]["density"], seed=3)
    frac = frac @ np.linalg.inv(cell0) + np.array([0.31, -1.2, 0.05])  # fractional, some outside the home cell
    seq = _cell_sequence(cell0)
    N = frac.shape[0]
    exact = {}
    for name, c in seq:
        pos = torch.from_numpy(frac @ c).cuda()
        exact[name] = (pos, ops.neighbor_list(pos, torch.from_numpy(c), True, R_MAX))
    counts = {name: ex["edge_index"].shape[1] for name, (_p, ex) in exact.items()}
    assert counts["small"] > 2 * counts["cell0"] and counts["compressed"] > counts["cell0"] > counts["expanded"]
    capacity = max(counts.values()) + 37
    plan = ops.NeighborListPlan(N, torch.from_numpy(cell0), True, R_MAX, capacity, variable_cell=True)
    nb = plan.nbins
    assert min(nb) > 1
    for name, c in seq:
        pos, ex = exact[name]
        plan.set_cell(torch.from_numpy(c) if name != "triclinic" else torch.from_numpy(c).cuda())
        assert plan.nbins == nb and tuple(plan._a.nb) == nb, "the bin grid is fixed for the plan's lifetime"
        np.testing.assert_array_equal(plan.pad_shift, ops.null_edge_shift(c, R_MAX))
        out = plan.run(pos)
        ei, sh, rp = (out["edge_index"].cpu().numpy(), out["edge_cell_shift"].cpu().numpy(),
                      out["row_ptr"].cpu().numpy())
        assert int(out["num_edges"]) == counts[name] and int(out["overflow"]) == 0
        _assert_rows_match(ei, sh, rp, ex, plan.pad_shift, c, name)
        gei, gsh, grp, ne, of = _guarded_dp_list(plan, pos, capacity)
        assert (ne, of) == (counts[name], 0)
        np.testing.assert_array_equal(gei, ei)
        np.testing.assert_array_equal(gsh, sh)
        np.testing.assert_array_equal(grp, rp)


def test_set_cell_checks_its_argument():
    cell = torch.eye(3, dtype=torch.float64) * 12.0
    plan = ops.NeighborListPlan(20, cell, True, R_MAX, 100, variable_cell=True)
    for bad in (torch.eye(2, dtype=torch.float64), torch.full((3, 3), float("nan"), dtype=torch.float64),
                torch.zeros(3, 3, dtype=torch.float64), cell.clone().fill_(1.0)):
        with pytest.raises(ValueError):
            plan.set_cell(bad)
        with pytest.raises(ValueError):
            plan.set_cell(bad.cuda())
    with pytest.raises(ValueError):
        ops.NeighborListPlan(20, cell, True, R_MAX, 100).set_cell(cell)


# ------------------------------------------------------------------------------------------------------------------
# the graphed NPT step
# ------------------------------------------------------------------------------------------------------------------
def _model(which, meta):
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"])
    if which == "S":
        m = NequIPEnergyModel.from_preset("S", strict_fast_path=True, **kw)
    else:
        dt = torch.float64 if which == "f64" else torch.float32
        m = NequIPEnergyModel(parity=True, l_max=2, num_layers=4, num_features=64, radial_mlp_depth=1,
                              radial_mlp_width=128, model_dtype=dt, strict_fast_path=(dt == torch.float32), **kw)
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _frame(n_side=6, seed=0):
    sysd = D.make_system("li3po4", n_side, r_max=R_MAX, seed=seed)
    meta = sysd.pop("_meta")
    dev = D.to_device({k: sysd[k] for k in ("pos", "atom_types", "cell")}, "cuda")
    return dev, meta


def _npt_frame(dev, pos0, t):
    S = D.oscillating_strain(t).cuda()
    return D.oscillating_positions(pos0, t, period=50, seed=7) @ S, dev["cell"] @ S


def _eager(model, pos, cell, dev):
    nl = ops.neighbor_list(pos, cell, True, R_MAX)
    out = model(dict(dev, pos=pos, cell=cell, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]),
                compute_stress=True)
    return out, nl["edge_index"].shape[1]


def _rel(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


def _assert_matches(out, ref, what, tol=2e-6):
    e_ref = float(ref["total_energy"])
    torch.testing.assert_close(out["total_energy"], ref["total_energy"], rtol=1e-12, atol=1e-9 * abs(e_ref), msg=what)
    for k in ("forces", "stress", "virial"):
        assert _rel(out[k], ref[k]) <= tol, (what, k, _rel(out[k], ref[k]))


def _follow(g, model, dev, pos0, steps, start=0):
    counts, devs = [], []
    for t in range(start, start + steps):
        pos, cell = _npt_frame(dev, pos0, t)
        # host (pinned) and device positions, host and device cells
        out = g(pos.cpu().pin_memory() if t % 2 else pos, cell.cpu() if t % 3 else cell)
        assert tuple(out["stress"].shape) == (1, 3, 3) and tuple(out["virial"].shape) == (1, 3, 3)
        ref, E = _eager(model, pos, cell, dev)
        assert int(out["num_edges"]) == E, f"step {t}"
        _assert_matches(out, ref, f"step {t}")
        devs.append(max(_rel(out[k], ref[k]) for k in ("forces", "stress", "virial")))
        counts.append(E)
    return counts, devs


def test_graphed_npt_step_follows_a_trajectory():
    dev, meta = _frame()
    model = _model("f32", meta)
    pos0 = dev["pos"].clone()
    g = GraphedMDStep(model, dev, variable_cell=True)
    steps = 60
    counts, devs = _follow(g, model, dev, pos0, steps)
    changed = sum(a != b for a, b in zip(counts, counts[1:]))
    assert changed >= 0.6 * (steps - 1), f"the edge count changed at only {changed} of {steps - 1} steps"
    assert g.capacity >= max(counts)
    print(f"max relative deviation of forces / stress / virial over {steps} steps: {max(devs):.3g}")


@pytest.mark.parametrize("which", ["f64", "S"])
def test_graphed_npt_step_other_models(which):
    dev, meta = _frame(n_side=5)
    model = _model(which, meta)
    g = GraphedMDStep(model, dev, variable_cell=True)
    _follow(g, model, dev, dev["pos"].clone(), 12, start=5)


def test_graphed_npt_step_deterministic_matches_the_exact_list():
    dev, meta = _frame(n_side=5)
    model = _model("f32", meta)
    prev = ops.deterministic()
    ops.set_deterministic(True)
    try:
        g = GraphedMDStep(model, dev, variable_cell=True)
        for t in (4, 17, 29):
            pos, cell = _npt_frame(dev, dev["pos"], t)
            out = {k: v.clone() for k, v in g(pos, cell).items()}
            ref, E = _eager(model, pos, cell, dev)
            assert int(out["num_edges"]) == E
            assert torch.equal(out["total_energy"], ref["total_energy"]), t
            for k in ("forces", "stress", "virial"):
                assert _rel(out[k], ref[k]) <= 1e-12, (t, k, _rel(out[k], ref[k]))
    finally:
        ops.set_deterministic(prev)


def test_graphed_npt_step_recaptures_once_on_compression():
    dev, meta = _frame(n_side=5)
    model = _model("f32", meta)
    g = GraphedMDStep(model, dev, variable_cell=True)
    cap0 = g.capacity
    out = g(dev["pos"], dev["cell"])
    assert g.recaptures == 0
    S = torch.diag(torch.tensor([0.95, 0.96, 0.95], dtype=torch.float64, device="cuda"))
    pos, cell = dev["pos"] @ S, dev["cell"] @ S
    out = g(pos, cell)
    ref, E = _eager(model, pos, cell, dev)
    assert E > cap0
    assert g.recaptures == 1 and g.capacity == math.ceil(1.02 * E) > cap0
    assert int(out["num_edges"]) == E
    _assert_matches(out, ref, "after re-capture")
    out = g(dev["pos"], dev["cell"])  # back to the first cell: fewer edges, no re-capture, the capacity stays
    ref, E0 = _eager(model, dev["pos"], dev["cell"], dev)
    assert g.recaptures == 1 and g.capacity == math.ceil(1.02 * E) and int(out["num_edges"]) == E0
    _assert_matches(out, ref, "back at the first cell")


def test_graphed_npt_replay_launches_nothing_eagerly():
    dev, meta = _frame(n_side=5)
    model = _model("f32", meta)
    g = GraphedMDStep(model, dev, variable_cell=True)
    pos, cell = _npt_frame(dev, dev["pos"], 3)
    g(pos, cell)
    n0 = _capi.launch_count()
    g(pos, cell.cpu())
    g(pos, cell)
    assert _capi.launch_count() == n0, "a replay launched nequip_b200 kernels eagerly"
    with pytest.raises(ValueError):
        g(pos)  # the cell is an input of every step
    fixed = GraphedMDStep(model, dev)
    with pytest.raises(ValueError):
        fixed(pos, cell)


def test_graphed_npt_step_at_a_left_handed_cell_matches_the_oracle():
    """Captured at a cubic cell, replayed at a triclinic left-handed one (det < 0) with atoms several cells away:
    energy, forces and stress within 1e-5 of the oracle on the brute-force list of that cell."""
    dev, meta = _frame(n_side=5)
    model = _model("f32", meta)
    g = GraphedMDStep(model, dev, variable_cell=True)
    f = cell_frame("li3po4", 5, "left", seed=0, outside=True)
    assert torch.equal(f["atom_types"], dev["atom_types"].cpu()) and float(torch.linalg.det(f["cell"])) < 0
    out = g(f["pos"].cuda(), f["cell"])
    assert int(out["num_edges"]) == f["edge_index"].shape[1]
    e_ref, f_ref, s_ref, _v = omodel.energy_forces_stress(model.state_dict(), model.config, f, torch.float32)
    escale = float(out["atomic_energy"].abs().sum())
    assert abs(float(out["total_energy"]) - float(e_ref)) <= 1e-5 * escale, (float(out["total_energy"]), float(e_ref))
    assert _rel(out["forces"].cpu(), f_ref) <= 1e-5, _rel(out["forces"].cpu(), f_ref)
    assert _rel(out["stress"].cpu(), s_ref) <= 1e-5, _rel(out["stress"].cpu(), s_ref)
