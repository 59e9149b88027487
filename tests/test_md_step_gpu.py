"""Capacity mode of the device neighbour list (nqb_nl_pad / nqb_nl_fill_capacity, ops.NeighborListPlan) and the
graphed MD step (graph.GraphedMDStep): the padded list holds the exact list's edges row by row plus null edges, the
model gives the same energies and forces on it, and one graph follows a trajectory whose edge count changes."""
import ctypes
import math

import numpy as np
import pytest
import torch

from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel

pytestmark = pytest.mark.gpu

R_MAX = 5.0


def _guarded_capacity_list(pos, cell, capacity):
    """nqb_nl_pad + nqb_nl_fill_capacity into guarded, poisoned outputs; returns numpy copies after checking that no
    sentinel word was touched and that every output element was written."""
    N = pos.shape[0]
    plan = ops.NeighborListPlan(N, cell, True, R_MAX, capacity)
    a, s = plan._a, plan._s
    ops._nl_rows(pos, a, s)
    ei, ck_ei = guarded(2, capacity, torch.int64)
    sh, ck_sh = guarded(capacity, 3, torch.float64)
    rp, ck_rp = guarded(1, N + 1, torch.int64)
    ne, ck_ne = guarded(1, 1, torch.int64)
    of, ck_of = guarded(1, 1, torch.int32)
    L, st = _capi.lib(), torch.cuda.current_stream().cuda_stream
    _capi.check(L.nqb_nl_pad(N, capacity, s["row_ptr"].data_ptr(), rp.data_ptr(), ne.data_ptr(), of.data_ptr(), st))
    _capi.check(L.nqb_nl_fill_capacity(N, capacity, a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max, s["wpos"].data_ptr(),
                                       s["cidx"].data_ptr(), s["base"].data_ptr(), s["order"].data_ptr(),
                                       s["bin_start"].data_ptr(), rp.data_ptr(), of.data_ptr(),
                                       _d3(plan.pad_shift), ei.data_ptr(), sh.data_ptr(), st))
    torch.cuda.synchronize()
    for ck, what in ((ck_ei, "edge_index"), (ck_sh, "shifts"), (ck_rp, "row_ptr_pad"), (ck_ne, "num_edges"),
                     (ck_of, "overflow")):
        ck(what)
    for t, what in ((ei, "edge_index"), (sh, "shifts"), (rp, "row_ptr_pad"), (ne, "num_edges"), (of, "overflow")):
        assert not bool(is_poison(t).any()), f"{what}: {int(is_poison(t).sum())} elements never written"
    return (ei.cpu().numpy(), sh.cpu().numpy(), rp.view(-1).cpu().numpy(), int(ne.item()), int(of.item()),
            plan.pad_shift)


def _d3(v):
    return (ctypes.c_double * 3)(*[float(x) for x in v])


def _check_against_exact(pos_np, cell_np, slacks):
    pos = torch.from_numpy(pos_np).cuda()
    cell = torch.from_numpy(cell_np)
    ex = ops.neighbor_list(pos, cell, True, R_MAX)
    ei_x, sh_x, rp_x = (ex["edge_index"].cpu().numpy(), ex["edge_cell_shift"].cpu().numpy(),
                        ex["row_ptr"].cpu().numpy())
    N, E = pos_np.shape[0], ei_x.shape[1]
    assert E > 0
    for slack in slacks:
        cap = E + slack
        ei, sh, rp, ne, of, pad_shift = _guarded_capacity_list(pos, cell, cap)
        assert (ne, of) == (E, 0)
        assert rp[0] == 0 and rp[N] == cap
        pads = np.diff(rp) - np.diff(rp_x)
        assert pads.min() >= 0 and pads.sum() == slack
        assert np.all(np.abs(pads - slack / N) < 1), "padding not spread evenly over the rows"
        for i in range(N):
            b, n, bx, nx = rp[i], rp[i + 1] - rp[i], rp_x[i], rp_x[i + 1] - rp_x[i]
            np.testing.assert_array_equal(ei[:, b:b + nx], ei_x[:, bx:bx + nx])
            np.testing.assert_array_equal(sh[b:b + nx], sh_x[bx:bx + nx])
            assert np.all(ei[:, b + nx:b + n] == i)
            assert np.all(sh[b + nx:b + n] == pad_shift)
        # the plan's own buffers hold the same list
        plan = ops.NeighborListPlan(N, cell, True, R_MAX, cap)
        out = plan.run(pos)
        np.testing.assert_array_equal(out["edge_index"].cpu().numpy(), ei)
        np.testing.assert_array_equal(out["edge_cell_shift"].cpu().numpy(), sh)
        np.testing.assert_array_equal(out["row_ptr"].cpu().numpy(), rp)
        assert int(out["num_edges"]) == E and int(out["overflow"]) == 0


@pytest.mark.parametrize("kind,n_side", [("li3po4", 12), ("water", 10), ("asi", 16)])
def test_capacity_list_matches_exact_list(kind, n_side):
    pos, cell = D.jittered_lattice(n_side, D.PRESETS[kind]["density"], seed=3)
    pos = pos + np.array([3.7, -11.2, 0.4])  # atoms outside the home cell
    N = pos.shape[0]
    _check_against_exact(pos, cell, [0, 1, N - 1, 3 * N + 5, 40 * N // 7])


def test_capacity_list_small_and_triclinic_cells():
    rng = np.random.default_rng(0)
    for L in (3.0, 6.5, 9.0):  # several images of the same neighbour; null-edge shift k = 3 for L = 3
        cell = np.diag([L, L * 1.1, L * 0.9])
        pos = rng.uniform(0, 1, (11, 3)) @ cell
        _check_against_exact(pos, cell, [0, 5, 23])
    cell = np.array([[11.0, 0.0, 0.0], [3.0, 10.0, 0.0], [-2.0, 1.5, 12.0]])
    pos = np.random.default_rng(2).uniform(0, 1, (150, 3)) @ cell
    _check_against_exact(pos, cell, [0, 149, 1000])


def test_capacity_overflow_flags_and_writes_only_null_edges():
    pos, cell = D.jittered_lattice(8, D.PRESETS["li3po4"]["density"], seed=1)
    N = pos.shape[0]
    E = ops.neighbor_list(torch.from_numpy(pos).cuda(), torch.from_numpy(cell), True, R_MAX)["edge_index"].shape[1]
    for cap in (E - 1, E // 2, N // 3):
        ei, sh, rp, ne, of, pad_shift = _guarded_capacity_list(torch.from_numpy(pos).cuda(), torch.from_numpy(cell), cap)
        assert (ne, of) == (E, 1)
        np.testing.assert_array_equal(rp, (cap * np.arange(N + 1)) // N)
        np.testing.assert_array_equal(ei[0], np.repeat(np.arange(N), np.diff(rp)))
        np.testing.assert_array_equal(ei[1], ei[0])
        assert np.all(sh == pad_shift)


# ------------------------------------------------------------------------------------------------------------------
# the model on the padded list
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
    return D.to_device(sysd, "cuda"), meta


@pytest.mark.parametrize("which", ["f32", "f64", "S"])
@pytest.mark.parametrize("deterministic", [False, True])
def test_model_on_padded_list_matches_exact_list(which, deterministic):
    dev, meta = _frame()
    model = _model(which, meta)
    N, E = dev["pos"].shape[0], dev["edge_index"].shape[1]
    plan = ops.NeighborListPlan(N, dev["cell"], True, R_MAX, E + math.ceil(0.05 * E))
    prev = ops.deterministic()
    ops.set_deterministic(deterministic)
    try:
        ref = model(dev)
        ref = {k: ref[k].clone() for k in ("total_energy", "atomic_energy", "forces")}
        nl = plan.run(dev["pos"])
        out = model(dict(dev, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))
    finally:
        ops.set_deterministic(prev)
    assert int(nl["num_edges"]) == E and int(nl["overflow"]) == 0
    # real edges keep their slots in each row and null edges add exact zeros
    assert torch.equal(out["total_energy"], ref["total_energy"]), (float(out["total_energy"]), float(ref["total_energy"]))
    assert torch.equal(out["atomic_energy"], ref["atomic_energy"])
    fs = float(ref["forces"].abs().max())
    df = float((out["forces"] - ref["forces"]).abs().max())
    assert df <= (1e-12 if deterministic else 2e-6) * fs, df / fs


# ------------------------------------------------------------------------------------------------------------------
# the graphed MD step
# ------------------------------------------------------------------------------------------------------------------
def _eager(model, pos, dev):
    nl = ops.neighbor_list(pos, dev["cell"], True, R_MAX)
    out = model(dict(dev, pos=pos, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))
    return out, nl["edge_index"].shape[1]


def _assert_matches(out, ref, what):
    e_ref = float(ref["total_energy"])
    torch.testing.assert_close(out["total_energy"], ref["total_energy"], rtol=1e-12, atol=1e-9 * abs(e_ref), msg=what)
    fs = float(ref["forces"].abs().max())
    df = float((out["forces"] - ref["forces"]).abs().max())
    assert df <= 2e-6 * fs, (what, df / fs)


def test_graphed_md_step_follows_a_trajectory():
    dev, meta = _frame()
    model = _model("f32", meta)
    pos0 = dev["pos"].clone()
    g = GraphedMDStep(model, dev)
    assert g.launches_per_replay > 20
    counts, steps = [], 60
    for t in range(steps):
        pos = D.oscillating_positions(pos0, t, period=50, seed=7)
        host = pos.cpu().pin_memory() if t % 2 else pos  # host (pinned) and device positions
        out = g(host)
        ref, E = _eager(model, pos, dev)
        assert int(out["num_edges"]) == E
        _assert_matches(out, ref, f"step {t}")
        counts.append(E)
    changed = sum(a != b for a, b in zip(counts, counts[1:]))
    assert changed >= 0.6 * (steps - 1), f"the edge count changed at only {changed} of {steps - 1} steps"
    assert g.capacity >= max(counts)


def test_graphed_md_step_recaptures_on_overflow():
    dev, meta = _frame(n_side=5)
    model = _model("f32", meta)
    E1 = dev["edge_index"].shape[1]
    # capture on a seeded random displacement of the frame, which has fewer edges than the frame itself (same cell)
    gen = torch.Generator().manual_seed(11)
    pos0 = dev["pos"] + 0.3 * torch.randn(tuple(dev["pos"].shape), generator=gen, dtype=torch.float64).cuda()
    E0 = ops.neighbor_list(pos0, dev["cell"], True, R_MAX)["edge_index"].shape[1]
    assert E1 > E0
    g = GraphedMDStep(model, dict(dev, pos=pos0), capacity=E0)
    out = g(pos0)
    assert int(out["num_edges"]) == E0 and g.recaptures == 0 and g.capacity == E0
    out = g(dev["pos"])  # E1 > capacity edges
    assert g.recaptures == 1 and g.capacity == math.ceil(1.02 * E1) > E0
    assert int(out["num_edges"]) == E1
    ref, _ = _eager(model, dev["pos"], dev)
    _assert_matches(out, ref, "after re-capture")
    out = g(pos0)  # fewer edges again: no re-capture, the capacity stays
    assert g.recaptures == 1 and int(out["num_edges"]) == E0


def test_graphed_md_step_replay_launches_nothing_and_is_deterministic():
    dev, meta = _frame(n_side=5)
    model = _model("f32", meta)
    prev = ops.deterministic()
    ops.set_deterministic(True)
    try:
        g = GraphedMDStep(model, dev)
        pos = D.oscillating_positions(dev["pos"], 3, seed=2)
        n0 = _capi.launch_count()
        a = {k: v.clone() for k, v in g(pos).items()}
        b = {k: v.clone() for k, v in g(pos).items()}
        assert _capi.launch_count() == n0, "a replay launched nequip_b200 kernels eagerly"
        ref, _ = _eager(model, pos, dev)
    finally:
        ops.set_deterministic(prev)
    assert torch.equal(a["total_energy"], b["total_energy"]) and torch.equal(a["atomic_energy"], b["atomic_energy"])
    fs = float(ref["forces"].abs().max())
    assert float((a["forces"] - b["forces"]).abs().max()) <= 1e-12 * fs
    assert float((a["forces"] - ref["forces"]).abs().max()) <= 1e-12 * fs
    assert torch.equal(a["total_energy"], ref["total_energy"])
