"""Captured MD steps of a batch of frames on the device: the rows of ``NeighborListPlan(batch=)`` against the batched
``neighbor_list`` (each frame's null edges with its own shift), overflow, capture and replay, the per-frame bounding
boxes of ``nqb_nl_bbox_frames``, ``set_cell`` with per-frame cells, the write contracts of the new entry points, and
batched ``GraphedMDStep`` against the eager batched model, per-frame steps and the float64 oracle."""
import math

import numpy as np
import pytest
import torch

import edge_type_oracle as eto
import open_grid
from batched_oracle import concat_frames, energy_forces_stress
from cell_frames import brute_list, cell_frame, named_cell
from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel

pytestmark = pytest.mark.gpu

R_MAX = 5.0
WATER_L2 = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)
LI3PO4_TABLE = {"Li": {"Li": 3.2, "O": 4.1}, "P": 3.6, "O": {"Li": 2.7, "O": 4.4}}


def _strip(d):
    return {k: v for k, v in d.items() if k != "_meta"}


def _mixed_frames():
    """(frames, pbcs): cubic, tilted, skewed, left-handed and small cells, a slab (TTF), a molecule, one atom and an
    empty frame."""
    fr, pbcs = [], []
    for s, name in enumerate(["cubic", "tilted", "skewed", "left"]):
        fr.append(_strip(cell_frame("li3po4", 3, name, seed=s, outside=True)))
        pbcs.append([True] * 3)
    fr.append(_strip(cell_frame("li3po4", 2, "small", seed=4, outside=True)))
    pbcs.append([True] * 3)
    fr.append(_strip(cell_frame("li3po4", 3, "tilted", seed=5, outside=True, pbc=(True, True, False))))
    pbcs.append([True, True, False])
    mol = _strip(cell_frame("li3po4", 3, "cubic", seed=6, pbc=False))
    mol.pop("cell")
    fr.append(mol)
    pbcs.append([False] * 3)
    one_cell = named_cell("small", 1)
    ei, sh = brute_list(np.zeros((1, 3)), one_cell, True, R_MAX)
    fr.append({"pos": torch.zeros((1, 3), dtype=torch.float64), "cell": torch.from_numpy(one_cell.copy()),
               "atom_types": torch.tensor([1]), "edge_index": torch.from_numpy(ei), "edge_cell_shift": torch.from_numpy(sh)})
    pbcs.append([True] * 3)
    fr.append({"pos": torch.zeros((0, 3), dtype=torch.float64), "cell": torch.from_numpy(named_cell("cubic", 2)),
               "atom_types": torch.zeros(0, dtype=torch.int64), "edge_index": torch.zeros((2, 0), dtype=torch.int64),
               "edge_cell_shift": torch.zeros((0, 3), dtype=torch.float64)})
    pbcs.append([True] * 3)
    return fr, pbcs


def _batch(frames, pbcs):
    return {k: v.cuda() for k, v in concat_frames(frames, pbcs).items()}


def _check_rows(out, ref, plan, capacity, what=""):
    """Row i of ``out``: the real edges of ``ref`` (the exact batched list), then null edges (i, i, pad_shift of i's
    frame) up to the padded row pointer; or only null edges on overflow."""
    N = plan.num_atoms
    frame = plan._fr["frame"].cpu().numpy()
    ei, sh = out["edge_index"].cpu().numpy(), out["edge_cell_shift"].cpu().numpy()
    rp = out["row_ptr"].cpu().numpy()
    ref_rp = ref["row_ptr"].cpu().numpy()
    E = int(ref_rp[-1])
    assert int(out["num_edges"]) == E, what
    over = E > capacity
    assert int(out["overflow"]) == int(over), what
    i = np.arange(N + 1)
    want_rp = capacity * i // N if over else ref_rp + (capacity - E) * i // N
    assert np.array_equal(rp, want_rp), what
    r_ei, r_sh = ref["edge_index"].cpu().numpy(), ref["edge_cell_shift"].cpu().numpy()
    for a in range(N):
        n_real = 0 if over else ref_rp[a + 1] - ref_rp[a]
        b0 = rp[a]
        if n_real:
            assert np.array_equal(ei[:, b0:b0 + n_real], r_ei[:, ref_rp[a]:ref_rp[a + 1]]), (what, a)
            assert np.array_equal(sh[b0:b0 + n_real], r_sh[ref_rp[a]:ref_rp[a + 1]]), (what, a)
        nulls = slice(b0 + n_real, rp[a + 1])
        assert np.all(ei[:, nulls] == a), (what, a)
        assert np.all(sh[nulls] == plan.pad_shift[frame[a]]), (what, a)


def _typed(T, N, seed):
    if not T:
        return {}
    types = torch.from_numpy(np.random.default_rng(seed).integers(0, T, size=N)).cuda()
    return dict(atom_types=types, edge_type_cutoff=torch.from_numpy(eto.random_table(T, R_MAX, seed=seed)))


# ------------------------------------------------------------------------------------------------------------------
# plan rows
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [0, 3], ids=["untyped", "T3"])
@pytest.mark.parametrize("slack", ["exact", "padded", "overflow"])
def test_plan_rows_match_the_batched_list(T, slack):
    frames, pbcs = _mixed_frames()
    b = _batch(frames, pbcs)
    N = b["pos"].shape[0]
    typed = _typed(T, N, 3)
    ref = ops.neighbor_list(b["pos"], b["cell"], b["pbc"], R_MAX, batch=b["batch"], **typed)
    E = ref["edge_index"].shape[1]
    cap = {"exact": E, "padded": E + 3 * N + 7, "overflow": E // 2}[slack]
    plan = ops.NeighborListPlan(N, b["cell"], b["pbc"], R_MAX, cap, batch=b["batch"], open_boundaries=True, **typed)
    # the molecule's cell is the identity, every other frame keeps its own
    np.testing.assert_array_equal(plan.cell[6].cpu().numpy(), np.eye(3))
    assert torch.equal(plan.cell[0], b["cell"][0])
    assert len({tuple(s) for s in plan.pad_shift.tolist()}) > 1  # the frames' null shifts differ
    out = plan.run(b["pos"])
    _check_rows(out, ref, plan, cap, slack)


def test_plan_writes_nothing_past_capacity():
    frames, pbcs = _mixed_frames()
    b = _batch(frames, pbcs)
    N = b["pos"].shape[0]
    ref = ops.neighbor_list(b["pos"], b["cell"], b["pbc"], R_MAX, batch=b["batch"])
    E = ref["edge_index"].shape[1]
    for cap in (E + 11, E // 3):
        plan = ops.NeighborListPlan(N, b["cell"], b["pbc"], R_MAX, cap, batch=b["batch"], open_boundaries=True)
        ei, chk_ei = guarded(2, cap, torch.int64)
        sh, chk_sh = guarded(cap, 3, torch.float64)
        plan.edge_index, plan.edge_cell_shift = ei, sh
        out = plan.run(b["pos"])
        torch.cuda.synchronize()
        chk_ei("edge_index")
        chk_sh("edge_cell_shift")
        assert not bool(is_poison(ei).any()) and not bool(is_poison(sh).any())
        _check_rows(out, ref, plan, cap, f"cap {cap}")


def test_captured_plan_follows_drifting_frames():
    """One captured plan over 30 steps of drifting molecules, a slab and a periodic frame, typed."""
    frames, pbcs = _mixed_frames()
    frames, pbcs = [frames[k] for k in (0, 5, 6, 7)], [pbcs[k] for k in (0, 5, 6, 7)]
    b = _batch(frames, pbcs)
    N = b["pos"].shape[0]
    typed = _typed(3, N, 9)
    E0 = ops.neighbor_list(b["pos"], b["cell"], b["pbc"], R_MAX, batch=b["batch"], **typed)["edge_index"].shape[1]
    cap = E0 + E0 // 4
    plan = ops.NeighborListPlan(N, b["cell"], b["pbc"], R_MAX, cap, batch=b["batch"], open_boundaries=True, **typed)
    static = b["pos"].clone()
    plan.run(static)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = plan.run(static)
    drift = torch.zeros_like(static)
    frame = b["batch"]
    drift[frame == 2] = torch.tensor([0.11, -0.05, 0.07], dtype=torch.float64, device="cuda")
    drift[frame == 1] = torch.tensor([0.0, 0.0, 0.09], dtype=torch.float64, device="cuda")
    for t in range(30):
        pos = D.oscillating_positions(b["pos"], t, period=20, seed=3) + t * drift
        scale = 1.0 + 0.5 * (t % 7 == 3)  # a molecule that suddenly spreads out
        pos[frame == 2] = pos[frame == 2] * scale
        static.copy_(pos)
        graph.replay()
        ref = ops.neighbor_list(pos, b["cell"], b["pbc"], R_MAX, batch=b["batch"], **typed)
        _check_rows(out, ref, plan, cap, f"step {t}")


def test_bbox_frames_writes_the_restated_grid():
    """The blocks after nqb_nl_bbox_frames against the numpy restatement of the kernel's arithmetic, bit for bit;
    for the molecule (identity cell) also against the host values of the batched neighbor_list."""
    frames, pbcs = _mixed_frames()
    b = _batch(frames, pbcs)
    N = b["pos"].shape[0]
    plan = ops.NeighborListPlan(N, b["cell"], b["pbc"], R_MAX, 10, batch=b["batch"], open_boundaries=True)
    packed = plan._params_dev.clone()
    torch.cuda.synchronize()
    _capi.check(_capi.lib().nqb_nl_bbox_frames(b["pos"].data_ptr(), plan.num_frames, plan._fr["atom_ptr"].data_ptr(),
                                               plan._params_dev.data_ptr(), 0), "nqb_nl_bbox_frames")
    torch.cuda.synchronize()
    nbytes = int(_capi.lib().nqb_nl_params_bytes())
    from test_batched_md_step import _Block
    got = [_Block.from_buffer_copy(bytes(plan._params_dev[f * nbytes:(f + 1) * nbytes].cpu().numpy()))
           for f in range(plan.num_frames)]
    before = [_Block.from_buffer_copy(bytes(packed[f * nbytes:(f + 1) * nbytes].cpu().numpy()))
              for f in range(plan.num_frames)]
    atom_ptr = plan._fr["atom_ptr"].cpu().numpy()
    pos = b["pos"].cpu().numpy()
    cells = plan.cell.cpu().numpy()
    for f, p in enumerate(pbcs):
        x = pos[atom_ptr[f]:atom_ptr[f + 1]]
        if all(p) or x.shape[0] == 0:
            assert bytes(got[f]) == bytes(before[f]), f
            continue
        frac = open_grid.frac_coords(x, cells[f])
        lo, hi = open_grid.bbox(frac)
        perp = 1.0 / np.linalg.norm(np.linalg.inv(cells[f]), axis=0)
        for d in range(3):
            if p[d]:
                assert (got[f].lo[d], got[f].width[d], got[f].nb[d]) == (before[f].lo[d], before[f].width[d],
                                                                        before[f].nb[d])
                continue
            l0, w, nb = open_grid.open_grid(lo[d], hi[d], perp[d], R_MAX, open_grid.bin_cap(x.shape[0]))
            assert (got[f].lo[d], got[f].width[d], got[f].nb[d], got[f].sr[d]) == (l0, w, nb, 1), (f, d)
    # the molecule: the host's min / max of pos @ I is pos itself
    mol = pos[atom_ptr[6]:atom_ptr[7]]
    assert list(got[6].lo) == mol.min(0).tolist()
    # the other fields of the blocks are untouched
    for f in range(plan.num_frames):
        assert list(got[f].pad_shift) == list(before[f].pad_shift) and got[f].cap == before[f].cap


def test_variable_cell_plan_follows_per_frame_cells():
    frames, pbcs = _mixed_frames()
    keep = [0, 1, 2, 3, 4, 7, 8]
    frames, pbcs = [frames[k] for k in keep], [pbcs[k] for k in keep]
    b = _batch(frames, pbcs)
    N = b["pos"].shape[0]
    E0 = ops.neighbor_list(b["pos"], b["cell"], True, R_MAX, batch=b["batch"])["edge_index"].shape[1]
    cap = 2 * E0
    plan = ops.NeighborListPlan(N, b["cell"], True, R_MAX, cap, batch=b["batch"], variable_cell=True)
    F = plan.num_frames
    for k, scale in enumerate([1.0, 0.93, 1.08, 0.97]):
        strain = torch.stack([D.oscillating_strain(3 * f + k, period=9).cuda() for f in range(F)]) * scale
        cells = b["cell"] @ strain
        pos = torch.cat([b["pos"][b["batch"] == f] @ strain[f] for f in range(F)])
        plan.set_cell(cells)
        out = plan.run(pos)
        ref = ops.neighbor_list(pos, cells, True, R_MAX, batch=b["batch"])
        _check_rows(out, ref, plan, cap, f"scale {scale}")
        np.testing.assert_array_equal(plan.pad_shift, np.stack([ops.null_edge_shift(c, R_MAX) for c in cells.cpu()]))
    with pytest.raises(ValueError, match=r"\[7, 3, 3\]"):
        plan.set_cell(b["cell"][:2])


def test_new_entry_points_write_contracts():
    """nqb_nl_fill_capacity_frames writes every slot of [2, capacity] and [capacity, 3] and nothing around them;
    nqb_nl_bbox_frames writes only the open-direction fields of the blocks of non-empty frames."""
    frames, pbcs = _mixed_frames()
    b = _batch(frames, pbcs)
    N = b["pos"].shape[0]
    L = _capi.lib()
    for T in (0, 3):
        typed = _typed(T, N, 4)
        plan = ops.NeighborListPlan(N, b["cell"], b["pbc"], R_MAX, 777, batch=b["batch"], open_boundaries=True, **typed)
        plan.run(b["pos"])
        ei, chk_ei = guarded(2, 777, torch.int64)
        sh, chk_sh = guarded(777, 3, torch.float64)
        s, fr, ty = plan._s, plan._fr, plan._ty
        types, rc2, TT = (0, 0, 0) if ty is None else (ty.types.data_ptr(), ty.rc2.data_ptr(), ty.T)
        _capi.check(L.nqb_nl_fill_capacity_frames(N, 777, plan._params_dev.data_ptr(), fr["frame"].data_ptr(),
                                                  fr["bin_base"].data_ptr(), s["wpos"].data_ptr(),
                                                  s["cidx"].data_ptr(), s["base"].data_ptr(), s["order"].data_ptr(),
                                                  s["bin_start"].data_ptr(), plan.row_ptr.data_ptr(),
                                                  plan.overflow.data_ptr(), types, rc2, TT, ei.data_ptr(),
                                                  sh.data_ptr(), 0), "nqb_nl_fill_capacity_frames")
        torch.cuda.synchronize()
        chk_ei("edge_index")
        chk_sh("shifts")
        assert not bool(is_poison(ei).any()) and not bool(is_poison(sh).any())
        assert torch.equal(ei, plan.edge_index) and torch.equal(sh, plan.edge_cell_shift)
    # the blocks as packed (before any run) in a guarded buffer: nothing outside them is written
    plan = ops.NeighborListPlan(N, b["cell"], b["pbc"], R_MAX, 777, batch=b["batch"], open_boundaries=True)
    nbytes = int(L.nqb_nl_params_bytes())
    F = plan.num_frames
    blocks, chk = guarded(F, nbytes // 8, torch.int64, body=plan._params_dev.view(torch.int64).view(F, -1).clone())
    before = blocks.clone()
    _capi.check(L.nqb_nl_bbox_frames(b["pos"].data_ptr(), F, plan._fr["atom_ptr"].data_ptr(), blocks.data_ptr(), 0),
                "nqb_nl_bbox_frames")
    torch.cuda.synchronize()
    chk("blocks")
    changed = (blocks != before).any(0).nonzero().view(-1).cpu().numpy() * 8
    from test_batched_md_step import _Block
    assert changed.size > 0 and changed.min() >= _Block.nb.offset and changed.max() < _Block.r2.offset


# ------------------------------------------------------------------------------------------------------------------
# captured batched steps
# ------------------------------------------------------------------------------------------------------------------
def _model(names, dtype, ann, table=None, zbl=False, preset=None):
    pp = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": list(names)} if zbl else None
    kw = dict(r_max=R_MAX, type_names=names, avg_num_neighbors=ann, model_dtype=dtype, pair_potential=pp,
              per_edge_type_cutoff=table, strict_fast_path=(dtype == torch.float32))
    m = (NequIPEnergyModel.from_preset(preset, **kw) if preset else NequIPEnergyModel(parity=True, **WATER_L2, **kw))
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _water_frames(F, n_side, cells=True):
    frames = []
    for k in range(F):
        s = D.make_system("water", n_side, r_max=R_MAX, seed=k)
        meta = s.pop("_meta")
        eps = np.random.default_rng(100 + k).uniform(-0.03, 0.03, size=(3, 3))
        m = torch.from_numpy(np.eye(3) + 0.5 * (eps + eps.T))
        d = {"pos": s["pos"].double() @ m, "atom_types": s["atom_types"].view(-1),
             "edge_index": torch.zeros((2, 0), dtype=torch.int64)}
        if cells:
            d["cell"] = s["cell"].double().view(3, 3) @ m
        frames.append(d)
    return frames, meta


def _li3po4_frames():
    """A cubic and a tilted periodic frame, a slab and a molecule."""
    fr, pbcs = [], []
    for s, (name, pbc) in enumerate([("cubic", True), ("left", True), ("tilted", (True, True, False))]):
        d = cell_frame("li3po4", 3, name, seed=10 + s, outside=True, pbc=pbc)
        meta = d.pop("_meta")
        fr.append(d)
        pbcs.append(list(pbc) if isinstance(pbc, tuple) else [True] * 3)
    mol = _strip(cell_frame("li3po4", 3, "cubic", seed=14, pbc=False))
    mol.pop("cell")
    fr.append(mol)
    pbcs.append([False] * 3)
    return fr, pbcs, meta


def _example(b, open_frames):
    ex = {k: b[k] for k in ("pos", "atom_types", "batch", "num_atoms", "cell")}
    if open_frames:
        ex["pbc"] = b["pbc"]
    return ex


CASES = {
    # name: (frames, model dtype, deterministic, per-edge-type table, ZBL, preset, capacity = E0 // 2, NPT)
    "water_f32": ("water", torch.float32, False, None, False, None, False, False),
    "water_f64_det": ("water", torch.float64, True, None, False, None, False, False),
    "water_npt": ("water", torch.float32, False, None, False, None, False, True),
    "water_S": ("water", torch.float32, False, None, False, "S", False, False),
    "li3po4_open_zbl_table": ("li3po4", torch.float32, False, LI3PO4_TABLE, True, None, False, False),
    "li3po4_recapture": ("li3po4", torch.float32, False, None, False, None, True, False),
    "water_npt_recapture": ("water", torch.float32, False, None, True, None, True, True),
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", list(CASES))
def test_graphed_batched_step_matches_eager(case):
    kind, dtype, det, table, zbl, preset, small, npt = CASES[case]
    if kind == "water":
        frames, meta = _water_frames(4, 4)
        pbcs = [[True] * 3] * 4
        names = meta["type_names"]
    else:
        frames, pbcs, meta = _li3po4_frames()
        names = ["Li", "P", "O"]
    b = _batch(frames, pbcs)
    open_frames = not all(all(p) for p in pbcs)
    model = _model(names, dtype, meta["avg_num_neighbors"], table, zbl, preset)
    et = {} if table is None else dict(atom_types=b["atom_types"], edge_type_cutoff=model.per_edge_type_cutoff)
    E0 = ops.neighbor_list(b["pos"], b["cell"], b["pbc"], R_MAX, batch=b["batch"], **et)["edge_index"].shape[1]
    F = len(frames)
    prev = ops.deterministic()
    ops.set_deterministic(det)
    try:
        g = GraphedMDStep(model, _example(b, open_frames), capacity=E0 // 2 if small else None, variable_cell=npt)
        if not small:
            assert g.capacity == E0 + math.ceil(0.02 * E0)
        pos0 = b["pos"].clone()
        drift = torch.zeros_like(pos0)
        if open_frames:
            drift[b["batch"] == 3] = torch.tensor([0.013, -0.007, 0.021], dtype=torch.float64, device="cuda")
        for t in range(24):
            pos = D.oscillating_positions(pos0, t, period=12, seed=7) + t * drift
            cells = b["cell"]
            if npt:
                strain = torch.stack([D.oscillating_strain(t + 5 * f, period=12).cuda() for f in range(F)])
                cells = b["cell"] @ strain
                pos = torch.cat([pos[b["batch"] == f] @ strain[f] for f in range(F)])
                out = {k: v.clone() for k, v in g(pos, cells).items()}
            else:
                out = {k: v.clone() for k, v in g(pos).items()}
            nl = ops.neighbor_list(pos, cells, b["pbc"], R_MAX, batch=b["batch"], **et)
            ref = model(dict(b, pos=pos, cell=cells, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]),
                        compute_stress=npt)
            assert out["total_energy"].shape == (F, 1)
            assert int(out["num_edges"]) == nl["edge_index"].shape[1], t
            # per-atom energies are bitwise; a frame's total is an index_add_ of them with float64 atomics, whose
            # order differs between any two calls, eager or captured
            assert torch.equal(out["atomic_energy"], ref["atomic_energy"]), t
            scale = torch.zeros_like(ref["total_energy"]).index_add_(0, b["batch"], ref["atomic_energy"].abs())
            assert bool(((out["total_energy"] - ref["total_energy"]).abs() <= 1e-13 * scale.clamp_min(1.0)).all()), t
            fs = float(ref["forces"].abs().max())
            df = float((out["forces"] - ref["forces"]).abs().max())
            assert df <= (1e-12 if det else 2e-6) * fs, (t, df / fs)
            if npt:
                assert out["stress"].shape == (F, 3, 3) and out["virial"].shape == (F, 3, 3)
                ss = float(ref["stress"].abs().max())
                assert float((out["stress"] - ref["stress"]).abs().max()) <= 2e-6 * ss, t
                assert float((out["virial"] - ref["virial"]).abs().max()) <= 2e-6 * float(ref["virial"].abs().max())
        if small:
            assert g.recaptures >= 1 and g.capacity > E0 // 2
        elif not open_frames:  # a drifting molecule may outgrow the 2 % slack; periodic oscillations do not
            assert g.recaptures == 0
        n0 = _capi.launch_count()
        g(pos, cells) if npt else g(pos)
        assert _capi.launch_count() == n0  # the whole step, list included, is in the graph
    finally:
        ops.set_deterministic(prev)


def test_graphed_batched_step_matches_per_frame_steps_and_the_oracle():
    frames, pbcs, meta = _li3po4_frames()
    b = _batch(frames, pbcs)
    model = _model(["Li", "P", "O"], torch.float32, meta["avg_num_neighbors"])
    g = GraphedMDStep(model, _example(b, True))
    out = {k: v.clone() for k, v in g(b["pos"]).items()}
    off = 0
    for f, (d, p) in enumerate(zip(frames, pbcs)):
        n = d["pos"].shape[0]
        ex = {"pos": d["pos"].cuda(), "atom_types": d["atom_types"].cuda(), "pbc": torch.tensor([p])}
        if d.get("cell") is not None:
            ex["cell"] = d["cell"].cuda()
        one = GraphedMDStep(model, ex)(ex["pos"])
        assert float((out["total_energy"][f] - one["total_energy"].view(1)).abs()) <= 1e-6 * max(
            1.0, float(one["total_energy"].abs()))
        fs = float(one["forces"].abs().max())
        assert float((out["forces"][off:off + n] - one["forces"]).abs().max()) <= 2e-6 * fs, f
        off += n
    # float64 against the float64 batched oracle on the exact list
    m64 = _model(["Li", "P", "O"], torch.float64, meta["avg_num_neighbors"])
    o64 = GraphedMDStep(m64, _example(b, True))(b["pos"])
    nl = ops.neighbor_list(b["pos"], b["cell"], b["pbc"], R_MAX, batch=b["batch"])
    cpu = {k: v.cpu() for k, v in b.items()}
    cpu.update(edge_index=nl["edge_index"].cpu(), edge_cell_shift=nl["edge_cell_shift"].cpu())
    e, _ea, f, _s, _v = energy_forces_stress({k: v.cpu() for k, v in m64.state_dict().items()}, m64.config, cpu)
    assert float((o64["total_energy"].cpu() - e).abs().max()) <= 1e-9 * max(1.0, float(e.abs().max()))
    assert float((o64["forces"].cpu() - f).abs().max()) <= 1e-9 * float(f.abs().max())


def test_moving_one_frame_leaves_the_others_unchanged():
    """Moving frame 1 leaves the other frames' per-atom energies bitwise unchanged, and their forces to the float64 atomic-order noise of the position gradient (deterministic mode; the
    edge-embedding backward accumulates dE/dpos with float64 atomics, so two replays of the same positions agree to
    that noise only)."""
    frames, meta = _water_frames(3, 3)
    b = _batch(frames, [[True] * 3] * 3)
    model = _model(meta["type_names"], torch.float32, meta["avg_num_neighbors"])
    prev = ops.deterministic()
    ops.set_deterministic(True)
    try:
        g = GraphedMDStep(model, _example(b, False))
        out0 = {k: v.clone() for k, v in g(b["pos"]).items()}
        pos = b["pos"].clone()
        sel = b["batch"] == 1
        pos[sel] = D.oscillating_positions(pos[sel], 3, seed=2)
        out1 = {k: v.clone() for k, v in g(pos).items()}
    finally:
        ops.set_deterministic(prev)
    fs = float(out0["forces"].abs().max())
    assert float((out1["forces"][sel] - out0["forces"][sel]).abs().max()) > 1e-3 * fs
    assert float((out1["forces"][~sel] - out0["forces"][~sel]).abs().max()) <= 1e-12 * fs
    assert torch.equal(out1["atomic_energy"][~sel], out0["atomic_energy"][~sel])


def test_single_frame_step_makes_no_frames_call(monkeypatch):
    frames, meta = _water_frames(1, 3)
    model = _model(meta["type_names"], torch.float32, meta["avg_num_neighbors"])
    L = _capi.lib()
    calls = []
    for name in [n for n in _capi.SIGNATURES if "_frames" in n]:
        def boom(*a, _n=name, **k):
            calls.append(_n)
            raise AssertionError(f"{_n} called")
        monkeypatch.setattr(L, name, boom)
    ex = {"pos": frames[0]["pos"].cuda(), "atom_types": frames[0]["atom_types"].cuda(), "cell": frames[0]["cell"].cuda()}
    GraphedMDStep(model, ex)(ex["pos"])
    GraphedMDStep(model, ex, variable_cell=True)(ex["pos"], ex["cell"])
    mol = {"pos": ex["pos"], "atom_types": ex["atom_types"]}
    GraphedMDStep(model, mol)(mol["pos"])
    assert calls == []
