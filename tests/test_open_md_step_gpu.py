"""Open boundary directions on the device: the bounding box kernel (nqb_nl_bbox), the neighbour-list plan built with
``open_boundaries=True`` and graph.GraphedMDStep on molecules without a cell and on slabs.  The plan's rows are those
of ops.neighbor_list and of the float64 brute-force list, its bins those of a numpy restatement of the device grid,
one plan (and one captured graph) follows frames whose bounding box moves, shrinks and grows, and the graphed step
gives the energies of the eager model on the exact list bit for bit."""
import numpy as np
import pytest
import torch

import open_grid
from cell_frames import brute_list, cell_frame
from kernel_contracts import guarded
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel

pytestmark = pytest.mark.gpu

R_MAX = 5.0
PBC = {"TTF": (True, True, False), "TFT": (True, False, True), "FFT": (False, False, True),
       "FFF": (False, False, False), "none": (False, False, False)}
# rc[source, target] of li3po4 (Li, P, O): asymmetric, every entry <= r_max
RC_LI3PO4 = np.array([[3.2, 5.0, 4.1], [3.6, 3.6, 3.6], [2.7, 5.0, 4.4]])
WATER_L2 = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)


def _frame(name, n_side=6, seed=0):
    """li3po4 frame on the tilted cell with periodicity ``name``; "none": the FFF frame without a cell."""
    f = cell_frame("li3po4", n_side, "tilted", seed=seed, outside=True, pbc=PBC[name])
    pos, types = f["pos"].numpy(), f["atom_types"].numpy()
    cell = None if name == "none" else f["cell"].numpy()
    return pos, cell, PBC[name], types


def _rows(out):
    return (out["edge_index"].cpu().numpy(), out["edge_cell_shift"].cpu().numpy(), out["row_ptr"].cpu().numpy(),
            int(out["num_edges"]), int(out["overflow"]))


def _assert_rows(out, ei_x, sh_x, N, pad_shift, what):
    """The padded list ``out`` holds the exact list (ei_x, sh_x) row by row, then null edges (or only null edges on
    overflow)."""
    ei, sh, rp, ne, of = _rows(out)
    cap, E = ei.shape[1], ei_x.shape[1]
    assert ne == E, (what, ne, E)
    assert rp[0] == 0 and rp[N] == cap, what
    rows = np.repeat(np.arange(N), np.diff(rp))
    np.testing.assert_array_equal(ei[0], rows, err_msg=what)
    if E > cap:
        assert of == 1, what
        np.testing.assert_array_equal(rp, (cap * np.arange(N + 1)) // N, err_msg=what)
        real = np.zeros(cap, dtype=bool)
    else:
        assert of == 0, what
        rp_x = np.searchsorted(ei_x[0], np.arange(N + 1))
        nx = np.diff(rp_x)
        assert np.all(np.diff(rp) >= nx), what
        slots = np.repeat(rp[:-1], nx) + (np.arange(E) - np.repeat(rp_x[:-1], nx))
        np.testing.assert_array_equal(ei[:, slots], ei_x, err_msg=what)
        np.testing.assert_array_equal(sh[slots], sh_x, err_msg=what)
        real = np.zeros(cap, dtype=bool)
        real[slots] = True
    np.testing.assert_array_equal(ei[1][~real], ei[0][~real], err_msg=what)
    assert np.all(sh[~real] == pad_shift), what


def _exact(pos, cell, pbc, types=None, rc=None):
    kw = {} if rc is None else dict(atom_types=torch.from_numpy(types), edge_type_cutoff=rc)
    ex = ops.neighbor_list(torch.from_numpy(pos).cuda(), None if cell is None else torch.from_numpy(cell), pbc, R_MAX,
                           **kw)
    return ex["edge_index"].cpu().numpy(), ex["edge_cell_shift"].cpu().numpy()


def _plan(N, cell, pbc, cap, types=None, rc=None):
    kw = {} if rc is None else dict(atom_types=torch.from_numpy(types), edge_type_cutoff=rc)
    return ops.NeighborListPlan(N, None if cell is None else torch.from_numpy(cell), pbc, R_MAX, cap,
                                open_boundaries=True, **kw)


def _assert_bins(plan, pos, cell, pbc, what):
    got = plan._s["cidx"].cpu().numpy()
    want = open_grid.bins(pos, cell, pbc, R_MAX, list(plan._a.nb))
    np.testing.assert_array_equal(got, want, err_msg=what)


# ------------------------------------------------------------------------------------------------------------------
# 1-2. rows and bins
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typed", [False, True])
@pytest.mark.parametrize("name", list(PBC))
def test_plan_rows_match_the_exact_lists(name, typed):
    pos, cell, pbc, types = _frame(name)
    N = pos.shape[0]
    rc = RC_LI3PO4 if typed else None
    ei_x, sh_x = _exact(pos, cell, pbc, types, rc)
    if not typed:
        ei_b, sh_b = brute_list(pos, cell, pbc, R_MAX)
        np.testing.assert_array_equal(ei_x, ei_b)
        np.testing.assert_array_equal(sh_x, sh_b)
    E = ei_x.shape[1]
    assert E > 0
    # real edges have shift 0 along every open direction
    assert np.all(sh_x[:, [d for d in range(3) if not pbc[d]]] == 0)
    for cap in (E, E + 3 * N + 5, E // 2):
        plan = _plan(N, cell, pbc, cap, types, rc)
        if cell is None:
            np.testing.assert_array_equal(plan.cell.cpu().numpy(), np.eye(3))
        assert plan.cell.is_cuda and plan.cell.dtype == torch.float64
        out = plan.run(torch.from_numpy(pos).cuda())
        _assert_rows(out, ei_x, sh_x, N, plan.pad_shift, f"{name} typed={typed} capacity={cap}")
        _assert_bins(plan, pos, cell, pbc, f"{name} capacity={cap}")


def _variants(pos0):
    """Frames of one plan: the frame, translated by 10^3 A, scaled about its centre by 0.3, 3 and 10, and its atoms
    on one line (zero width in two directions)."""
    c = pos0.mean(0)
    N = pos0.shape[0]
    line = np.stack([1.7 * np.arange(N), np.zeros(N), np.zeros(N)], 1) + np.array([0.4, 2.1, -3.3])
    return [("frame", pos0), ("translated", pos0 + np.array([1e3, -1e3, 1e3])), ("x0.3", c + 0.3 * (pos0 - c)),
            ("x3", c + 3.0 * (pos0 - c)), ("x10", c + 10.0 * (pos0 - c)), ("line", line)]


def _captured(plan, static):
    """``plan.run(static)`` captured in a CUDA graph (after a warm-up on a side stream)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        plan.run(static)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = plan.run(static)
    return g, out


@pytest.mark.parametrize("name", ["none", "TTF", "FFT"])
def test_one_plan_follows_moving_shrinking_and_growing_frames(name):
    pos0, cell, pbc, _types = _frame(name)
    N = pos0.shape[0]
    variants = _variants(pos0)
    exact = {v: _exact(p, cell, pbc) for v, p in variants}
    cap = max(e.shape[1] for e, _s in exact.values()) + 2 * N
    perp = 1.0 / np.linalg.norm(np.linalg.inv(np.eye(3) if cell is None else cell), axis=0)
    for v, p in variants:  # the x10 frame needs the most bins the plan has along its open directions
        lo, hi = open_grid.bbox(open_grid.frac_coords(p, cell))
        nbs = [open_grid.open_grid(lo[d], hi[d], perp[d], R_MAX, open_grid.bin_cap(N))[2]
               for d in range(3) if not pbc[d]]
        if v == "x10":
            assert nbs and all(nb == open_grid.bin_cap(N) for nb in nbs), nbs
        if v == "line" and name == "none":
            assert nbs[1:] == [1, 1]
    plan = _plan(N, cell, pbc, cap)
    static = torch.from_numpy(pos0).cuda()
    g, out = _captured(plan, static)
    eager = _plan(N, cell, pbc, cap)
    for rnd in range(2):
        for v, p in (variants if rnd == 0 else variants[::-1]):
            static.copy_(torch.from_numpy(p))
            g.replay()
            torch.cuda.synchronize()
            ei_x, sh_x = exact[v]
            _assert_rows(out, ei_x, sh_x, N, plan.pad_shift, f"{name} {v} replay {rnd}")
            _assert_bins(plan, p, cell, pbc, f"{name} {v} replay {rnd}")
            e = eager.run(torch.from_numpy(p).cuda())
            for k in ("edge_index", "edge_cell_shift", "row_ptr", "num_edges", "overflow"):
                assert torch.equal(e[k], out[k]), (name, v, k)
    # the bounding box work words are left zero by every run
    assert int(plan._bbox_work.abs().sum()) == 0 and int(eager._bbox_work.abs().sum()) == 0


@pytest.mark.parametrize("name", ["none", "TTF"])
def test_single_atom_plan(name):
    _pos, cell, pbc, _types = _frame(name)
    pos = np.array([[0.3, -1.1, 2.5]])
    plan = _plan(1, cell, pbc, 3)
    static = torch.from_numpy(pos).cuda()
    g, out = _captured(plan, static)
    for p in (pos, pos + 1e3, pos * -7.0):
        static.copy_(torch.from_numpy(p))
        g.replay()
        torch.cuda.synchronize()
        ei_x, sh_x = _exact(p, cell, pbc)
        assert ei_x.shape[1] == 0
        _assert_rows(out, ei_x, sh_x, 1, plan.pad_shift, f"{name} N=1")
        _assert_bins(plan, p, cell, pbc, f"{name} N=1")


# ------------------------------------------------------------------------------------------------------------------
# 4. write contracts
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["none", "TTF", "FFT"])
def test_bbox_write_contract(name):
    """nqb_nl_bbox writes the block in place (nothing past it), leaves the periodic part and the trailing fields as
    packed, and leaves its work words zero; the block it writes is the one plan.run uses."""
    pos, cell, pbc, _types = _frame(name)
    N = pos.shape[0]
    plan = _plan(N, cell, pbc, 10)
    L, st = _capi.lib(), torch.cuda.current_stream().cuda_stream
    packed = plan._params_dev.clone()  # as packed on the host: nqb_nl_bbox has not run yet
    nwords = packed.numel() // 8
    block, ck_block = guarded(1, nwords, torch.int64, body=packed.view(torch.int64).view(1, nwords).cpu())
    work, ck_work = guarded(1, 8, torch.int64, body=torch.zeros((1, 8), dtype=torch.int64))
    gpos, ck_pos = guarded(N, 3, torch.float64, body=torch.from_numpy(pos))
    for _ in range(2):  # a second call starts from the work words the first left
        _capi.check(L.nqb_nl_bbox(gpos.data_ptr(), N, block.data_ptr(), work.data_ptr(), st), "nqb_nl_bbox")
        torch.cuda.synchronize()
        ck_block("block")
        ck_work("work")
        ck_pos("pos")
        assert int(work.abs().sum()) == 0
        plan.run(torch.from_numpy(pos).cuda())
        torch.cuda.synchronize()
        assert torch.equal(block.view(-1).view(torch.uint8), plan._params_dev)
    # only the NlParams part changes: pad_shift and the appended fields (last 72 bytes) stay as packed
    changed = np.nonzero(block.view(-1).view(torch.uint8).cpu().numpy() != packed.cpu().numpy())[0]
    assert changed.size > 0 and changed.max() < packed.numel() - 72


# ------------------------------------------------------------------------------------------------------------------
# 5. the graphed step against the eager model
# ------------------------------------------------------------------------------------------------------------------
def _model(names, dtype, ann, table=None, zbl=False):
    pp = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": list(names)} if zbl else None
    m = NequIPEnergyModel(parity=True, r_max=R_MAX, type_names=names, avg_num_neighbors=ann, model_dtype=dtype,
                          pair_potential=pp, per_edge_type_cutoff=table, strict_fast_path=(dtype == torch.float32),
                          **WATER_L2).cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _water_cube():
    """The water_1k frame without its cell (a cube of water in vacuum)."""
    sysd = D.make_system("water", 10, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    ex = {"pos": sysd["pos"].cuda(), "atom_types": sysd["atom_types"].cuda()}
    return ex, meta["type_names"], meta["avg_num_neighbors"]


def _slab():
    """The li3po4 frame of 6^3 atoms on the tilted cell, periodic in x and y, open in z."""
    f = cell_frame("li3po4", 6, "tilted", seed=1, outside=True, pbc=PBC["TTF"])
    meta = f.pop("_meta")
    ex = {"pos": f["pos"].cuda(), "atom_types": f["atom_types"].cuda(), "cell": f["cell"].cuda(),
          "pbc": torch.tensor([[True, True, False]])}
    return ex, meta["type_names"], meta["avg_num_neighbors"]


CASES = {
    # name: (frame, model dtype, deterministic, per-edge-type table, ZBL, capacity = E0 // 2)
    "water_f32": ("water", torch.float32, False, None, False, False),
    "water_f64_det": ("water", torch.float64, True, None, False, False),
    "slab_f32": ("slab", torch.float32, False, None, False, False),
    "water_zbl": ("water", torch.float32, False, None, True, False),
    "water_typed": ("water", torch.float32, False, {"H": 3.1, "O": {"H": 4.2, "O": 4.7}}, False, False),
    "slab_typed_zbl": ("slab", torch.float32, False, {"Li": 3.6, "O": {"Li": 2.9, "O": 4.4}}, True, False),
    "water_recapture": ("water", torch.float32, False, None, False, True),
    "slab_recapture": ("slab", torch.float32, False, None, False, True),
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", list(CASES))
def test_graphed_open_step_matches_eager(case):
    kind, dtype, det, table, zbl, small = CASES[case]
    ex, names, ann = _water_cube() if kind == "water" else _slab()
    model = _model(names, dtype, ann, table, zbl)
    cell, pbc = ex.get("cell"), tuple(bool(b) for b in ex.get("pbc", torch.zeros(3, dtype=torch.bool)).view(-1))
    et = {} if table is None else dict(atom_types=ex["atom_types"], edge_type_cutoff=model.per_edge_type_cutoff)
    E0 = ops.neighbor_list(ex["pos"], cell, pbc, R_MAX, **et)["edge_index"].shape[1]
    prev = ops.deterministic()
    ops.set_deterministic(det)
    try:
        g = GraphedMDStep(model, ex, capacity=E0 // 2 if small else None)
        assert torch.equal(g.static["cell"], g.plan.cell)
        if cell is None:
            np.testing.assert_array_equal(g.plan.cell.cpu().numpy(), np.eye(3))
        pos0 = ex["pos"].clone()
        drift = torch.tensor([0.013, -0.007, 0.021], dtype=torch.float64, device="cuda")
        for t in range(100):
            pos = D.oscillating_positions(pos0, t, period=50, seed=7) + t * drift
            out = {k: v.clone() for k, v in g(pos).items()}
            nl = ops.neighbor_list(pos, cell, pbc, R_MAX, **et)
            d = {"pos": pos, "atom_types": ex["atom_types"], "edge_index": nl["edge_index"]}
            if cell is not None:
                d.update(cell=cell, edge_cell_shift=nl["edge_cell_shift"])
            ref = model(d)
            assert int(out["num_edges"]) == nl["edge_index"].shape[1], t
            assert torch.equal(out["total_energy"], ref["total_energy"]), (t, float(out["total_energy"]),
                                                                          float(ref["total_energy"]))
            assert torch.equal(out["atomic_energy"], ref["atomic_energy"]), t
            fs = float(ref["forces"].abs().max())
            df = float((out["forces"] - ref["forces"]).abs().max())
            assert df <= (1e-12 if det else 2e-6) * fs, (t, df / fs)
        if small:
            assert g.recaptures >= 1 and g.capacity > E0 // 2
        else:
            assert g.recaptures == 0
        # a replay launches nothing eagerly: the bounding box is part of the graph
        n0 = _capi.launch_count()
        g(pos)
        assert _capi.launch_count() == n0
    finally:
        ops.set_deterministic(prev)


# ------------------------------------------------------------------------------------------------------------------
# 6. the periodic path
# ------------------------------------------------------------------------------------------------------------------
def test_periodic_step_calls_no_open_entry_point(monkeypatch):
    sysd = cell_frame("li3po4", 4, "tilted", seed=2, outside=True)
    meta = sysd.pop("_meta")
    dev = D.to_device(sysd, "cuda")
    model = _model(meta["type_names"], torch.float32, meta["avg_num_neighbors"])
    L = _capi.lib()
    calls = []
    for name in ("nqb_nl_bbox", "nqb_nl_params_pack_open"):
        def boom(*a, _n=name, **k):
            calls.append(_n)
            raise AssertionError(f"{_n} called")
        monkeypatch.setattr(L, name, boom)
    g = GraphedMDStep(model, dev)
    g(dev["pos"])
    GraphedMDStep(model, dict(dev, pbc=torch.tensor([True, True, True])))(dev["pos"])
    GraphedMDStep(model, dev, variable_cell=True)(dev["pos"], dev["cell"])
    ops.NeighborListPlan(dev["pos"].shape[0], dev["cell"], True, R_MAX, 5000).run(dev["pos"])
    ops.NeighborListPlan(dev["pos"].shape[0], dev["cell"], True, R_MAX, 5000, open_boundaries=True).run(dev["pos"])
    assert calls == []
