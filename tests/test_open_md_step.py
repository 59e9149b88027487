"""Open boundary directions of the capturable neighbour list (ops.NeighborListPlan(open_boundaries=True)) and of
graph.GraphedMDStep, on the host: argument checks, the device grid formula restated, the packed parameter block
(nqb_nl_params_pack_open) and, on the float64 oracle, that a cell-less frame with the identity as its cell, zero
shifts and null edges gives the energy and forces of the frame without a cell."""
import ctypes

import numpy as np
import pytest
import torch

import open_grid
from cell_frames import brute_list
from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel
from oracle import pair as opair

R_MAX = 5.0
CELL = torch.eye(3, dtype=torch.float64) * 12.0
ZBL = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal"}


# ------------------------------------------------------------------------------------------------------------------
# argument checks
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pbc", [(True, True, False), (False, True, True), False, (True, False, True)])
def test_plan_without_the_opt_in_still_rejects_open_directions(pbc):
    with pytest.raises(ValueError):
        ops.NeighborListPlan(10, CELL, pbc, R_MAX, 100)
    with pytest.raises(ValueError):
        ops.NeighborListPlan(10, None, pbc, R_MAX, 100)


@pytest.mark.parametrize("pbc", [True, (True, True, False), (False, False, True)])
def test_open_plan_without_a_cell_needs_every_direction_open(pbc):
    with pytest.raises(ValueError, match="periodic direction needs a cell"):
        ops.NeighborListPlan(10, None, pbc, R_MAX, 100, open_boundaries=True)


def test_open_plan_rejects_variable_cell_and_bad_cells():
    with pytest.raises(ValueError, match="variable_cell"):
        ops.NeighborListPlan(10, CELL, (True, True, False), R_MAX, 100, variable_cell=True, open_boundaries=True)
    with pytest.raises(ValueError, match="variable_cell"):
        ops.NeighborListPlan(10, None, False, R_MAX, 100, variable_cell=True, open_boundaries=True)
    singular = torch.tensor([[10.0, 0.0, 0.0], [0.0, 10.0, 0.0], [5.0, 5.0, 0.0]], dtype=torch.float64)
    for pbc in [(True, True, False), True, False]:
        with pytest.raises(ValueError, match="singular"):
            ops.NeighborListPlan(10, singular, pbc, R_MAX, 100, open_boundaries=True)
    with pytest.raises(ValueError, match="not finite"):
        ops.NeighborListPlan(10, CELL * float("nan"), (True, True, False), R_MAX, 100, open_boundaries=True)
    with pytest.raises(ValueError):
        ops.NeighborListPlan(10, CELL, (True, False), R_MAX, 100, open_boundaries=True)
    with pytest.raises(ValueError):
        ops.NeighborListPlan(0, None, False, R_MAX, 100, open_boundaries=True)


def test_graphed_md_step_checks_periodicity_before_anything_else():
    pos = torch.zeros((4, 3), dtype=torch.float64)
    types = torch.zeros(4, dtype=torch.int64)
    model = None  # never reached
    with pytest.raises(ValueError, match="needs a cell"):
        GraphedMDStep(model, {"pos": pos, "atom_types": types, "pbc": torch.tensor([True, True, False])})
    with pytest.raises(ValueError, match="variable_cell"):
        GraphedMDStep(model, {"pos": pos, "atom_types": types}, variable_cell=True)
    with pytest.raises(ValueError, match="variable_cell"):
        GraphedMDStep(model, {"pos": pos, "atom_types": types, "cell": CELL,
                              "pbc": torch.tensor([[True, True, False]])}, variable_cell=True)
    with pytest.raises(ValueError, match="3 flags"):
        GraphedMDStep(model, {"pos": pos, "atom_types": types, "cell": CELL, "pbc": torch.tensor([True, False])})
    # no CPU path
    with pytest.raises(RuntimeError):
        GraphedMDStep(model, {"pos": pos, "atom_types": types})


def test_periodicity_of_an_example():
    per = GraphedMDStep._periodicity
    assert per({"cell": CELL}) == (True, True, True)
    assert per({}) == (False, False, False)
    assert per({"cell": CELL, "pbc": torch.tensor([[True, True, False]])}) == (True, True, False)
    assert per({"cell": CELL, "pbc": torch.tensor([False, True, True])}) == (False, True, True)
    assert per({"cell": CELL, "pbc": False}) == (False, False, False)


# ------------------------------------------------------------------------------------------------------------------
# the device grid, restated
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_atoms", [1, 2, 21, 1000, 10648])
def test_open_grid_stays_within_one_and_cap(n_atoms):
    cap = open_grid.bin_cap(n_atoms)
    assert cap == ops._nl_bin_cap(n_atoms)
    inf, nan = float("inf"), float("nan")
    extents = [(0.0, 0.0), (1.0, 1.0), (-3.0, 5.0), (0.0, 1e-300), (-1e300, 1e300), (0.0, 1e308), (-inf, inf),
               (0.0, inf), (-inf, 0.0), (inf, -inf), (nan, nan), (0.0, nan), (nan, 1.0), (5.0, -5.0)]
    for perp in (1.0, 12.3, 1e-12, 1e300):
        for fmin, fmax in extents:
            _lo, width, nb = open_grid.open_grid(fmin, fmax, perp, R_MAX, cap)
            assert 1 <= nb <= cap, (fmin, fmax, perp, nb)
            assert width >= 1e-9, (fmin, fmax, width)
    # the formula of ops.neighbor_list on a regular extent: floor(perp * width / r_max) bins, each >= r_max wide
    _lo, width, nb = open_grid.open_grid(-0.5, 2.5, 10.0, R_MAX, 100)
    assert nb == 6 and 10.0 * width / nb >= R_MAX
    # huge extents give cap bins, zero and NaN extents one
    assert open_grid.open_grid(0.0, 1e300, 1.0, R_MAX, cap)[2] == cap
    assert open_grid.open_grid(0.0, 0.0, 1.0, R_MAX, cap)[2] == 1
    assert open_grid.open_grid(nan, nan, 1.0, R_MAX, cap)[2] == 1


def test_restated_bins_match_the_host_grid_of_neighbor_list():
    """On a frame where the host and device boxes agree, the restated grid is the one ops.neighbor_list builds."""
    rng = np.random.default_rng(3)
    pos = rng.uniform(-4.0, 17.0, (300, 3))
    pbc, cell_np, inv_np = ops._nl_cell(None, False)
    frac = open_grid.frac_coords(pos, None)
    lo, hi = open_grid.bbox(frac)
    width = np.array([max(hi[d] - lo[d], 1e-9) * (1 + 1e-9) for d in range(3)])
    a = ops._NlArgs(300, cell_np, inv_np, pbc, R_MAX, lo, width)
    for d in range(3):
        l0, w, nb = open_grid.open_grid(lo[d], hi[d], 1.0, R_MAX, open_grid.bin_cap(300))
        assert (l0, w, nb) == (lo[d], width[d], a.nb[d])


# ------------------------------------------------------------------------------------------------------------------
# the packed block
# ------------------------------------------------------------------------------------------------------------------
def _pack_args(cell_np, pbc, nb=(3, 4, 5)):
    inv = np.linalg.inv(cell_np)
    D9, D3, I3 = ctypes.c_double * 9, ctypes.c_double * 3, ctypes.c_int * 3
    return (D9(*cell_np.reshape(-1)), D9(*inv.reshape(-1)), I3(*[int(b) for b in pbc]), I3(*nb), I3(1, 1, 2), R_MAX,
            D3(7.0, 0.0, 0.0))


def test_pack_open_writes_the_whole_block_and_nothing_else():
    L = _capi.lib()
    nbytes = int(L.nqb_nl_params_bytes())
    assert nbytes % 8 == 0
    cell = np.array([[11.0, 0.0, 0.0], [3.0, 10.0, 0.0], [-2.0, 1.5, 12.0]])
    perp = (ctypes.c_double * 3)(*(1.0 / np.linalg.norm(np.linalg.inv(cell), axis=0)))
    out, check = guarded(1, nbytes // 8, torch.int64, device="cpu")
    _capi.check(L.nqb_nl_params_pack_open(*_pack_args(cell, (True, True, False)), 12, perp, out.data_ptr()))
    check("block")
    assert not bool(is_poison(out).any())


def test_pack_open_agrees_with_pack_on_periodic_directions():
    """With every direction periodic the block starts with the bytes of nqb_nl_params_pack (the parameters and the
    null-edge shift the existing kernels read)."""
    L = _capi.lib()
    nbytes = int(L.nqb_nl_params_bytes())
    cell = np.array([[11.0, 0.0, 0.0], [3.0, 10.0, 0.0], [-2.0, 1.5, 12.0]])
    perp = (ctypes.c_double * 3)(1.0, 2.0, 3.0)
    a, b = ctypes.create_string_buffer(nbytes), ctypes.create_string_buffer(nbytes)
    _capi.check(L.nqb_nl_params_pack(*_pack_args(cell, (True,) * 3), a))
    _capi.check(L.nqb_nl_params_pack_open(*_pack_args(cell, (True,) * 3), 9, perp, b))
    # the appended open-direction fields follow pad_shift: compare everything up to them
    a_raw, b_raw = a.raw, b.raw
    assert a_raw != b_raw
    prefix = next(k for k in range(nbytes) if a_raw[k] != b_raw[k])
    assert prefix >= nbytes - 48, prefix  # open[3] + cap, perp[3], r_max
    # an open direction differs from the periodic pack
    c = ctypes.create_string_buffer(nbytes)
    _capi.check(L.nqb_nl_params_pack_open(*_pack_args(cell, (True, True, False)), 9, perp, c))
    assert c.raw[:prefix] != b_raw[:prefix]


def test_pack_open_rejects_bad_arguments():
    L = _capi.lib()
    buf = ctypes.create_string_buffer(int(L.nqb_nl_params_bytes()))
    cell = np.diag([10.0, 11.0, 12.0])
    good = (ctypes.c_double * 3)(10.0, 11.0, 12.0)
    assert L.nqb_nl_params_pack_open(*_pack_args(cell, (True, False, False)), 5, good, buf) == 0
    for cap in (0, -3):
        assert L.nqb_nl_params_pack_open(*_pack_args(cell, (True, False, False)), cap, good, buf) != 0
    for bad in ((0.0, 1.0, 1.0), (1.0, -1.0, 1.0), (1.0, 1.0, float("nan")), (float("inf"), 1.0, 1.0)):
        assert L.nqb_nl_params_pack_open(*_pack_args(cell, (True, False, False)), 5, (ctypes.c_double * 3)(*bad),
                                         buf) != 0
    # a periodic direction still needs a valid grid
    assert L.nqb_nl_params_pack_open(*_pack_args(cell, (True, False, False), nb=(0, 1, 1)), 5, good, buf) != 0
    # the fixed-cell pack keeps rejecting open directions
    assert L.nqb_nl_params_pack(*_pack_args(cell, (True, False, False)), buf) != 0


# ------------------------------------------------------------------------------------------------------------------
# the identity cell on the oracle
# ------------------------------------------------------------------------------------------------------------------
def _cluster(n_side: int, seed: int):
    sysd = D.make_system("water", n_side, r_max=R_MAX, seed=seed)
    meta = sysd.pop("_meta")
    pos = sysd["pos"].numpy()
    ei, sh = brute_list(pos, None, False, R_MAX)
    assert np.all(sh == 0)
    frame = {"pos": torch.from_numpy(pos.copy()), "atom_types": sysd["atom_types"],
             "edge_index": torch.from_numpy(ei)}
    return frame, meta["type_names"]


@pytest.mark.parametrize("n_side,pair", [(3, False), (4, False), (4, True)])
def test_identity_cell_with_null_edges_changes_nothing_on_the_oracle(n_side, pair):
    frame, type_names = _cluster(n_side, seed=n_side)
    N, E = frame["pos"].shape[0], frame["edge_index"].shape[1]
    kw = dict(pair_potential=dict(ZBL, chemical_species=list(type_names))) if pair else {}
    model = NequIPEnergyModel(r_max=R_MAX, type_names=type_names, parity=True, l_max=2, num_layers=3,
                              num_features=16, radial_mlp_depth=1, radial_mlp_width=16, avg_num_neighbors=E / N,
                              model_dtype=torch.float64, **kw)
    oracle = opair if pair else omodel
    pad_shift = ops.null_edge_shift(np.eye(3), R_MAX)
    assert pad_shift.tolist() == [7.0, 0.0, 0.0]  # 7 Angstrom > r_max + |a_0| in the identity cell
    rng = np.random.default_rng(5)
    extra = rng.integers(0, 4, N)
    ei = frame["edge_index"].numpy()
    rows, shs = [], []
    for i in range(N):
        sel = ei[0] == i
        rows.append(np.concatenate([ei[:, sel], np.full((2, extra[i]), i, dtype=np.int64)], 1))
        shs.append(np.concatenate([np.zeros((int(sel.sum()), 3)), np.tile(pad_shift, (extra[i], 1))], 0))
    assert extra.sum() > 0
    padded = dict(frame, edge_index=torch.from_numpy(np.concatenate(rows, 1)),
                  edge_cell_shift=torch.from_numpy(np.concatenate(shs, 0)), cell=torch.eye(3, dtype=torch.float64))
    e0, ea0, f0 = oracle.energy_and_forces(model.state_dict(), model.config, frame, torch.float64)
    e1, ea1, f1 = oracle.energy_and_forces(model.state_dict(), model.config, padded, torch.float64)
    assert float(f0.abs().max()) > 0
    assert abs(float(e1) - float(e0)) <= 1e-13 * float(ea0.abs().sum())
    assert float((ea1 - ea0).abs().max()) <= 1e-13 * float(ea0.abs().max())
    assert float((f1 - f0).abs().max()) <= 1e-13 * float(f0.abs().max())
