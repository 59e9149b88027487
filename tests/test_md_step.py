"""Null edges of the capacity-mode neighbour list (ops.NeighborListPlan, graph.GraphedMDStep): on the CPU oracle, a
list padded with (i, i, pad_shift) edges gives the energy and forces of the exact list, and the plan's argument checks."""
import numpy as np
import pytest
import torch

from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel

R_MAX = 5.0


def _pad_rows(edge_index, shifts, n_atoms, pad_shift, seed):
    """The list with 0..3 null edges appended to the end of every row (random counts, some rows without)."""
    rng = np.random.default_rng(seed)
    extra = rng.integers(0, 4, n_atoms)
    ei, sh = edge_index.numpy(), shifts.numpy()
    rows, shs = [], []
    for i in range(n_atoms):
        sel = ei[0] == i
        rows.append(np.concatenate([ei[:, sel], np.full((2, extra[i]), i, dtype=np.int64)], 1))
        shs.append(np.concatenate([sh[sel], np.tile(pad_shift, (extra[i], 1))], 0))
    return torch.from_numpy(np.concatenate(rows, 1)), torch.from_numpy(np.concatenate(shs, 0)), int(extra.sum())


def _small_cell_frame():
    """11 atoms in a cell shorter than r_max along every direction: k = floor(r_max / |a|) + 2 = 3."""
    rng = np.random.default_rng(4)
    cell = np.diag([3.6, 4.2, 3.9])
    pos = rng.uniform(0, 1, (11, 3)) @ cell
    ei, sh = D.neighbor_list(pos, cell, R_MAX)
    types = rng.integers(0, 2, 11)
    return {"pos": torch.from_numpy(pos), "cell": torch.from_numpy(cell), "atom_types": torch.from_numpy(types),
            "edge_index": torch.from_numpy(ei), "edge_cell_shift": torch.from_numpy(sh)}, ["H", "O"]


def _frame(kind):
    if kind == "small":
        return _small_cell_frame()
    sysd = D.make_system(kind, 4, r_max=R_MAX, seed=1)
    meta = sysd.pop("_meta")
    return sysd, meta["type_names"]


@pytest.mark.parametrize("kind", ["li3po4", "water", "small"])
def test_null_edges_change_nothing_on_the_oracle(kind):
    sysd, type_names = _frame(kind)
    N = sysd["pos"].shape[0]
    model = NequIPEnergyModel(r_max=R_MAX, type_names=type_names, parity=True, l_max=2, num_layers=3, num_features=16,
                              radial_mlp_depth=1, radial_mlp_width=16,
                              avg_num_neighbors=sysd["edge_index"].shape[1] / N, model_dtype=torch.float64)
    pad_shift = ops.null_edge_shift(sysd["cell"], R_MAX)
    if kind == "small":
        assert pad_shift.max() == 3
    ei, sh, added = _pad_rows(sysd["edge_index"], sysd["edge_cell_shift"], N, pad_shift, seed=5)
    assert added > 0
    padded = dict(sysd, edge_index=ei, edge_cell_shift=sh)
    e0, ea0, f0 = omodel.energy_and_forces(model.state_dict(), model.config, sysd, torch.float64)
    e1, ea1, f1 = omodel.energy_and_forces(model.state_dict(), model.config, padded, torch.float64)
    assert float(f0.abs().max()) > 0
    assert abs(float(e1) - float(e0)) <= 1e-13 * float(ea0.abs().sum())
    assert float((ea1 - ea0).abs().max()) <= 1e-13 * float(ea0.abs().max())
    assert float((f1 - f0).abs().max()) <= 1e-13 * float(f0.abs().max())


@pytest.mark.parametrize("cell", [
    np.diag([20.0, 21.0, 19.5]),  # orthorhombic, longer than r_max
    np.array([[11.0, 0.0, 0.0], [3.0, 10.0, 0.0], [-2.0, 1.5, 12.0]]),  # triclinic
    np.diag([3.0, 3.3, 2.7]),  # every lattice vector shorter than r_max
    np.array([[2.0, 0.0, 0.0], [1.9, 0.8, 0.0], [0.3, 0.2, 1.1]]),  # small and triclinic
])
def test_null_edge_shift_reaches_past_the_cutoff(cell):
    shift = ops.null_edge_shift(torch.from_numpy(cell), R_MAX)
    lengths = np.linalg.norm(cell, axis=1)
    d = int(np.argmax(lengths))
    assert np.count_nonzero(shift) == 1 and shift[d] == np.floor(R_MAX / lengths[d]) + 2
    assert np.all(shift == np.round(shift))
    length = float(np.linalg.norm(shift @ cell))
    assert length >= R_MAX + lengths[d] > R_MAX


def test_plan_rejects_missing_cell_and_open_directions():
    cell = torch.eye(3, dtype=torch.float64) * 12.0
    with pytest.raises(ValueError):
        ops.NeighborListPlan(10, None, True, R_MAX, 100)
    for pbc in [(True, True, False), (False, True, True), False, (True, False, True)]:
        with pytest.raises(ValueError):
            ops.NeighborListPlan(10, cell, pbc, R_MAX, 100)
    with pytest.raises(ValueError):
        ops.NeighborListPlan(0, cell, True, R_MAX, 100)
