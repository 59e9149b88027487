"""Variable-cell neighbour list (ops.NeighborListPlan(variable_cell=True).set_cell) on the host: the packed parameter
block of every cell on a fixed bin grid, the per-cell null-edge shift, and on the float64 oracle that null edges with
that shift leave energy, forces, stress and virial unchanged on strained triclinic cells."""
import ctypes

import numpy as np
import pytest
import torch

from cell_frames import brute_list
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel

R_MAX = 5.0
N_ATOMS = 1000
CELL0 = np.diag([22.0, 21.0, 23.0])


def _variants(cell0):
    """cell0 and strained, sheared, triclinic and shorter-than-r_max versions of it."""
    sheared = cell0 @ np.array([[1.0, 0.03, 0.0], [0.03, 1.0, -0.02], [0.0, -0.02, 1.0]])
    return {
        "cell0": cell0,
        "expanded": cell0 * 1.03,
        "compressed": cell0 * 0.97,
        "strained": cell0 @ np.diag([1.02, 0.98, 1.01]),
        "sheared": sheared,
        "triclinic": cell0 @ np.array([[1.0, 0.0, 0.0], [0.25, 1.0, 0.0], [-0.15, 0.1, 1.0]]),
        "oscillating": cell0 @ D.oscillating_strain(13).numpy(),
        "sub_r_max": np.array([[4.6, 0.0, 0.0], [0.7, 4.2, 0.0], [-0.3, 0.5, 4.4]]),
    }


def _grid(cell, n=N_ATOMS):
    _, cell_np, inv_np = ops._nl_cell(cell, True)
    return tuple(ops._NlArgs(n, cell_np, inv_np, [True] * 3, R_MAX, np.zeros(3), np.ones(3)).nb)


@pytest.mark.parametrize("name", list(_variants(CELL0)))
def test_packed_block_of_each_cell_on_the_fixed_grid(name):
    nb = _grid(CELL0)
    assert min(nb) > 1
    cell = _variants(CELL0)[name]
    a, pad_shift, block = ops._nl_cell_block(torch.from_numpy(cell), R_MAX, nb, N_ATOMS)
    assert tuple(a.nb) == nb, "the bin grid must stay the construction cell's"
    # the search range covers the cutoff on this grid for this cell
    perp = 1.0 / np.linalg.norm(np.linalg.inv(cell), axis=0)
    for d in range(3):
        assert a.sr[d] * perp[d] / nb[d] >= R_MAX, (d, a.sr[d], perp[d], nb[d])
    # the null shift reaches past the cutoff of THIS cell
    lengths = np.linalg.norm(cell, axis=1)
    d = int(np.argmax(lengths))
    np.testing.assert_array_equal(pad_shift, ops.null_edge_shift(cell, R_MAX))
    assert np.linalg.norm(pad_shift @ cell) >= R_MAX + lengths[d]
    # the block holds exactly the by-value arguments: _NlArgs with that grid, neighbor_list's inverse, that shift
    _, cell_np, inv_np = ops._nl_cell(torch.from_numpy(cell), True)
    np.testing.assert_array_equal(inv_np, np.linalg.inv(cell))
    ref = ops._NlArgs(N_ATOMS, cell_np, inv_np, [True] * 3, R_MAX, np.zeros(3), np.ones(3), nb=nb)
    assert list(ref.sr) == list(a.sr)
    L = _capi.lib()
    nbytes = int(L.nqb_nl_params_bytes())
    assert len(block) == nbytes
    want = ctypes.create_string_buffer(nbytes)
    _capi.check(L.nqb_nl_params_pack(ref.cell, ref.inv, ref.pbc, ref.nb, ref.sr, ref.r_max,
                                     (ctypes.c_double * 3)(*pad_shift), want))
    assert block.raw == want.raw
    # and a different search range or shift gives a different block
    for sr, sh in (([s + 1 for s in ref.sr], pad_shift), (list(ref.sr), pad_shift + 1)):
        other = ctypes.create_string_buffer(nbytes)
        _capi.check(L.nqb_nl_params_pack(ref.cell, ref.inv, ref.pbc, ref.nb, (ctypes.c_int * 3)(*sr), ref.r_max,
                                         (ctypes.c_double * 3)(*sh), other))
        assert other.raw != want.raw


def test_frozen_shift_would_fall_inside_the_cutoff():
    """Why the shift follows the cell: the shift of a long cell is too short once the cell has shrunk."""
    long_cell, short = np.diag([11.0, 10.5, 10.8]), np.diag([2.4, 2.3, 2.35])
    frozen = ops.null_edge_shift(long_cell, R_MAX)
    assert np.linalg.norm(frozen @ short) < R_MAX
    assert np.linalg.norm(ops.null_edge_shift(short, R_MAX) @ short) >= R_MAX + np.linalg.norm(short, axis=1).max()


def test_pack_rejects_open_directions_and_bad_grids():
    _, cell_np, inv_np = ops._nl_cell(CELL0, True)
    a = ops._NlArgs(10, cell_np, inv_np, [True] * 3, R_MAX, np.zeros(3), np.ones(3))
    L = _capi.lib()
    out = ctypes.create_string_buffer(int(L.nqb_nl_params_bytes()))
    I3, D3 = ctypes.c_int * 3, ctypes.c_double * 3
    assert L.nqb_nl_params_pack(a.cell, a.inv, I3(1, 0, 1), a.nb, a.sr, a.r_max, D3(0, 0, 3), out) != 0
    assert L.nqb_nl_params_pack(a.cell, a.inv, a.pbc, I3(0, 1, 1), a.sr, a.r_max, D3(0, 0, 3), out) != 0
    assert L.nqb_nl_params_pack(a.cell, a.inv, a.pbc, a.nb, I3(1, -1, 1), a.r_max, D3(0, 0, 3), out) != 0
    assert L.nqb_nl_params_pack(a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max, D3(0, 0, 3), out) == 0


# ------------------------------------------------------------------------------------------------------------------
# null edges with the per-cell shift on the float64 oracle, stress and virial included
# ------------------------------------------------------------------------------------------------------------------
def _pad_rows(ei, sh, n_atoms, pad_shift, seed):
    rng = np.random.default_rng(seed)
    extra = rng.integers(0, 4, n_atoms)
    rows, shs = [], []
    for i in range(n_atoms):
        sel = ei[0] == i
        rows.append(np.concatenate([ei[:, sel], np.full((2, extra[i]), i, dtype=np.int64)], 1))
        shs.append(np.concatenate([sh[sel], np.tile(pad_shift, (extra[i], 1))], 0))
    return np.concatenate(rows, 1), np.concatenate(shs, 0), int(extra.sum())


def _strained_frames():
    sysd = D.make_system("li3po4", 4, r_max=R_MAX, seed=1)
    meta = sysd.pop("_meta")
    pos0, cell0 = sysd["pos"].numpy(), sysd["cell"].numpy()
    frames = []
    for t in (7, 19, 31):
        S = D.oscillating_strain(t).numpy()
        frames.append((pos0 @ S, cell0 @ S, sysd["atom_types"]))
    # shrunk below r_max and sheared: several images of each neighbour, k = 3
    rng = np.random.default_rng(4)
    small = np.array([[3.7, 0.0, 0.0], [0.6, 4.1, 0.0], [-0.4, 0.3, 3.9]])
    frames.append((rng.uniform(0, 1, (11, 3)) @ small, small, torch.from_numpy(rng.integers(0, 2, 11))))
    return frames, meta


def test_null_edges_change_nothing_on_the_oracle_with_stress():
    frames, meta = _strained_frames()
    for pos, cell, types in frames:
        assert np.count_nonzero(cell - np.diag(np.diagonal(cell))) > 0, "the frames are triclinic"
        N = pos.shape[0]
        ei, sh = brute_list(pos, cell, True, R_MAX)
        type_names = meta["type_names"] if int(types.max()) >= 2 else ["H", "O"]
        model = NequIPEnergyModel(r_max=R_MAX, type_names=type_names, parity=True, l_max=2, num_layers=3,
                                  num_features=16, radial_mlp_depth=1, radial_mlp_width=16,
                                  avg_num_neighbors=ei.shape[1] / N, model_dtype=torch.float64)
        pad_shift = ops.null_edge_shift(cell, R_MAX)
        assert np.linalg.norm(pad_shift @ cell) >= R_MAX + np.linalg.norm(cell, axis=1).max()
        pei, psh, added = _pad_rows(ei, sh, N, pad_shift, seed=N)
        assert added > 0
        base = {"pos": torch.from_numpy(pos), "cell": torch.from_numpy(cell), "atom_types": types}
        exact = dict(base, edge_index=torch.from_numpy(ei), edge_cell_shift=torch.from_numpy(sh))
        padded = dict(base, edge_index=torch.from_numpy(pei), edge_cell_shift=torch.from_numpy(psh))
        e0, f0, s0, v0 = omodel.energy_forces_stress(model.state_dict(), model.config, exact, torch.float64)
        e1, f1, s1, v1 = omodel.energy_forces_stress(model.state_dict(), model.config, padded, torch.float64)
        assert float(f0.abs().max()) > 0 and float(s0.abs().max()) > 0
        assert abs(float(e1) - float(e0)) <= 1e-13 * abs(float(e0))
        assert float((f1 - f0).abs().max()) <= 1e-13 * float(f0.abs().max())
        assert float((s1 - s0).abs().max()) <= 1e-13 * float(s0.abs().max())
        assert float((v1 - v0).abs().max()) <= 1e-13 * float(v0.abs().max())


# ------------------------------------------------------------------------------------------------------------------
# set_cell's argument checks
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cell", [
    np.eye(2) * 10.0,  # wrong shape
    np.ones(9) * 10.0,
    np.diag([10.0, np.nan, 10.0]),  # not finite
    np.diag([10.0, np.inf, 10.0]),
    np.array([[10.0, 0.0, 0.0], [0.0, 10.0, 0.0], [10.0, 10.0, 0.0]]),  # singular
    np.array([[10.0, 0.0, 0.0], [20.0, 1e-14, 0.0], [0.0, 0.0, 10.0]]),  # numerically singular
])
def test_set_cell_rejects_bad_cells(cell):
    with pytest.raises(ValueError):
        ops._nl_cell_block(cell, R_MAX, (3, 3, 3), 100)
    with pytest.raises(ValueError):
        ops._nl_cell_block(torch.from_numpy(np.asarray(cell)), R_MAX, (3, 3, 3), 100)


def test_set_cell_needs_a_variable_cell_plan():
    plan = ops.NeighborListPlan(10, torch.from_numpy(CELL0), True, R_MAX, 100, device="cpu")
    assert not plan.variable_cell
    with pytest.raises(ValueError):
        plan.set_cell(CELL0 * 1.01)
    # [1, 3, 3] is accepted like [3, 3]
    a1, s1, b1 = ops._nl_cell_block(CELL0[None], R_MAX, (3, 3, 3), 100)
    a2, s2, b2 = ops._nl_cell_block(CELL0, R_MAX, (3, 3, 3), 100)
    assert b1.raw == b2.raw
