"""The shared cell helpers of tests/cell_frames.py, pinned on the host before the GPU tests rely on them: the brute-force
list equals the host list of nequip_b200/data.py wherever that one applies, does not depend on the choice of cell
basis, and the float64 oracle's stress on triclinic and left-handed cells is the strain derivative of its energy."""
import numpy as np
import pytest
import torch

from cell_frames import CELL_SHAPES, brute_list, cell_frame, named_cell, perp_widths
from nequip_b200 import data as D
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel

R_MAX = 5.0


def test_named_cells():
    assert np.linalg.det(named_cell("left", 6)) < 0
    for name in ("tilted", "skewed", "small", "cubic"):
        assert np.linalg.det(named_cell(name, 6)) > 0
    skew = CELL_SHAPES["skewed"]
    assert max(abs(skew[1, 0]), abs(skew[2, 0]), abs(skew[2, 1])) >= 0.5
    assert perp_widths(named_cell("small", 2)).max() < R_MAX
    assert perp_widths(named_cell("tilted", 6)).min() > R_MAX


def _orthorhombic_cases():
    rng = np.random.default_rng(0)
    pos8, cell8 = D.jittered_lattice(8, D.PRESETS["li3po4"]["density"], seed=3)  # the host cell-list path
    pos5, cell5 = D.jittered_lattice(5, D.PRESETS["water"]["density"], seed=4)  # the host brute force
    small = np.diag([3.0, 3.3, 2.7])  # r_max > L: several images of each neighbour
    slab = np.diag([9.0, 8.5, 9.5])
    return {
        "cell_list": (pos8, cell8, True),
        "cell_list_outside": (pos8 + np.array([3.7, -11.2, 0.4]), cell8, True),
        "brute_outside": (pos5 - np.array([0.0, 13.1, 2.2]), cell5, True),
        "small": (rng.uniform(0, 1, (11, 3)) @ small + np.array([0.0, 4.0, -3.5]), small, True),
        "open": (rng.uniform(-3, 11, (150, 3)), None, False),
        "TTF": (rng.uniform(-4, 12, (160, 3)), slab, (True, True, False)),
        "TFT": (rng.uniform(-4, 12, (160, 3)), slab, (True, False, True)),
        "FFT": (rng.uniform(-4, 12, (160, 3)), slab, (False, False, True)),
    }


@pytest.mark.parametrize("case", list(_orthorhombic_cases()))
def test_brute_list_equals_host_list_on_orthorhombic_cells(case):
    pos, cell, pbc = _orthorhombic_cases()[case]
    ei_ref, sh_ref = D.neighbor_list(pos, cell, R_MAX, pbc=pbc)
    ei, sh = brute_list(pos, cell, pbc, R_MAX)
    assert ei.shape[1] > 0
    np.testing.assert_array_equal(ei, ei_ref)
    np.testing.assert_array_equal(sh, sh_ref)


def _edge_vectors(pos, cell, ei, sh):
    """(i, j, vector) rows in a canonical order (vectors rounded only for the ordering)."""
    vec = pos[ei[1]] - pos[ei[0]] + sh @ cell
    r = np.round(vec, 6)
    o = np.lexsort((r[:, 2], r[:, 1], r[:, 0], ei[1], ei[0]))
    return ei[:, o], vec[o]


@pytest.mark.parametrize("name,n_side", [("tilted", 5), ("skewed", 5), ("small", 2)])
@pytest.mark.parametrize("U", [
    [[1, 1, 0], [0, 1, 0], [0, -1, 1]],  # det +1
    [[0, 1, 0], [1, 0, 1], [0, 0, 1]],  # det -1
])
def test_brute_list_does_not_depend_on_the_basis(name, n_side, U):
    U = np.array(U, dtype=np.float64)
    assert abs(abs(np.linalg.det(U)) - 1.0) < 1e-12
    f = cell_frame("water", n_side, name, seed=1, outside=True)
    pos, cell = f["pos"].numpy(), f["cell"].numpy()
    cell2 = U @ cell
    frac2 = pos @ np.linalg.inv(cell2)
    pos2 = (frac2 - np.floor(frac2)) @ cell2  # re-wrapped into the new cell
    ei_a, v_a = _edge_vectors(pos, cell, f["edge_index"].numpy(), f["edge_cell_shift"].numpy())
    ei_b, v_b = _edge_vectors(pos2, cell2, *brute_list(pos2, cell2, True, R_MAX))
    np.testing.assert_array_equal(ei_b, ei_a)
    np.testing.assert_allclose(v_b, v_a, rtol=0, atol=1e-11)


@pytest.mark.parametrize("name", ["tilted", "left"])
def test_oracle_stress_is_the_strain_derivative(name):
    """All six components of the float64 oracle's stress against central differences of the strained energy."""
    f = cell_frame("water", 4, name, seed=2, outside=True)
    meta = f.pop("_meta")
    cell = f["cell"]
    assert np.count_nonzero(cell.numpy() - np.diag(np.diagonal(cell.numpy()))) > 0
    assert float(f["edge_cell_shift"].abs().max()) > 1
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], parity=True, l_max=2, num_layers=3,
                              num_features=16, radial_mlp_depth=1, radial_mlp_width=16,
                              avg_num_neighbors=meta["avg_num_neighbors"], model_dtype=torch.float64)
    sd, cfg = model.state_dict(), model.config
    _e, _f, stress, virial = omodel.energy_forces_stress(sd, cfg, f, torch.float64)
    vol = abs(float(torch.linalg.det(cell)))
    torch.testing.assert_close(virial, -stress * vol, rtol=1e-13, atol=0)
    eps = 1e-5
    for a, b in [(0, 0), (1, 1), (2, 2), (0, 1), (1, 2), (2, 0)]:
        es = []
        for sgn in (+1, -1):
            strain = torch.eye(3, dtype=torch.float64)
            strain[a, b] += sgn * eps / 2
            strain[b, a] += sgn * eps / 2
            e, _ = omodel.energy(sd, cfg, dict(f, pos=f["pos"] @ strain, cell=cell @ strain), torch.float64)
            es.append(float(e))
        fd = (es[0] - es[1]) / (2 * eps) / vol
        got = float(stress[0, a, b])
        assert abs(fd - got) <= 1e-6 * float(stress.abs().max()), (name, a, b, fd, got)
