"""Oracle-free symmetry checks of energy, forces and stress in general cells, at sizes the oracle cannot reach: the
bench model family (l_max 2, 4 layers, 64 features, radial 1x128, frozen weights, tensor-core dense blocks) and its
float64 twin, on a few thousand atoms with device neighbour lists.

* another basis of the same lattice (``U @ cell``, integer U with det +-1, atoms re-wrapped) is the same crystal;
* a 2x2x1 supercell of a triclinic frame has 4x the energy, the same per-atom energies and forces on every copy and
  the same stress;
* a rigid rotation R of positions and cell leaves the energy unchanged and rotates forces (F R^T) and stress
  (R sigma R^T).

float64 must agree to 1e-11 relative (seen: 9e-14 at most).  float32 differs by rounding only (the edge vectors change
in their last bits): the largest relative deviation seen on an H100 SXM (80 GB, 700 W power limit) was 5.3e-7, on the
supercell's per-atom energies, and the bound is about 10x that."""
import numpy as np
import pytest
import torch

from cell_frames import cell_frame
from nequip_b200 import ops
from nequip_b200.nn.model import NequIPEnergyModel

pytestmark = pytest.mark.gpu

R_MAX = 5.0
F64_TOL = 1e-11
F32_TOL = 5e-6


def _models(meta):
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], parity=True, avg_num_neighbors=meta["avg_num_neighbors"],
              l_max=2, num_layers=4, num_features=64, radial_mlp_depth=1, radial_mlp_width=128)
    m32 = NequIPEnergyModel(strict_fast_path=True, **kw).cuda()
    m64 = NequIPEnergyModel(model_dtype=torch.float64, **kw).cuda()
    m64.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in m32.state_dict().items()})
    for m in (m32, m64):
        for p in m.parameters():
            p.requires_grad_(False)
    return {"f32": m32, "f64": m64}


def _setup(n_side):
    f = cell_frame("li3po4", n_side, "tilted", seed=21, outside=True)
    return f, _models(f["_meta"])


@pytest.fixture(scope="module")
def big():
    """13^3 = 2197 atoms in the tilted cell: basis change and rotation."""
    return _setup(13)


@pytest.fixture(scope="module")
def base():
    """9^3 = 729 atoms in the tilted cell, 2916 in its 2x2x1 supercell."""
    return _setup(9)


def _run(model, pos, cell, types):
    pos, cell = torch.as_tensor(pos).cuda(), torch.as_tensor(cell).cuda()
    nl = ops.neighbor_list(pos, cell, True, R_MAX)
    out = model({"pos": pos, "cell": cell, "atom_types": types.cuda(), "edge_index": nl["edge_index"],
                 "edge_cell_shift": nl["edge_cell_shift"]}, compute_stress=True)
    return {k: out[k].detach().double().cpu() for k in ("total_energy", "atomic_energy", "forces", "stress")}


def _rel(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


def _compare(got, ref, dtype, what):
    tol = F64_TOL if dtype == "f64" else F32_TOL
    errs = {k: _rel(got[k], ref[k]) for k in ("atomic_energy", "forces", "stress")}
    errs["total_energy"] = abs(float(got["total_energy"]) - float(ref["total_energy"])) / float(ref["atomic_energy"].abs().sum())
    print(f"{what} {dtype}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v <= tol, (what, dtype, k, v)


@pytest.mark.parametrize("dtype", ["f64", "f32"])
@pytest.mark.parametrize("U", [
    [[1, 1, 0], [0, 1, 0], [0, -1, 1]],  # det +1
    [[0, 1, 0], [1, 0, 1], [0, 0, 1]],  # det -1: a left-handed basis of the same lattice
], ids=["det+1", "det-1"])
def test_another_basis_of_the_same_lattice(big, U, dtype):
    f, models = big
    pos, cell = f["pos"].numpy(), f["cell"].numpy()
    U = np.array(U, dtype=np.float64)
    cell2 = U @ cell
    frac2 = pos @ np.linalg.inv(cell2)
    pos2 = (frac2 - np.floor(frac2)) @ cell2
    assert np.abs(pos2 - pos).max() > 10.0, "the atoms were re-wrapped"
    ref = _run(models[dtype], pos, cell, f["atom_types"])
    got = _run(models[dtype], pos2, cell2, f["atom_types"])
    _compare(got, ref, dtype, f"basis det {np.linalg.det(U):+.0f}")


@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_supercell_2x2x1(base, dtype):
    f, models = base
    pos, cell, types = f["pos"].numpy(), f["cell"].numpy(), f["atom_types"]
    n = pos.shape[0]
    copies = [(a, b) for a in range(2) for b in range(2)]  # atom c * n + k is atom k moved by a a_0 + b a_1
    sup = np.concatenate([pos + a * cell[0] + b * cell[1] for a, b in copies], 0)
    sup_cell = np.diag([2.0, 2.0, 1.0]) @ cell
    ref = _run(models[dtype], pos, cell, types)
    got = _run(models[dtype], sup, sup_cell, types.repeat(4))
    tiled = {"total_energy": 4 * ref["total_energy"], "atomic_energy": ref["atomic_energy"].repeat(4, 1),
             "forces": ref["forces"].repeat(4, 1), "stress": ref["stress"]}
    assert got["forces"].shape == (4 * n, 3)
    _compare(got, tiled, dtype, "supercell 2x2x1")


@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_rigid_rotation(big, dtype):
    f, models = big
    pos, cell = f["pos"].numpy(), f["cell"].numpy()
    q, r = np.linalg.qr(np.random.default_rng(3).normal(size=(3, 3)))
    R = q * np.sign(np.diag(r))
    if np.linalg.det(R) < 0:
        R[:, 0] = -R[:, 0]
    assert abs(np.linalg.det(R) - 1.0) < 1e-12
    ref = _run(models[dtype], pos, cell, f["atom_types"])
    got = _run(models[dtype], pos @ R.T, cell @ R.T, f["atom_types"])
    Rt = torch.from_numpy(R)
    rotated = {"total_energy": ref["total_energy"], "atomic_energy": ref["atomic_energy"],
               "forces": ref["forces"] @ Rt.T, "stress": (Rt @ ref["stress"][0] @ Rt.T)[None]}
    _compare(got, rotated, dtype, "rotation")
