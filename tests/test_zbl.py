"""ZBL pair potential, host side: the oracle against LAMMPS (tests/golden/zbl_lammps.npy), units, the config block, the
symbol table, the per-type-pair table and the checkpoint key map.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

from nequip_b200 import data as D
from nequip_b200.nn.checkpoint import load_reference_state_dict, reference_key_map, to_reference_state_dict
from nequip_b200.nn.model import NequIPEnergyModel
from nequip_b200.nn.pair import ATOMIC_NUMBERS, QQR2E, ZBL, parse_pair_potential
from oracle import model as omodel
from oracle import pair as opair

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "zbl_lammps.npy")
SPECIES = ["H", "O", "C", "N", "Cu", "Au"]  # the fixture's elements
NL_RMAX, ZBL_RMAX, ZBL_P = 8.0, 9.0, 80.0  # pair_style zbl 8.0 8.0; a cutoff envelope that is irrelevant below 8


def _oracle_pair(r, zi, zj, units="metal"):
    """Energy and x-forces of two atoms on the x axis, from the host neighbour list (r_max 8) and the oracle ZBL."""
    m = ZBL(SPECIES, SPECIES, units, polynomial_cutoff_p=ZBL_P, model_dtype=torch.float64)
    types = torch.tensor([SPECIES.index(s) for s in (zi, zj)])
    pos_np = np.array([[0.0, 0.0, 0.0], [r, 0.0, 0.0]])
    ei, _ = D.neighbor_list(pos_np, None, NL_RMAX, pbc=False)
    ei = torch.from_numpy(ei)
    pos = torch.from_numpy(pos_np).requires_grad_(True)
    vec = pos[ei[1]] - pos[ei[0]]
    e = opair.zbl_atom_energy(m.atomic_numbers, m._qqr2exesquare, ZBL_P, ZBL_RMAX, vec, types, ei, 2, torch.float64)
    (g,) = torch.autograd.grad(e.sum(), pos)
    return float(e.detach().sum()), -g[:, 0].numpy()


def test_oracle_reproduces_lammps():
    ref = np.load(GOLDEN)
    assert ref.shape == (1800, 6)
    zname = {z: s for s, z in ATOMIC_NUMBERS.items()}
    n = 0
    for r, zi, zj, pe, fxi, fxj in ref:
        if r >= NL_RMAX:
            continue
        e, fx = _oracle_pair(r, zname[int(zi)], zname[int(zj)])
        np.testing.assert_allclose(fx, [fxi, fxj], atol=1e-5)
        np.testing.assert_allclose(e, pe, atol=1e-4)
        n += 1
    assert n == 1764


def test_real_units_scale_metal_units():
    for r, a, b in [(0.5, "H", "Au"), (1.3, "Cu", "O"), (3.1, "C", "N")]:
        em, fm = _oracle_pair(r, a, b, "metal")
        er, fr = _oracle_pair(r, a, b, "real")
        ratio = 332.06371 / 14.399645
        assert er == pytest.approx(em * ratio, rel=1e-14)
        np.testing.assert_allclose(fr, fm * ratio, rtol=1e-14)


def test_atomic_numbers():
    assert [ATOMIC_NUMBERS[s] for s in ("H", "C", "N", "O", "Cu", "Au")] == [1, 6, 7, 8, 29, 79]
    assert len(ATOMIC_NUMBERS) == 118 and ATOMIC_NUMBERS["Og"] == 118 and ATOMIC_NUMBERS["Fe"] == 26


def test_parse_pair_potential():
    tut = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["C", "H", "O", "Cu"]}
    assert parse_pair_potential(tut, 4) == dict(units="metal", chemical_species=["C", "H", "O", "Cu"],
                                                polynomial_cutoff_p=6.0)
    no_target = {k: v for k, v in tut.items() if k != "_target_"}
    assert parse_pair_potential(dict(no_target, polynomial_cutoff_p=80), 4)["polynomial_cutoff_p"] == 80.0
    assert parse_pair_potential(None, 4) is None
    bad = [
        dict(tut, _target_="nequip.nn.pair_potential.LennardJones"),
        dict(tut, chemical_species=["C", "H", "O", "Xx"]),
        dict(tut, chemical_species=["C", "H", "O"]),
        dict(tut, units="lj"),
        {k: v for k, v in tut.items() if k != "units"},
        dict(tut, polynomial_cutoff_p=1.0),
        dict(tut, lj_sigma=1.0),
    ]
    for spec in bad:
        with pytest.raises(ValueError):
            parse_pair_potential(spec, 4)
    with pytest.raises(ValueError):
        NequIPEnergyModel(r_max=5.0, type_names=["H", "O"], num_layers=1, pair_potential=dict(tut))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_pair_table(dtype):
    m = ZBL(["a", "b", "c"], ["H", "Cu", "Au"], "metal", model_dtype=dtype)
    assert m.atomic_numbers.dtype == dtype and m._qqr2exesquare.dtype == torch.float64
    assert float(m._qqr2exesquare) == 0.5 * QQR2E["metal"]
    t = ZBL.pair_table(m.atomic_numbers, m._qqr2exesquare)
    assert t.shape == (3, 3, 2) and t.dtype == torch.float64
    z = [1, 29, 79]
    for i in range(3):
        for j in range(3):
            assert float(t[i, j, 0]) == 0.5 * 14.399645 * z[i] * z[j]
            zi, zj = torch.tensor(float(z[i]), dtype=dtype), torch.tensor(float(z[j]), dtype=dtype)
            s = torch.pow(zi, 0.23) + torch.pow(zj, 0.23)  # rounded to the model dtype, then widened
            assert float(t[i, j, 1]) == float(s)
    if dtype == torch.float32:  # the float32 table is not the float64 one
        t64 = ZBL.pair_table(m.atomic_numbers.double(), m._qqr2exesquare)
        assert float((t[..., 1] - t64[..., 1]).abs().max()) > 0


TUTORIAL = dict(l_max=1, num_layers=4, num_features=32, radial_mlp_depth=2, radial_mlp_width=64)
TUTORIAL_ZBL = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["C", "H", "O", "Cu"]}


def _tutorial(pair_potential=None, **kw):
    return NequIPEnergyModel(r_max=5.0, type_names=["C", "H", "O", "Cu"], pair_potential=pair_potential,
                             **TUTORIAL, **kw)


def test_model_without_pair_potential_keeps_its_state_dict_and_config():
    base = NequIPEnergyModel(r_max=5.0, type_names=["C", "H", "O", "Cu"], **TUTORIAL)
    none = _tutorial(None)
    assert list(base.state_dict()) == list(none.state_dict())
    assert not any("pair_potential" in k for k in base.state_dict())
    assert "pair_potential" not in base.config and base.pair_potential is None
    assert reference_key_map(4, 2) == reference_key_map(4, 2, pair_potential=False)
    zbl = _tutorial(TUTORIAL_ZBL)
    assert set(zbl.state_dict()) == set(base.state_dict()) | {"pair_potential.atomic_numbers",
                                                             "pair_potential._qqr2exesquare"}
    assert zbl.config["pair_potential"] == dict(TUTORIAL_ZBL, polynomial_cutoff_p=6.0)
    assert zbl.pair_potential.atomic_numbers.tolist() == [6.0, 1.0, 8.0, 29.0]
    # the recorded config builds the same model
    again = NequIPEnergyModel(**zbl.config)
    assert list(again.state_dict()) == list(zbl.state_dict())


def test_checkpoint_key_map_round_trips():
    src = _tutorial(TUTORIAL_ZBL, seed=1)
    with torch.no_grad():
        src.pair_potential._qqr2exesquare.fill_(0.5 * QQR2E["real"])  # a rescaled checkpoint: the value travels
    ref_sd = to_reference_state_dict(src)
    assert "model.func.pair_potential.atomic_numbers" in ref_sd and "model.func.pair_potential._qqr2exesquare" in ref_sd
    dst = _tutorial(TUTORIAL_ZBL, seed=2)
    missing, unexpected = load_reference_state_dict(dst, ref_sd, strict=True)
    assert missing == [] and unexpected == []
    for k, v in src.state_dict().items():
        assert torch.equal(dst.state_dict()[k], v), k
    t = dst.pair_potential.table("cpu")
    assert float(t[0, 0, 0]) == 0.5 * QQR2E["real"] * 36
    # a model without ZBL reports the pair-potential keys as unexpected
    plain = _tutorial(None, seed=2)
    with pytest.raises(KeyError):
        load_reference_state_dict(plain, ref_sd, strict=True)
    _missing, unexpected = load_reference_state_dict(plain, ref_sd, strict=False)
    assert sorted(unexpected) == ["model.func.pair_potential._qqr2exesquare", "model.func.pair_potential.atomic_numbers"]


def test_oracle_model_with_zbl_stress_matches_finite_differences():
    """The float64 oracle of a model with ZBL: the energy is the network's plus the pair term, and its forces and
    stress are the derivatives of that energy (central differences in positions and in a symmetric strain)."""
    sysd = D.make_system("water", 3, r_max=5.0, seed=1)
    meta = sysd.pop("_meta")
    model = NequIPEnergyModel(r_max=5.0, type_names=meta["type_names"], l_max=1, num_layers=2, num_features=8,
                              model_dtype=torch.float64, pair_potential=dict(TUTORIAL_ZBL, chemical_species=["H", "O"]))
    sd, cfg = model.state_dict(), model.config
    e, f, s, _v = opair.energy_forces_stress(sd, cfg, sysd, torch.float64)
    e_net, _ = omodel.energy(sd, cfg, sysd, torch.float64)
    vec = omodel.edge_vectors(sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"])
    e_zbl = opair.zbl_atom_energy(sd["pair_potential.atomic_numbers"], sd["pair_potential._qqr2exesquare"], 6.0, 5.0,
                                  vec, sysd["atom_types"], sysd["edge_index"], sysd["pos"].shape[0], torch.float64)
    assert float(e_zbl.sum()) > 1e-3 * abs(float(e_net.sum()))
    assert float(e) == pytest.approx(float(e_net.sum() + e_zbl.sum()), rel=1e-13)
    eps, vol = 1e-5, float(torch.linalg.det(sysd["cell"]).abs())

    def en(d):
        return float(opair.energy(sd, cfg, d, torch.float64)[0].detach())

    for i, c in [(0, 0), (5, 2)]:
        es = []
        for sgn in (+1, -1):
            p = sysd["pos"].clone()
            p[i, c] += sgn * eps
            es.append(en(dict(sysd, pos=p)))
        assert float(f[i, c]) == pytest.approx(-(es[0] - es[1]) / (2 * eps), rel=1e-6, abs=1e-8)
    for a, b in [(0, 0), (0, 1)]:
        es = []
        for sgn in (+1, -1):
            strain = torch.zeros(3, 3, dtype=torch.float64)
            strain[a, b] += sgn * eps / 2
            strain[b, a] += sgn * eps / 2
            m = torch.eye(3, dtype=torch.float64) + strain
            es.append(en(dict(sysd, pos=sysd["pos"] @ m, cell=sysd["cell"] @ m)))
        assert float(s[0, a, b]) == pytest.approx((es[0] - es[1]) / (2 * eps) / vol, rel=1e-6, abs=1e-10)
