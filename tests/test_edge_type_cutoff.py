"""Per-edge-type cutoffs, host side: the table's parsing, the pruned host neighbour list against the brute-force list,
the float64 oracle on full and pruned lists (and its derivatives), the checkpoint key and a model without the option.
No GPU needed."""
import numpy as np
import pytest
import torch

import edge_type_oracle as eto
from cell_frames import brute_list, cell_frame
from nequip_b200 import data as D
from nequip_b200.nn.checkpoint import load_reference_state_dict, reference_key_map, to_reference_state_dict
from nequip_b200.nn.model import NequIPEnergyModel, parse_per_edge_type_cutoff
from oracle import model as omodel
from oracle import pair as opair

SMALL = dict(l_max=1, num_layers=2, num_features=8)
ZBL_CO = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["C", "O", "H"]}


def test_aspirin_table_parses_to_the_reference_matrix():
    t = parse_per_edge_type_cutoff(eto.ASPIRIN_CUTOFFS, eto.ASPIRIN_TYPES, 5.0)
    assert t.dtype == torch.float64 and tuple(t.shape) == (3, 3)
    assert t.tolist() == eto.ASPIRIN_TABLE
    assert t[0, 2] == 4.0 and t[2, 0] == 2.0  # asymmetric: C -> H 4.0, H -> C 2.0
    # missing sources and targets default to r_max, ints are accepted
    assert parse_per_edge_type_cutoff({"C": {"O": 3}}, ["C", "O"], 5.0).tolist() == [[5.0, 3.0], [5.0, 5.0]]
    assert parse_per_edge_type_cutoff({}, ["C", "O"], 4.5).tolist() == [[4.5, 4.5], [4.5, 4.5]]
    assert parse_per_edge_type_cutoff({"O": 5.0}, ["C", "O"], 5.0).tolist() == [[5.0, 5.0], [5.0, 5.0]]


@pytest.mark.parametrize("spec", [
    {"N": 2.0},                      # unknown source type
    {"C": {"N": 2.0}},               # unknown target type
    {"C": 0.0},                      # rc <= 0
    {"C": {"H": -1.0}},
    {"H": 5.5},                      # rc > r_max
    {"C": {"O": 5.0000001}},
    {"C": [2.0, 3.0, 4.0]},          # bad nesting
    {"C": {"H": {"O": 2.0}}},
    {"C": "2.0"},
    {"C": True},
    [("C", 2.0)],
])
def test_bad_tables_raise(spec):
    with pytest.raises(ValueError):
        parse_per_edge_type_cutoff(spec, eto.ASPIRIN_TYPES, 5.0)
    with pytest.raises(ValueError):
        NequIPEnergyModel(r_max=5.0, type_names=eto.ASPIRIN_TYPES, per_edge_type_cutoff=spec, **SMALL)


def test_model_surface():
    m = NequIPEnergyModel(r_max=5.0, type_names=eto.ASPIRIN_TYPES, per_edge_type_cutoff=eto.ASPIRIN_CUTOFFS, **SMALL)
    assert m.per_edge_type_cutoff.dtype == torch.float64 and m.per_edge_type_cutoff.tolist() == eto.ASPIRIN_TABLE
    assert m.rmax_recip.dtype == torch.float64 and tuple(m.rmax_recip.shape) == (9,)
    assert torch.equal(m.rmax_recip, torch.tensor(eto.ASPIRIN_TABLE, dtype=torch.float64).reciprocal().reshape(-1))
    assert m.config["per_edge_type_cutoff"] == eto.ASPIRIN_CUTOFFS
    again = NequIPEnergyModel(**m.config)  # the recorded config builds the same model
    assert torch.equal(again.per_edge_type_cutoff, m.per_edge_type_cutoff)
    assert list(again.state_dict()) == list(m.state_dict())
    # through from_preset's keyword arguments
    s = NequIPEnergyModel.from_preset("S", r_max=5.0, type_names=eto.ASPIRIN_TYPES,
                                      per_edge_type_cutoff=eto.ASPIRIN_CUTOFFS)
    assert s.per_edge_type_cutoff.tolist() == eto.ASPIRIN_TABLE


def test_model_without_the_option_is_unchanged():
    base = NequIPEnergyModel(r_max=5.0, type_names=eto.ASPIRIN_TYPES, **SMALL)
    none = NequIPEnergyModel(r_max=5.0, type_names=eto.ASPIRIN_TYPES, per_edge_type_cutoff=None, **SMALL)
    assert base.per_edge_type_cutoff is None and not hasattr(base, "rmax_recip")
    assert "per_edge_type_cutoff" not in base.config and base.config == none.config
    assert list(base.state_dict()) == list(none.state_dict())
    typed = NequIPEnergyModel(r_max=5.0, type_names=eto.ASPIRIN_TYPES, per_edge_type_cutoff=eto.ASPIRIN_CUTOFFS,
                              **SMALL)
    assert set(typed.state_dict()) == set(base.state_dict()) | {"rmax_recip"}
    assert reference_key_map(2) == reference_key_map(2, per_edge_type_cutoff=False)
    assert not any("rmax_recip" in k for k in to_reference_state_dict(base))


@pytest.mark.parametrize("cell,pbc", [("cubic", True), ("cubic", (True, True, False)), ("cubic", (False, False, True)),
                                      (None, False)])
def test_pruned_host_list_matches_brute_force(cell, pbc):
    n_side = 8  # 17 A cell: the periodic case takes the host list's cell-list path
    fr = cell_frame("li3po4", n_side, "cubic", seed=3, pbc=pbc)
    pos = fr["pos"].numpy()
    c = None if cell is None else fr["cell"].numpy()
    types = fr["atom_types"].numpy()
    for table in (np.array([[4.0, 3.1, 5.0], [2.6, 4.4, 3.7], [5.0, 3.3, 2.9]]), eto.random_table(3, 5.0, seed=4)):
        want = eto.pruned_brute_list(pos, c, pbc, 5.0, types, table)
        got = D.neighbor_list(pos, c, 5.0, pbc=pbc, atom_types=types, cutoffs=table)
        o = np.lexsort((got[1][:, 2], got[1][:, 1], got[1][:, 0], got[0][1], got[0][0]))
        assert np.array_equal(got[0][:, o], want[0]) and np.array_equal(got[1][o], want[1])
        assert 0 < want[0].shape[1] < brute_list(pos, c, pbc, 5.0)[0].shape[1]
    # a table of r_max everywhere gives the list without it, bit for bit
    full = D.neighbor_list(pos, c, 5.0, pbc=pbc)
    same = D.neighbor_list(pos, c, 5.0, pbc=pbc, atom_types=types, cutoffs=np.full((3, 3), 5.0))
    assert np.array_equal(full[0], same[0]) and np.array_equal(full[1], same[1])


def test_pruned_list_refuses_pairs_at_the_cutoff():
    pos = np.array([[0.0, 0.0, 0.0], [3.0, 0.0, 0.0], [0.0, 4.2, 0.0]])
    with pytest.raises(AssertionError):
        eto.pruned_brute_list(pos, None, False, 5.0, [0, 1, 1], [[5.0, 3.0], [3.0 + 1e-12, 5.0]])
    # asymmetric: 0 -> 2 (4.2 < 4.5) is kept, 2 -> 0 (4.2 >= 3.5) is dropped; 1 - 2 is beyond r_max
    ei, _ = eto.pruned_brute_list(pos, None, False, 5.0, [0, 1, 1], [[5.0, 4.5], [3.5, 5.0]])
    assert ei.T.tolist() == [[0, 1], [0, 2], [1, 0]]


def test_host_list_arguments():
    pos = np.zeros((2, 3))
    with pytest.raises(ValueError):
        D.neighbor_list(pos, None, 5.0, pbc=False, cutoffs=np.full((1, 1), 5.0))  # no types
    with pytest.raises(ValueError):
        D.neighbor_list(pos, None, 5.0, pbc=False, atom_types=[0, 1], cutoffs=np.full((1, 1), 5.0))  # type 1 >= T
    with pytest.raises(ValueError):
        D.neighbor_list(pos, None, 5.0, pbc=False, atom_types=[0, 0], cutoffs=np.full((1, 1), 6.0))  # rc > r_max


def _frame_and_model(zbl: bool, seed: int = 1):
    fr = D.make_system("li3po4", 4, r_max=5.0, seed=seed)
    fr.pop("_meta")
    model = NequIPEnergyModel(r_max=5.0, type_names=["Li", "P", "O"], model_dtype=torch.float64,
                              per_edge_type_cutoff={"Li": {"Li": 3.2, "O": 4.1}, "P": 3.6, "O": {"Li": 2.7}},
                              pair_potential=dict(ZBL_CO, chemical_species=["Li", "P", "O"]) if zbl else None, **SMALL)
    return fr, model


def _pruned(fr, model):
    ei, sh = D.neighbor_list(fr["pos"].numpy(), fr["cell"].numpy(), 5.0, atom_types=fr["atom_types"].numpy(),
                             cutoffs=model.per_edge_type_cutoff.numpy())
    return dict(fr, edge_index=torch.from_numpy(ei), edge_cell_shift=torch.from_numpy(sh))


@pytest.mark.parametrize("zbl", [False, True])
def test_oracle_energy_on_full_and_pruned_lists(zbl):
    fr, model = _frame_and_model(zbl)
    sd, cfg = model.state_dict(), model.config
    mod = opair if zbl else omodel
    pr = _pruned(fr, model)
    assert pr["edge_index"].shape[1] < 0.8 * fr["edge_index"].shape[1]
    with eto.per_edge_cutoffs(eto.edge_recip(fr["atom_types"], fr["edge_index"], model.per_edge_type_cutoff)):
        e_full, ea_full = mod.energy(sd, cfg, fr, torch.float64)
    with eto.per_edge_cutoffs(eto.edge_recip(pr["atom_types"], pr["edge_index"], model.per_edge_type_cutoff)):
        e_pr, ea_pr = mod.energy(sd, cfg, pr, torch.float64)
    assert float(e_pr) == pytest.approx(float(e_full), rel=1e-12)
    torch.testing.assert_close(ea_pr, ea_full, rtol=1e-11, atol=1e-12)
    # and the table changes the function: the oracle without it gives another energy
    e_plain, _ = mod.energy(sd, cfg, fr, torch.float64)
    assert abs(float(e_plain) - float(e_full)) > 1e-6 * abs(float(e_full))


@pytest.mark.parametrize("zbl", [False, True])
def test_oracle_forces_and_stress_match_finite_differences(zbl):
    fr, model = _frame_and_model(zbl, seed=2)
    fr = _pruned(fr, model)
    sd, cfg = model.state_dict(), model.config
    mod = opair if zbl else omodel
    eps, vol = 1e-5, float(torch.linalg.det(fr["cell"]).abs())
    with eto.per_edge_cutoffs(eto.edge_recip(fr["atom_types"], fr["edge_index"], model.per_edge_type_cutoff)):
        _e, f, s, _v = mod.energy_forces_stress(sd, cfg, fr, torch.float64)

        def en(d):
            return float(mod.energy(sd, cfg, d, torch.float64)[0].detach())

        for i, c in [(0, 0), (7, 2), (30, 1)]:
            es = []
            for sgn in (+1, -1):
                p = fr["pos"].clone()
                p[i, c] += sgn * eps
                es.append(en(dict(fr, pos=p)))
            assert float(f[i, c]) == pytest.approx(-(es[0] - es[1]) / (2 * eps), rel=1e-6, abs=1e-8)
        for a, b in [(0, 0), (1, 2)]:
            es = []
            for sgn in (+1, -1):
                strain = torch.zeros(3, 3, dtype=torch.float64)
                strain[a, b] += sgn * eps / 2
                strain[b, a] += sgn * eps / 2
                m = torch.eye(3, dtype=torch.float64) + strain
                es.append(en(dict(fr, pos=fr["pos"] @ m, cell=fr["cell"] @ m)))
            assert float(s[0, a, b]) == pytest.approx((es[0] - es[1]) / (2 * eps) / vol, rel=1e-6, abs=1e-10)


def test_checkpoint_round_trip_and_mismatches():
    kw = dict(r_max=5.0, type_names=eto.ASPIRIN_TYPES, **SMALL)
    src = NequIPEnergyModel(per_edge_type_cutoff=eto.ASPIRIN_CUTOFFS, seed=1, **kw)
    ref_sd = to_reference_state_dict(src)
    assert torch.equal(ref_sd["model.func.edge_norm._rmax_recip"], src.rmax_recip)
    dst = NequIPEnergyModel(per_edge_type_cutoff=eto.ASPIRIN_CUTOFFS, seed=2, **kw)
    missing, unexpected = load_reference_state_dict(dst, ref_sd, strict=True)
    assert missing == [] and unexpected == []
    for k, v in src.state_dict().items():
        assert torch.equal(dst.state_dict()[k], v), k
    # a table that differs from the model's raises
    other = NequIPEnergyModel(per_edge_type_cutoff={"H": 2.5}, **kw)
    with pytest.raises(ValueError):
        load_reference_state_dict(other, ref_sd, strict=True)
    # a non-trivial table into a model built without the option raises
    plain = NequIPEnergyModel(**kw)
    with pytest.raises(ValueError):
        load_reference_state_dict(plain, ref_sd, strict=False)
    # the scalar 1 / r_max every reference checkpoint holds loads into a model without the option
    sd_plain = to_reference_state_dict(NequIPEnergyModel(seed=3, **kw))
    sd_plain["model.func.edge_norm._rmax_recip"] = torch.tensor(1.0 / 5.0, dtype=torch.float64)
    missing, unexpected = load_reference_state_dict(plain, sd_plain, strict=True)
    assert missing == [] and unexpected == []
    # ... and a table model without its table in the checkpoint misses it; a scalar does not match a real table
    with pytest.raises(KeyError):
        load_reference_state_dict(dst, to_reference_state_dict(NequIPEnergyModel(seed=3, **kw)), strict=True)
    with pytest.raises(ValueError):
        load_reference_state_dict(dst, sd_plain, strict=True)
    # a table of r_max everywhere is the scalar
    flat = NequIPEnergyModel(per_edge_type_cutoff={"C": 5.0}, **kw)
    load_reference_state_dict(flat, sd_plain, strict=True)
