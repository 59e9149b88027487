"""Per-edge-type cutoffs on the device: the typed edge-embedding, ZBL and neighbour-list kernels against the float64
oracle and the brute-force list, their write contracts, whole models on a tilted cell, full against pruned lists, the
reference's locality test per type pair, captured MD steps, the reverse-edge pair map and the unchanged path of models
without a table."""
import math

import numpy as np
import pytest
import torch

import edge_type_oracle as eto
from cell_frames import CELL_SHAPES, cell_frame
from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel
from oracle import pair as opair
from oracle import sh as osh

pytestmark = pytest.mark.gpu

R_MAX = 5.0
WATER_L2 = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)  # water_1k family
TUTORIAL = dict(l_max=1, num_layers=4, num_features=32, radial_mlp_depth=2, radial_mlp_width=64)
LI3PO4_TABLE = {"Li": {"Li": 3.2, "O": 4.1}, "P": 3.6, "O": {"Li": 2.7, "O": 4.4}}  # asymmetric: Li-O 4.1, O-Li 2.7
LI3PO4_SYM = {"Li": {"Li": 3.2, "P": 3.6, "O": 4.1}, "P": 3.6, "O": {"Li": 4.1, "P": 3.6, "O": 4.4}}


def _rel(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max()) / float(b.abs().max())


def _recip_dev(table):
    return table.reciprocal().reshape(-1).cuda()


# ------------------------------------------------------------------------------------------------------------------
# edge-embedding kernels
# ------------------------------------------------------------------------------------------------------------------
def _embed_oracle(sysd, table, lmax, dtype, gy, ge):
    """Oracle y, emb and the vector-Jacobian products with (gy, ge) w.r.t. pos and the edge vectors."""
    pos = sysd["pos"].clone().requires_grad_(True)
    vec = omodel.edge_vectors(pos, sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"])
    vec.retain_grad()
    r = vec.square().sum(1, keepdim=True).sqrt()
    y = osh.spherical_harmonics(lmax, vec, normalize=True).to(dtype)
    with eto.per_edge_cutoffs(eto.edge_recip(sysd["atom_types"], sysd["edge_index"], table)):
        emb = omodel.radial_embedding(r, R_MAX, 8, 6.0, dtype)
    ((y.double() * gy).sum() + (emb.double() * ge).sum()).backward()
    return y.detach(), emb.detach(), pos.grad, vec.grad


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("lmax", [0, 1, 2, 3, 4])
def test_typed_embedding_matches_oracle(lmax, dtype):
    sysd = cell_frame("li3po4", 5, "tilted", seed=lmax, outside=True)
    sysd.pop("_meta")
    table = torch.as_tensor(eto.random_table(3, R_MAX, seed=lmax), dtype=torch.float64)
    dev = D.to_device(sysd, "cuda")
    E = sysd["edge_index"].shape[1]
    g = torch.Generator().manual_seed(7)
    gy = torch.randn(E, (lmax + 1) ** 2, generator=g, dtype=torch.float64)
    ge = torch.randn(E, 8, generator=g, dtype=torch.float64)
    y_ref, emb_ref, gpos_ref, gvec_ref = _embed_oracle(sysd, table, lmax, dtype, gy, ge)
    tol = 1e-5 if dtype == torch.float32 else 1e-12
    kw = dict(lmax=lmax, num_bessel=8, r_max=R_MAX, prefactor=2 * math.pi / R_MAX ** 2, out_dtype=dtype,
              types=dev["atom_types"], edge_type_recip=_recip_dev(table))
    pos = dev["pos"].clone().requires_grad_(True)
    sink = {}
    _v, y, emb = ops.edge_embed(pos, dev["edge_index"], dev["edge_cell_shift"], dev["cell"], edge_grad_sink=sink, **kw)
    assert _rel(y, y_ref) <= tol and _rel(emb, emb_ref) <= tol
    ((y.double() * gy.cuda()).sum() + (emb.double() * ge.cuda()).sum()).backward()
    assert _rel(pos.grad, gpos_ref) <= tol * 10 and _rel(sink["edge_vector_grad"], gvec_ref) <= tol * 10
    # pruning matters: some edges of the r_max list are zeroed by their pair's cutoff
    assert int((emb_ref.abs().sum(1) == 0).sum()) > 0.2 * E
    # the edge-vector branch: made-up positions for the geometry, the types from the real edge_index
    vec = dev["pos"][dev["edge_index"][1]] - dev["pos"][dev["edge_index"][0]] + dev["edge_cell_shift"] @ dev["cell"]
    vec = vec.detach().requires_grad_(True)
    yv, ev = ops.edge_embed_from_vectors(vec, edge_index=dev["edge_index"], **kw)
    assert _rel(yv, y_ref) <= tol and _rel(ev, emb_ref) <= tol
    ((yv.double() * gy.cuda()).sum() + (ev.double() * ge.cuda()).sum()).backward()
    assert _rel(vec.grad, gvec_ref) <= tol * 10
    # E = 0
    _v0, y0, e0 = ops.edge_embed(dev["pos"], dev["edge_index"][:, :0], dev["edge_cell_shift"][:0], dev["cell"], **kw)
    assert y0.shape == (0, (lmax + 1) ** 2) and e0.shape == (0, 8)


def test_typed_write_contracts():
    """Every output of the new entry points fully written, nothing outside it; grad_pos accumulated into."""
    sysd = cell_frame("li3po4", 4, "tilted", seed=1, outside=True)
    sysd.pop("_meta")
    dev = D.to_device(sysd, "cuda")
    N, E = sysd["pos"].shape[0], sysd["edge_index"].shape[1]
    table = torch.as_tensor(eto.random_table(3, R_MAX, seed=2), dtype=torch.float64)
    recip = _recip_dev(table)
    L, st = _capi.lib(), torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()  # noqa: E731
    for dt, code in ((torch.float32, 0), (torch.float64, 1)):
        vec, ck_v = guarded(E, 3, torch.float64)
        y, ck_y = guarded(E, 9, dt)
        emb, ck_e = guarded(E, 8, dt)
        _capi.check(L.nqb_edge_embed_fwd_typed(2, 8, R_MAX, 6.0, 1.0, p(dev["pos"]), p(dev["edge_index"]),
                                               p(dev["edge_cell_shift"]), p(dev["cell"]), N, E, p(dev["atom_types"]),
                                               p(dev["edge_index"]), p(recip), 3, code, p(vec), p(y), p(emb), st))
        gy, ge = torch.randn(E, 9, device="cuda", dtype=dt), torch.randn(E, 8, device="cuda", dtype=dt)
        gpos, ck_p = guarded(N, 3, torch.float64, body="random", generator=torch.Generator().manual_seed(3))
        base = gpos.detach().cpu().clone()
        gvec, ck_g = guarded(E, 3, torch.float64)
        _capi.check(L.nqb_edge_embed_bwd_typed(2, 8, R_MAX, 6.0, 1.0, p(vec), p(dev["edge_index"]), N, E,
                                               p(dev["atom_types"]), p(dev["edge_index"]), p(recip), 3, code, p(gy),
                                               p(ge), p(gpos), p(gvec), st))
        torch.cuda.synchronize()
        for ck, what in ((ck_v, "vec"), (ck_y, "y"), (ck_e, "emb"), (ck_p, "grad_pos"), (ck_g, "grad_vec")):
            ck(what)
        for t in (vec, y, emb, gvec):
            assert not bool(is_poison(t).any())
        # grad_pos = base + scatter of grad_vec
        ei = sysd["edge_index"]
        want = base.clone().index_add_(0, ei[1], gvec.cpu()).index_add_(0, ei[0], -gvec.cpu())
        assert float((gpos.cpu() - want).abs().max()) <= 1e-12 * float(want.abs().max())
    # ZBL
    from nequip_b200.nn.pair import ZBL

    zt = ZBL(["Li", "P", "O"], ["Li", "P", "O"], "metal", model_dtype=torch.float64).table("cuda")
    csr = ops.build_csr(dev["edge_index"][0].contiguous(), N)
    geom = (p(dev["pos"]), p(dev["edge_index"]), p(dev["edge_cell_shift"]), p(dev["cell"]), 0, p(dev["atom_types"]),
            p(zt), 3)
    e_atom, ck_a = guarded(N, 1, torch.float64)
    _capi.check(L.nqb_zbl_fwd_typed(*geom, p(csr.row_ptr), 0, N, E, R_MAX, 6.0, 0, p(recip), p(e_atom), st))
    ga = torch.randn(N, device="cuda", dtype=torch.float64)
    gvec, ck_g = guarded(E, 3, torch.float64)
    _capi.check(L.nqb_zbl_bwd_typed(*geom, N, E, R_MAX, 6.0, 0, p(recip), p(ga), 0, p(gvec), st))
    torch.cuda.synchronize()
    ck_a("e_atom")
    ck_g("zbl grad_vec")
    assert not bool(is_poison(e_atom).any()) and not bool(is_poison(gvec).any())
    vec = omodel.edge_vectors(sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"])
    with eto.per_edge_cutoffs(eto.edge_recip(sysd["atom_types"], sysd["edge_index"], table)):
        m = ZBL(["Li", "P", "O"], ["Li", "P", "O"], "metal", model_dtype=torch.float64)
        ref = opair.zbl_atom_energy(m.atomic_numbers, m._qqr2exesquare, 6.0, R_MAX, vec, sysd["atom_types"],
                                    sysd["edge_index"], N, torch.float64)
    assert _rel(e_atom, ref) <= 1e-12


# ------------------------------------------------------------------------------------------------------------------
# device neighbour lists
# ------------------------------------------------------------------------------------------------------------------
def _sorted(ei, sh):
    o = np.lexsort((sh[:, 2], sh[:, 1], sh[:, 0], ei[1], ei[0]))
    return ei[:, o], sh[o]


def _real(out, plan):
    """Mask of the real edges of a capacity list (null edges are (i, i, pad_shift))."""
    real = out["edge_index"][0] != out["edge_index"][1]
    return real | (out["edge_cell_shift"] != torch.as_tensor(plan.pad_shift, device="cuda")).any(1)


@pytest.mark.parametrize("pbc", [(True, True, True), (True, True, False), (False, False, True)])
@pytest.mark.parametrize("cell", sorted(CELL_SHAPES))
def test_device_list_matches_pruned_brute_force(cell, pbc):
    n_side = 2 if cell == "small" else 6
    fr = cell_frame("li3po4", n_side, cell, seed=4, outside=True, pbc=pbc)
    pos, c, types = fr["pos"].numpy(), fr["cell"].numpy(), fr["atom_types"].numpy()
    table = torch.tensor([[4.0, 3.1, 5.0], [2.6, 4.4, 3.7], [5.0, 3.3, 2.9]], dtype=torch.float64)
    want = eto.pruned_brute_list(pos, c, pbc, R_MAX, types, table.numpy())
    nl = ops.neighbor_list(fr["pos"].cuda(), fr["cell"], pbc, R_MAX, atom_types=fr["atom_types"].cuda(),
                           edge_type_cutoff=table)
    got = _sorted(nl["edge_index"].cpu().numpy(), nl["edge_cell_shift"].cpu().numpy())
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert bool((nl["edge_index"][0][1:] >= nl["edge_index"][0][:-1]).all())  # grouped by centre
    if not all(pbc):
        return
    E = want[0].shape[1]
    for variable in (False, True):  # capacity lists, fixed and variable cell
        plan = ops.NeighborListPlan(pos.shape[0], fr["cell"], True, R_MAX, E + 37, variable_cell=variable,
                                    atom_types=fr["atom_types"].cuda(), edge_type_cutoff=table)
        plan.edge_index.fill_(-7)
        out = plan.run(fr["pos"].cuda())
        assert int(out["num_edges"]) == E and int(out["overflow"]) == 0
        real = _real(out, plan)
        assert torch.equal(out["edge_index"][:, real].cpu(), nl["edge_index"].cpu())
        assert torch.equal(out["edge_cell_shift"][real].cpu(), nl["edge_cell_shift"].cpu())
        if variable:  # set_cell to a strained cell gives that cell's pruned list
            S = D.oscillating_strain(3)
            plan.set_cell(fr["cell"] @ S)
            out = plan.run(fr["pos"].cuda() @ S.cuda())
            ref = ops.neighbor_list(fr["pos"].cuda() @ S.cuda(), fr["cell"] @ S, True, R_MAX,
                                    atom_types=fr["atom_types"].cuda(), edge_type_cutoff=table)
            assert int(out["num_edges"]) == ref["edge_index"].shape[1]
            assert torch.equal(out["edge_index"][:, _real(out, plan)].cpu(), ref["edge_index"].cpu())


def test_device_list_many_types():
    """T = 89 with a random asymmetric table (the table and the types are read from device memory)."""
    fr = cell_frame("li3po4", 7, "tilted", seed=9, outside=True)
    T = 89
    types = torch.randint(0, T, fr["atom_types"].shape, generator=torch.Generator().manual_seed(1))
    table = torch.as_tensor(eto.random_table(T, R_MAX, seed=5), dtype=torch.float64)
    want = eto.pruned_brute_list(fr["pos"].numpy(), fr["cell"].numpy(), True, R_MAX, types.numpy(), table.numpy())
    nl = ops.neighbor_list(fr["pos"].cuda(), fr["cell"], True, R_MAX, atom_types=types.cuda(), edge_type_cutoff=table)
    got = _sorted(nl["edge_index"].cpu().numpy(), nl["edge_cell_shift"].cpu().numpy())
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    plan = ops.NeighborListPlan(types.numel(), fr["cell"], True, R_MAX, want[0].shape[1], atom_types=types,
                                edge_type_cutoff=table)
    out = plan.run(fr["pos"].cuda())
    assert int(out["overflow"]) == 0 and torch.equal(out["edge_index"].cpu(), nl["edge_index"].cpu())
    with pytest.raises(ValueError):
        ops.neighbor_list(fr["pos"].cuda(), fr["cell"], True, R_MAX, atom_types=types.cuda(), edge_type_cutoff=table * 2)


# ------------------------------------------------------------------------------------------------------------------
# whole models
# ------------------------------------------------------------------------------------------------------------------
def _model(arch, names, dtype, ann, table, species=None, preset=None):
    pp = None if species is None else {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal",
                                       "chemical_species": species}
    common = dict(r_max=R_MAX, type_names=names, avg_num_neighbors=ann, model_dtype=dtype, pair_potential=pp,
                  per_edge_type_cutoff=table, strict_fast_path=(dtype == torch.float32))
    m = NequIPEnergyModel.from_preset(preset, **common) if preset else NequIPEnergyModel(parity=True, **arch, **common)
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


@pytest.mark.timeout(900)
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.float64, 1e-9)])
@pytest.mark.parametrize("which", ["water_1k_l2_f32", "tutorial_zbl", "preset_S"])
def test_models_match_oracle(which, dtype, tol):
    import preset_oracle as po

    sysd = cell_frame("li3po4", 5, "tilted", seed=5, outside=True)
    meta = sysd.pop("_meta")
    species = ["Li", "P", "O"] if which == "tutorial_zbl" else None
    preset = "S" if which == "preset_S" else None
    arch = TUTORIAL if which == "tutorial_zbl" else WATER_L2
    model = _model(arch, meta["type_names"], dtype, meta["avg_num_neighbors"], LI3PO4_TABLE, species, preset)
    mod = po if preset else (opair if species else omodel)
    sd, cfg = model.state_dict(), model.config
    out = model(D.to_device(sysd, "cuda"), compute_stress=True)
    vec = omodel.edge_vectors(sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"])
    d = {k: v for k, v in sysd.items() if k not in ("cell", "edge_cell_shift")}
    d["edge_vectors"] = vec
    with eto.per_edge_cutoffs(eto.edge_recip(sysd["atom_types"], sysd["edge_index"], model.per_edge_type_cutoff)):
        e_ref, f_ref, s_ref, v_ref = mod.energy_forces_stress(sd, cfg, sysd, dtype)
        _e, ea_ref, _f = mod.energy_and_forces(sd, cfg, sysd, dtype)
        e_ref_v, g_ref = mod.edge_forces(sd, cfg, d, dtype)
    escale = float(ea_ref.abs().sum())
    assert abs(float(out["total_energy"]) - float(e_ref)) <= tol * escale
    assert _rel(out["atomic_energy"], ea_ref) <= tol
    for k, ref in (("forces", f_ref), ("stress", s_ref), ("virial", v_ref)):
        assert _rel(out[k], ref) <= tol, (k, _rel(out[k], ref))
    out_v = model(D.to_device(d, "cuda"))
    assert _rel(out_v["edge_forces"], g_ref) <= tol
    assert abs(float(out_v["total_energy"]) - float(e_ref_v)) <= tol * escale
    # the table changes the result (the comparison would be vacuous otherwise)
    _e0, ea0, _f0 = mod.energy_and_forces(sd, cfg, sysd, dtype)
    assert _rel(ea0, ea_ref) > 1e-3


@pytest.mark.parametrize("zbl", [False, True])
def test_full_list_equals_pruned_list(zbl):
    sysd = cell_frame("li3po4", 6, "tilted", seed=6, outside=True)
    meta = sysd.pop("_meta")
    model = _model(WATER_L2, meta["type_names"], torch.float32, meta["avg_num_neighbors"], LI3PO4_TABLE,
                   ["Li", "P", "O"] if zbl else None)
    dev = D.to_device(sysd, "cuda")
    nl = ops.neighbor_list(dev["pos"], dev["cell"], True, R_MAX, atom_types=dev["atom_types"],
                           edge_type_cutoff=model.per_edge_type_cutoff)
    assert nl["edge_index"].shape[1] < 0.8 * dev["edge_index"].shape[1]
    full = model(dev)
    pruned = model(dict(dev, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))
    # Every dropped edge adds exact zeros, but not bitwise the same sums: the TP + scatter kernels spread a row's
    # edges over sub-lanes by position, and the zero edges sit between the kept ones (a padded list's null edges
    # come after them and leave the sums bitwise unchanged).  So the bound is float32 rounding.
    escale = float(full["atomic_energy"].abs().sum())
    assert abs(float(full["total_energy"]) - float(pruned["total_energy"])) <= 1e-6 * escale
    assert _rel(pruned["atomic_energy"], full["atomic_energy"]) <= 2e-6
    assert _rel(pruned["forces"], full["forces"]) <= 2e-6


def test_partial_force_locality_per_type_pair():
    """The reference's partial-force locality test (nequip/utils/unittests/model_tests_basic.py), per ordered type pair
    of the aspirin table: for a centre a and a neighbour b at distance d, a's energy depends on b's position at
    d = 0.5 rc_ab and not at d = rc_ab or 1.1 rc_ab.  Both edges are in the list (the full r_max one), so the kernels'
    zeroing is what is checked, not the pruning."""
    names = eto.ASPIRIN_TYPES
    model = _model(dict(WATER_L2, num_features=8), names, torch.float64, 1.0, eto.ASPIRIN_CUTOFFS)
    table = model.per_edge_type_cutoff
    for a in range(3):
        for b in range(3):
            rc = float(table[a, b])
            at_rc = rc
            while at_rc * (1.0 / rc) < 1.0:  # the length whose normalised value x = r * (1 / rc) is 1
                at_rc = float(np.nextafter(at_rc, np.inf))
            for d, nonzero in ((0.5 * rc, True), (at_rc, False), (1.1 * rc, False)):
                if d >= R_MAX:
                    continue
                pos = torch.tensor([[0.0, 0.0, 0.0], [d, 0.0, 0.0]], dtype=torch.float64, device="cuda")
                pos.requires_grad_(True)
                data = dict(pos=pos, atom_types=torch.tensor([a, b], device="cuda"),
                            edge_index=torch.tensor([[0, 1], [1, 0]], device="cuda"))
                with torch.enable_grad():
                    e_atom = model.energy(dict(data))["atomic_energy"]
                    (g,) = torch.autograd.grad(e_atom[0].sum(), pos)
                assert bool((g[1].abs() > 0).any()) == nonzero, (names[a], names[b], d, g[1].tolist())


# ------------------------------------------------------------------------------------------------------------------
# captured MD steps
# ------------------------------------------------------------------------------------------------------------------
def _md(n_side, spec=LI3PO4_TABLE):
    sysd = D.make_system("li3po4", n_side, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    dev = D.to_device(sysd, "cuda")
    model = _model(WATER_L2, meta["type_names"], torch.float32, meta["avg_num_neighbors"], spec, ["Li", "P", "O"])
    return dev, model


def _eager(model, pos, cell, dev, stress=False):
    nl = ops.neighbor_list(pos, cell, True, R_MAX, atom_types=dev["atom_types"],
                           edge_type_cutoff=model.per_edge_type_cutoff)
    out = model(dict(dev, pos=pos, cell=cell, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]),
                compute_stress=stress)
    return out, nl


def _assert_matches(out, ref, what, keys=("forces",)):
    e_ref = float(ref["total_energy"])
    torch.testing.assert_close(out["total_energy"], ref["total_energy"], rtol=1e-12, atol=1e-9 * abs(e_ref), msg=what)
    for k in keys:
        assert _rel(out[k], ref[k]) <= 2e-6, (what, k, _rel(out[k], ref[k]))


def test_graphed_md_step_fixed_cell_and_recapture():
    dev, model = _md(6)
    pos0 = dev["pos"].clone()
    g = GraphedMDStep(model, dev)
    E0 = ops.neighbor_list(pos0, dev["cell"], True, R_MAX, atom_types=dev["atom_types"],
                           edge_type_cutoff=model.per_edge_type_cutoff)["edge_index"].shape[1]
    assert g.capacity == E0 + math.ceil(0.02 * E0)  # sized from the pruned count
    for t in range(10):
        pos = D.oscillating_positions(pos0, t, period=50, seed=7)
        out = g(pos)
        ref, nl = _eager(model, pos, dev["cell"], dev)
        assert int(out["num_edges"]) == nl["edge_index"].shape[1]
        _assert_matches(out, ref, f"step {t}")
        pl = g.plan  # the padded list holds the exact list
        padded = dict(edge_index=pl.edge_index, edge_cell_shift=pl.edge_cell_shift)
        assert torch.equal(pl.edge_index[:, _real(padded, pl)], nl["edge_index"])
    # a frame with more edges than the capacity is re-captured
    g = GraphedMDStep(model, dev, capacity=E0 - 10)
    out = g(dev["pos"])
    assert g.recaptures == 1 and g.capacity >= E0
    ref, nl = _eager(model, dev["pos"], dev["cell"], dev)
    assert int(out["num_edges"]) == nl["edge_index"].shape[1] == E0
    _assert_matches(out, ref, "after re-capture")


def test_graphed_md_step_variable_cell():
    dev, model = _md(5)
    pos0 = dev["pos"].clone()
    g = GraphedMDStep(model, dev, variable_cell=True)
    for t in range(8):
        S = D.oscillating_strain(t).cuda()
        pos, cell = D.oscillating_positions(pos0, t, period=50, seed=7) @ S, dev["cell"] @ S
        out = g(pos, cell)
        ref, nl = _eager(model, pos, cell, dev, stress=True)
        assert int(out["num_edges"]) == nl["edge_index"].shape[1]
        _assert_matches(out, ref, f"step {t}", keys=("forces", "stress", "virial"))


# ------------------------------------------------------------------------------------------------------------------
# reverse-edge pairs, and models without a table
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("symmetric", [True, False])
def test_edge_pairs_with_a_table(symmetric):
    dev, model = _md(22, LI3PO4_SYM if symmetric else LI3PO4_TABLE)  # the bench frame: Li3PO4, 10 648 atoms
    nl = ops.neighbor_list(dev["pos"], dev["cell"], True, R_MAX, atom_types=dev["atom_types"],
                           edge_type_cutoff=model.per_edge_type_cutoff)
    ei, sh = nl["edge_index"], nl["edge_cell_shift"]
    E = ei.shape[1]
    assert torch.equal(model.per_edge_type_cutoff, model.per_edge_type_cutoff.t()) == symmetric
    _v, _y, emb = ops.edge_embed(dev["pos"], ei, sh, dev["cell"], lmax=2, num_bessel=8, r_max=R_MAX,
                                 prefactor=2 * math.pi / R_MAX ** 2, types=dev["atom_types"],
                                 edge_type_recip=model.rmax_recip)
    csr = ops.build_csr(ei[0].contiguous(), dev["pos"].shape[0])
    pairs = ops.edge_pairs(ei, sh, emb, csr)
    U = int(pairs[1])
    if symmetric:
        assert 2 * U == E
    else:
        assert E // 2 < U < E  # one-way edges get a slot of their own
    types = dev["atom_types"]
    tc = model.layers[0].conv._tensor_core_blocks(model.type_embed.weight[types], types, model.type_embed.weight)
    assert torch.equal(tc["mlp"](emb, pairs), tc["mlp"](emb, None))


def test_model_without_table_calls_no_typed_entry_point(monkeypatch):
    sysd = cell_frame("li3po4", 4, "tilted", seed=2, outside=True)
    meta = sysd.pop("_meta")
    dev = D.to_device(sysd, "cuda")
    plain = _model(WATER_L2, meta["type_names"], torch.float32, meta["avg_num_neighbors"], None, ["Li", "P", "O"])
    L = _capi.lib()
    calls = []
    for name in [n for n in _capi.SIGNATURES if n.endswith("_typed")]:
        def boom(*a, _n=name, **k):
            calls.append(_n)
            raise AssertionError(f"{_n} called")
        monkeypatch.setattr(L, name, boom)
    plain(dev)
    plain(dev, compute_stress=True)
    vec = omodel.edge_vectors(sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"]).cuda()
    plain({k: v for k, v in dev.items() if k not in ("cell", "edge_cell_shift")} | {"edge_vectors": vec})
    ops.neighbor_list(dev["pos"], dev["cell"], True, R_MAX)
    GraphedMDStep(plain, dev)(dev["pos"])
    assert calls == []
