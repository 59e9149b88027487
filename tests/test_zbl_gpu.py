"""ZBL pair potential on the device (nqb_zbl_fwd / nqb_zbl_bwd, ops.zbl_energy, NequIPEnergyModel(pair_potential=...)):
LAMMPS' numbers, the float64 oracle, the write contract, whole models, a close pair, captured MD steps (fixed and
variable cell) and the unchanged path of models without a pair potential."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from cell_frames import cell_frame
from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel
from nequip_b200.nn.pair import ATOMIC_NUMBERS, ZBL
from oracle import model as omodel
from oracle import pair as opair

pytestmark = pytest.mark.gpu

R_MAX = 5.0
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "zbl_lammps.npy")
LAMMPS_SPECIES = ["H", "O", "C", "N", "Cu", "Au"]
TUTORIAL = dict(l_max=1, num_layers=4, num_features=32, radial_mlp_depth=2, radial_mlp_width=64)
WATER_L2 = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)  # bench_md water_1k


def _rel(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max()) / float(b.abs().max())


def _zbl_spec(species, **kw):
    return dict({"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": list(species)}, **kw)


# ------------------------------------------------------------------------------------------------------------------
# LAMMPS fixture
# ------------------------------------------------------------------------------------------------------------------
def _lammps_pairs():
    """Every fixture row with r < 8 as one frame of isolated two-atom pairs 100 A apart (the list of each pair is what
    a neighbour list with r_max 8 gives: both directions)."""
    ref = np.load(GOLDEN)
    ref = ref[ref[:, 0] < 8.0]
    M = ref.shape[0]
    zidx = {ATOMIC_NUMBERS[s]: k for k, s in enumerate(LAMMPS_SPECIES)}
    pos = np.zeros((2 * M, 3))
    pos[:, 1] = 100.0 * np.repeat(np.arange(M), 2)
    pos[1::2, 0] = ref[:, 0]
    types = np.array([[zidx[int(a)], zidx[int(b)]] for a, b in ref[:, 1:3]]).reshape(-1)
    a = 2 * np.arange(M)
    ei = np.stack([np.stack([a, a + 1], 1).reshape(-1), np.stack([a + 1, a], 1).reshape(-1)])
    return ref, torch.from_numpy(pos), torch.from_numpy(types), torch.from_numpy(ei)


def _check_lammps(ref, e_atom, forces):
    pe = e_atom.view(-1, 2).sum(1).cpu().numpy()
    fx = forces[:, 0].reshape(-1, 2).cpu().numpy()
    np.testing.assert_allclose(fx[:, 0], ref[:, 4], atol=1e-5)
    np.testing.assert_allclose(fx[:, 1], ref[:, 5], atol=1e-5)
    np.testing.assert_allclose(pe, ref[:, 3], atol=1e-4)


def test_kernels_reproduce_lammps():
    ref, pos, types, ei = _lammps_pairs()
    m = ZBL(LAMMPS_SPECIES, LAMMPS_SPECIES, "metal", polynomial_cutoff_p=80.0, model_dtype=torch.float64)
    p = pos.cuda().requires_grad_(True)
    e = ops.zbl_energy(p, ei.cuda(), types.cuda(), m.table("cuda"), r_max=9.0, poly_p=80.0)
    (g,) = torch.autograd.grad(e.sum(), p)
    _check_lammps(ref, e.detach(), -g)


def test_model_reproduces_lammps():
    """A float64 model whose readout is zeroed: its energy and forces are the ZBL term alone."""
    ref, pos, types, ei = _lammps_pairs()
    model = NequIPEnergyModel(r_max=9.0, type_names=LAMMPS_SPECIES, num_layers=2, l_max=1, num_features=8,
                              model_dtype=torch.float64,
                              pair_potential=_zbl_spec(LAMMPS_SPECIES, polynomial_cutoff_p=80)).cuda()
    with torch.no_grad():
        model.readout.mlp[0].weight.zero_()
    out = model({"pos": pos.cuda(), "atom_types": types.cuda(), "edge_index": ei.cuda()})
    _check_lammps(ref, out["atomic_energy"], out["forces"])


# ------------------------------------------------------------------------------------------------------------------
# kernels against the float64 oracle
# ------------------------------------------------------------------------------------------------------------------
def _frame(kind, n_side, seed=0):
    sysd = D.make_system(kind, n_side, r_max=R_MAX, seed=seed)
    meta = sysd.pop("_meta")
    return sysd, meta


SPECIES = {"water": ["Cu", "Au"], "li3po4": ["H", "Cu", "Au"]}


def _oracle(sysd, m, p, w):
    """e_atom, d(w . e_atom)/dpos and d(w . e_atom)/d(edge vectors) of the oracle ZBL (float64, CPU)."""
    ei, types, N = sysd["edge_index"], sysd["atom_types"], sysd["atom_types"].numel()
    pos = sysd["pos"].detach().clone().requires_grad_(True)
    vec = omodel.edge_vectors(pos, ei, sysd.get("cell"), sysd.get("edge_cell_shift"))
    args = (m.atomic_numbers.cpu(), m._qqr2exesquare.cpu(), p, R_MAX)
    e = opair.zbl_atom_energy(*args, vec, types, ei, N, torch.float64)
    (gpos,) = torch.autograd.grad(e, pos, w)
    v = vec.detach().requires_grad_(True)
    (gvec,) = torch.autograd.grad(opair.zbl_atom_energy(*args, v, types, ei, N, torch.float64), v, w)
    return e.detach(), gpos, gvec


def _kernel(sysd, m, p, w):
    sink = {}
    pos = sysd["pos"].cuda().requires_grad_(True)
    cell = sysd.get("cell")
    e = ops.zbl_energy(pos, sysd["edge_index"].cuda(), sysd["atom_types"].cuda(), m.table("cuda"),
                       shift=None if cell is None else sysd["edge_cell_shift"].cuda(),
                       cell=None if cell is None else cell.cuda(), r_max=R_MAX, poly_p=p, edge_grad_sink=sink)
    (gpos,) = torch.autograd.grad(e, pos, w.cuda())
    return e.detach().cpu(), gpos.cpu(), sink["pair_edge_vector_grad"].cpu()


def _compare(sysd, m, p=6.0, seed=0):
    N = sysd["atom_types"].numel()
    w = torch.randn(N, 1, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    got, ref = _kernel(sysd, m, p, w), _oracle(sysd, m, p, w)
    for what, a, b in zip(("e_atom", "grad_pos", "grad_vec"), got, ref):
        if b.numel() and float(b.abs().max()) > 0:
            assert _rel(a, b) <= 1e-12, (what, _rel(a, b))
        else:
            assert float(a.abs().max()) == 0 if a.numel() else True, what
    return got


@pytest.mark.timeout(600)
@pytest.mark.parametrize("kind,n_side", [("water", 10), ("li3po4", 22)])
def test_kernels_match_oracle(kind, n_side):
    sysd, meta = _frame(kind, n_side)
    m = ZBL(meta["type_names"], SPECIES[kind], "metal", model_dtype=torch.float64)
    got = _compare(sysd, m)
    assert float(got[0].abs().sum()) > 1.0  # ZBL is not negligible on these frames
    if kind == "water":
        # unsorted edges: the destination CSR carries a permutation
        E = sysd["edge_index"].shape[1]
        perm = torch.randperm(E, generator=torch.Generator().manual_seed(3))
        shuffled = dict(sysd, edge_index=sysd["edge_index"][:, perm], edge_cell_shift=sysd["edge_cell_shift"][perm])
        e2, g2, v2 = _compare(shuffled, m, p=9.0, seed=1)
        # atoms without edges: drop every row of the first 100 atoms
        keep = sysd["edge_index"][0] >= 100
        holes = dict(sysd, edge_index=sysd["edge_index"][:, keep], edge_cell_shift=sysd["edge_cell_shift"][keep])
        e3, _g3, _v3 = _compare(holes, m)
        assert bool((e3[:100] == 0).all()) and bool((e3[100:] != 0).any())
        # no edges at all
        empty = dict(sysd, edge_index=sysd["edge_index"][:, :0], edge_cell_shift=sysd["edge_cell_shift"][:0])
        e4, g4, v4 = _kernel(empty, m, 6.0, torch.ones(sysd["atom_types"].numel(), 1, dtype=torch.float64))
        assert e4.shape == (sysd["atom_types"].numel(), 1) and bool((e4 == 0).all()) and bool((g4 == 0).all())
        assert v4.shape == (0, 3)


def test_float32_cutoff_rounding():
    """cutoff_dtype=float32 rounds f_c as a float32 model does: each edge energy moves by at most half a float32 ulp of
    itself, and the result matches the oracle with a float32 model dtype at the float32 tolerance."""
    sysd, meta = _frame("water", 6)
    m = ZBL(meta["type_names"], SPECIES["water"], "metal", model_dtype=torch.float32)
    pos, ei, types = sysd["pos"].cuda(), sysd["edge_index"].cuda(), sysd["atom_types"].cuda()
    kw = dict(shift=sysd["edge_cell_shift"].cuda(), cell=sysd["cell"].cuda(), r_max=R_MAX)
    e32 = ops.zbl_energy(pos, ei, types, m.table("cuda"), cutoff_dtype=torch.float32, **kw).cpu()
    e64 = ops.zbl_energy(pos, ei, types, m.table("cuda"), cutoff_dtype=torch.float64, **kw).cpu()
    assert not torch.equal(e32, e64)
    assert bool(((e32 - e64).abs() <= (2.0 ** -24 + 1e-13) * e64.abs()).all())
    vec = omodel.edge_vectors(sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"])
    ref = opair.zbl_atom_energy(m.atomic_numbers, m._qqr2exesquare, 6.0, R_MAX, vec, sysd["atom_types"],
                                sysd["edge_index"], sysd["atom_types"].numel(), torch.float32)
    assert _rel(e32, ref) <= 1e-5


def test_write_contract():
    sysd, meta = _frame("water", 6)
    m = ZBL(meta["type_names"], SPECIES["water"], "metal", model_dtype=torch.float64)
    dev = D.to_device(sysd, "cuda")
    N, E = dev["atom_types"].numel(), dev["edge_index"].shape[1]
    table = m.table("cuda")
    csr = ops.build_csr(dev["edge_index"][0].contiguous(), N)
    L, st = _capi.lib(), torch.cuda.current_stream().cuda_stream
    geom = (dev["pos"].data_ptr(), dev["edge_index"].data_ptr(), dev["edge_cell_shift"].data_ptr(),
            dev["cell"].data_ptr(), 0, dev["atom_types"].data_ptr(), table.data_ptr(), table.shape[0])
    e_atom, ck_e = guarded(N, 1, torch.float64)
    _capi.check(L.nqb_zbl_fwd(*geom, csr.row_ptr.data_ptr(), 0, N, E, R_MAX, 6.0, 0, e_atom.data_ptr(), st))
    ge = torch.randn(N, generator=torch.Generator().manual_seed(2), dtype=torch.float64).cuda()
    gen = torch.Generator().manual_seed(5)
    gpos, ck_p = guarded(N, 3, torch.float64, body="random", generator=gen)
    base = gpos.detach().cpu().clone()
    gvec, ck_v = guarded(E, 3, torch.float64)
    _capi.check(L.nqb_zbl_bwd(*geom, N, E, R_MAX, 6.0, 0, ge.data_ptr(), gpos.data_ptr(), gvec.data_ptr(), st))
    torch.cuda.synchronize()
    for ck, what in ((ck_e, "e_atom"), (ck_p, "grad_pos"), (ck_v, "grad_vec")):
        ck(what)
    assert not bool(is_poison(e_atom).any()) and not bool(is_poison(gvec).any())
    w = ge.cpu().view(-1, 1)
    e_ref, gpos_ref, gvec_ref = _oracle(sysd, m, 6.0, w)
    assert _rel(e_atom, e_ref) <= 1e-12
    assert _rel(gvec, gvec_ref) <= 1e-12
    assert float((gpos.cpu() - base - gpos_ref).abs().max()) <= 1e-12 * float(gpos_ref.abs().max()) + 1e-12 * float(base.abs().max())
    # the forward is bitwise repeatable
    e2, _ = guarded(N, 1, torch.float64)
    _capi.check(L.nqb_zbl_fwd(*geom, csr.row_ptr.data_ptr(), 0, N, E, R_MAX, 6.0, 0, e2.data_ptr(), st))
    assert torch.equal(e2, e_atom)


# ------------------------------------------------------------------------------------------------------------------
# whole models against the oracle
# ------------------------------------------------------------------------------------------------------------------
def _model(arch, type_names, species, dtype, ann, **kw):
    m = NequIPEnergyModel(r_max=R_MAX, type_names=type_names, parity=True, avg_num_neighbors=ann, model_dtype=dtype,
                          pair_potential=_zbl_spec(species), strict_fast_path=(dtype == torch.float32), **arch, **kw)
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _tilted(kind, n_side, ntypes=None, seed=5):
    sysd = cell_frame(kind, n_side, "tilted", seed=seed, outside=True)
    meta = sysd.pop("_meta")
    if ntypes is not None:  # relabel the atoms with ntypes types
        sysd["atom_types"] = torch.randint(0, ntypes, sysd["atom_types"].shape, generator=torch.Generator().manual_seed(seed))
    return sysd, meta


@pytest.mark.timeout(600)
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.float64, 1e-9)])
@pytest.mark.parametrize("which", ["tutorial", "water_1k_l2_f32"])
def test_models_match_oracle(which, dtype, tol):
    if which == "tutorial":
        sysd, meta = _tilted("water", 5, ntypes=4)
        model = _model(TUTORIAL, ["C", "H", "O", "Cu"], ["C", "H", "O", "Cu"], dtype, meta["avg_num_neighbors"])
    else:
        sysd, meta = _tilted("water", 5)
        model = _model(WATER_L2, meta["type_names"], ["H", "O"], dtype, meta["avg_num_neighbors"])
    out = model(D.to_device(sysd, "cuda"), compute_stress=True)
    e_ref, f_ref, s_ref, v_ref = opair.energy_forces_stress(model.state_dict(), model.config, sysd, dtype)
    _e, ea_ref, _f = opair.energy_and_forces(model.state_dict(), model.config, sysd, dtype)
    escale = float(ea_ref.abs().sum())
    assert abs(float(out["total_energy"]) - float(e_ref)) <= tol * escale
    assert _rel(out["atomic_energy"], ea_ref) <= tol
    for k, ref in (("forces", f_ref), ("stress", s_ref), ("virial", v_ref)):
        assert _rel(out[k], ref) <= tol, (k, _rel(out[k], ref))
    # the pair term is a sizeable part of the result (the comparison would be vacuous otherwise)
    no_zbl = dict(model.config, pair_potential=None)
    sd = {k: v for k, v in model.state_dict().items() if not k.startswith("pair_potential.")}
    _e0, ea0, f0 = omodel.energy_and_forces(sd, no_zbl, sysd, dtype)
    assert _rel(ea0, ea_ref) > 1e-2 and _rel(f0, f_ref) > 1e-2
    # ML-IAP branch: edge vectors in, edge forces out
    vec = omodel.edge_vectors(sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"])
    d = {k: v for k, v in sysd.items() if k not in ("cell", "edge_cell_shift")}
    d["edge_vectors"] = vec
    out_v = model(D.to_device(d, "cuda"))
    e_ref_v, g_ref = opair.edge_forces(model.state_dict(), model.config, d, dtype)
    assert _rel(out_v["edge_forces"], g_ref) <= tol
    assert abs(float(out_v["total_energy"]) - float(e_ref_v)) <= tol * escale
    # compute_forces=False gives the same energy
    e_only = model(D.to_device(sysd, "cuda"), compute_forces=False)
    assert abs(float(e_only["total_energy"]) - float(out["total_energy"])) <= 1e-12 * escale


def test_close_pair_finite_differences():
    """One pair pushed to 0.6 A, where ZBL dominates: forces == central differences of the energy (float64)."""
    sysd, meta = _frame("water", 4, seed=2)
    pos = sysd["pos"].clone()
    ei, sh = sysd["edge_index"], sysd["edge_cell_shift"]
    vec = omodel.edge_vectors(pos, ei, sysd["cell"], sh)
    e0 = int(torch.argmin(vec.norm(dim=1)))
    i, j = int(ei[0, e0]), int(ei[1, e0])
    pos[j] += (0.6 / float(vec[e0].norm()) - 1.0) * vec[e0]
    new_ei, new_sh = D.neighbor_list(pos.numpy(), sysd["cell"].numpy(), R_MAX)
    sysd = dict(sysd, pos=pos, edge_index=torch.from_numpy(new_ei), edge_cell_shift=torch.from_numpy(new_sh))
    model = _model(WATER_L2, meta["type_names"], ["H", "O"], torch.float64, meta["avg_num_neighbors"])
    dev = D.to_device(sysd, "cuda")
    out = model(dev)
    e_pair = model.pair_potential(dev["atom_types"], dev["edge_index"], R_MAX, pos=dev["pos"],
                                  shift=dev["edge_cell_shift"], cell=dev["cell"]).view(-1)
    assert float(e_pair[i]) > 1.0  # eV: the pair term dominates atom i
    f = out["forces"].cpu()
    eps = 1e-5
    for a in (i, j, (i + 7) % pos.shape[0]):
        for c in range(3):
            es = []
            for sgn in (+1, -1):
                p = dev["pos"].clone()
                p[a, c] += sgn * eps
                es.append(float(model(dict(dev, pos=p), compute_forces=False)["total_energy"]))
            fd = -(es[0] - es[1]) / (2 * eps)
            assert abs(fd - float(f[a, c])) <= 1e-6 * max(1.0, abs(fd)), (a, c, fd, float(f[a, c]))


# ------------------------------------------------------------------------------------------------------------------
# captured MD steps
# ------------------------------------------------------------------------------------------------------------------
def _md_frame(n_side=6, seed=0):
    sysd, meta = _frame("li3po4", n_side, seed)
    return D.to_device(sysd, "cuda"), meta


def _md_model(meta):
    return _model(WATER_L2, meta["type_names"], ["Cu", "P", "Au"], torch.float32, meta["avg_num_neighbors"])


def _eager(model, pos, cell, dev, stress=False):
    nl = ops.neighbor_list(pos, cell, True, R_MAX)
    out = model(dict(dev, pos=pos, cell=cell, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]),
                compute_stress=stress)
    return out, nl["edge_index"].shape[1]


def _assert_matches(out, ref, what, keys=("forces",)):
    e_ref = float(ref["total_energy"])
    torch.testing.assert_close(out["total_energy"], ref["total_energy"], rtol=1e-12, atol=1e-9 * abs(e_ref), msg=what)
    for k in keys:
        assert _rel(out[k], ref[k]) <= 2e-6, (what, k, _rel(out[k], ref[k]))


def test_graphed_md_step_fixed_cell():
    dev, meta = _md_frame()
    model = _md_model(meta)
    pos0 = dev["pos"].clone()
    g = GraphedMDStep(model, dev)
    for t in range(20):
        pos = D.oscillating_positions(pos0, t, period=50, seed=7)
        out = g(pos.cpu().pin_memory() if t % 2 else pos)
        ref, E = _eager(model, pos, dev["cell"], dev)
        assert int(out["num_edges"]) == E
        _assert_matches(out, ref, f"step {t}")


def test_graphed_md_step_variable_cell():
    dev, meta = _md_frame(n_side=5)
    model = _md_model(meta)
    pos0 = dev["pos"].clone()
    g = GraphedMDStep(model, dev, variable_cell=True)
    for t in range(12):
        S = D.oscillating_strain(t).cuda()
        pos, cell = D.oscillating_positions(pos0, t, period=50, seed=7) @ S, dev["cell"] @ S
        out = g(pos, cell.cpu() if t % 2 else cell)
        ref, E = _eager(model, pos, cell, dev, stress=True)
        assert int(out["num_edges"]) == E
        _assert_matches(out, ref, f"step {t}", keys=("forces", "stress", "virial"))


def test_padded_list_is_bitwise_the_exact_list():
    dev, meta = _md_frame()
    model = _md_model(meta)
    N, E = dev["pos"].shape[0], dev["edge_index"].shape[1]
    plan = ops.NeighborListPlan(N, dev["cell"], True, R_MAX, E + math.ceil(0.05 * E))
    nl = plan.run(dev["pos"])
    assert int(nl["num_edges"]) == E and int(nl["overflow"]) == 0
    table = model.pair_potential.table(dev["pos"].device)
    kw = dict(cell=dev["cell"], r_max=R_MAX, cutoff_dtype=torch.float32)
    exact = ops.zbl_energy(dev["pos"], dev["edge_index"], dev["atom_types"], table, shift=dev["edge_cell_shift"], **kw)
    padded = ops.zbl_energy(dev["pos"], nl["edge_index"], dev["atom_types"], table, shift=nl["edge_cell_shift"], **kw)
    assert torch.equal(exact, padded) and float(exact.abs().sum()) > 0
    ref = model(dev)
    out = model(dict(dev, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))
    assert torch.equal(out["atomic_energy"], ref["atomic_energy"]) and torch.equal(out["total_energy"], ref["total_energy"])


def test_graphed_md_step_recaptures():
    dev, meta = _md_frame(n_side=5)
    model = _md_model(meta)
    gen = torch.Generator().manual_seed(11)
    pos0 = dev["pos"] + 0.3 * torch.randn(tuple(dev["pos"].shape), generator=gen, dtype=torch.float64).cuda()
    E0 = ops.neighbor_list(pos0, dev["cell"], True, R_MAX)["edge_index"].shape[1]
    g = GraphedMDStep(model, dict(dev, pos=pos0), capacity=E0)
    g(pos0)
    out = g(dev["pos"])  # more edges than the capacity
    assert g.recaptures == 1
    ref, E1 = _eager(model, dev["pos"], dev["cell"], dev)
    assert int(out["num_edges"]) == E1 > E0
    _assert_matches(out, ref, "after re-capture")


# ------------------------------------------------------------------------------------------------------------------
# no pair potential: nothing new runs
# ------------------------------------------------------------------------------------------------------------------
def test_model_without_pair_potential_never_calls_zbl(monkeypatch):
    calls = []

    def boom(*a, **k):
        calls.append(1)
        raise AssertionError("ops.zbl_energy called")

    sysd, meta = _tilted("water", 4)
    dev = D.to_device(sysd, "cuda")
    plain = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
                              **WATER_L2).cuda()
    with_zbl = _model(WATER_L2, meta["type_names"], ["H", "O"], torch.float32, meta["avg_num_neighbors"])
    monkeypatch.setattr(ops, "zbl_energy", boom)
    plain(dev)
    plain(dev, compute_stress=True)
    plain(dev, compute_forces=False)
    vec = omodel.edge_vectors(sysd["pos"], sysd["edge_index"], sysd["cell"], sysd["edge_cell_shift"]).cuda()
    plain({k: v for k, v in dev.items() if k not in ("cell", "edge_cell_shift")} | {"edge_vectors": vec})
    assert calls == []
    with pytest.raises(AssertionError):
        with_zbl(dev)
    assert calls == [1]


# ------------------------------------------------------------------------------------------------------------------
# sharded step (two GPUs)
# ------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _shard_worker(rank, world, port, sysd, meta, ret):
    import torch.distributed as dist

    from nequip_b200 import parallel as P

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        model = _model(WATER_L2, meta["type_names"], ["Cu", "P", "Au"], torch.float32, meta["avg_num_neighbors"]).to(dev)
        grid = P.brick_grid(world, torch.diagonal(sysd["cell"]).tolist())
        plan = P.make_plans(sysd["edge_index"], P.brick_owner(sysd["pos"], grid), world)[rank]
        local = D.to_device(P.shard_data(sysd, plan), dev)
        halo = P.HaloExchange(plan, dev)
        e, f_own = P.sharded_energy_forces(model, local, plan, halo, reduce_forces="owner")
        ret[f"f{rank}"] = (plan.owned.cpu(), f_own.cpu())
        if rank == 0:
            ret["e"] = e.cpu()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(900)
def test_sharded_step_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    sysd, meta = _frame("li3po4", 10, seed=2)
    torch.manual_seed(123)
    ref = _model(WATER_L2, meta["type_names"], ["Cu", "P", "Au"], torch.float32, meta["avg_num_neighbors"])(
        D.to_device(sysd, "cuda:0"))
    ret = mp.Manager().dict()
    mp.spawn(_shard_worker, args=(2, _free_port(), sysd, meta, ret), nprocs=2, join=True)
    f = torch.zeros_like(ref["forces"].cpu())
    for r in range(2):
        ids, fo = ret[f"f{r}"]
        f[ids] = fo
    assert abs(float(ret["e"]) - float(ref["total_energy"])) <= 1e-5 * float(ref["atomic_energy"].abs().sum())
    assert _rel(f, ref["forces"]) <= 1e-5
