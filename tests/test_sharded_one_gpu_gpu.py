"""The halo-sharded model on ONE GPU: W gloo ranks (separate processes) share cuda:0 and run the product's own
``parallel.HaloExchange`` / ``owner_reduce`` / ``sharded_energy_forces`` and ``NequIPEnergyModel.energy_owned`` on the
CUDA kernels.  gloo moves CUDA tensors through the host (NCCL refuses two ranks on one device), so the atom-partitioned
path is checked on a one-GPU box: the transport bitwise against a hand computation, and every case per atom against
the unsharded model on the same GPU and the float64 CPU oracle.

Each case reaches something only a sharded frame feeds the kernels: rows without in-edges (every ghost), source
indices past ``n_own``, GEMMs on prefix views ``x[:n_own]``, local pair maps with unpaired boundary edges, ghost types
deciding per-edge-type cutoffs, ZBL truncated to the owned rows, and ghosts reached through several cell shifts.
The sharded CUDA graph stays with the NCCL test (gloo collectives cannot be captured)."""
import os
import socket
import warnings
from datetime import timedelta

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import edge_type_oracle as eto
import preset_oracle as po
from cell_frames import brute_list, cell_frame
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200 import parallel as P
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel
from oracle import pair as opair

pytestmark = pytest.mark.gpu

R_MAX = 5.0
BENCH = dict(l_max=2, num_layers=4, num_features=64, radial_mlp_depth=1, radial_mlp_width=128)
SMALL = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)
TUTORIAL = dict(l_max=1, num_layers=4, num_features=32, radial_mlp_depth=2, radial_mlp_width=64)
# the asymmetric partial table of the edge-type tests: Li-O 4.1, O-Li 2.7
LI3PO4_TABLE = {"Li": {"Li": 3.2, "O": 4.1}, "P": 3.6, "O": {"Li": 2.7, "O": 4.4}}
ZBL_LI3PO4 = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "O"]}


# ------------------------------------------------------------------------------------------------------------------
# harness
# ------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _init(rank, world, port, ret):
    """Every rank on cuda:0, gloo; a rank that waits more than 120 s for the others fails instead of hanging."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=120))
    ret[f"joined{rank}"] = True


def _spawn(worker, world, args):
    """``mp.spawn(worker, (world, port, *args, ret))`` -> ``ret`` as a plain dict.  The port is probed before the
    workers bind it, so a rendezvous can lose it to another process: only then is the spawn repeated, on a fresh port.
    A failure after every rank has joined is a failure of the test body and is raised as it is."""
    for attempt in range(2):
        with mp.Manager() as mgr:
            ret = mgr.dict()
            try:
                mp.spawn(worker, args=(world, _free_port(), *args, ret), nprocs=world, join=True)
                return dict(ret)
            except Exception:  # noqa: BLE001 - re-raised unless the rendezvous itself failed
                if attempt or all(ret.get(f"joined{r}", False) for r in range(world)):
                    raise


def _rel(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max()) / float(b.abs().max())


def _per_element(what, got, ref, rtol):
    """|got - ref| <= rtol |ref| + rtol max|ref| element by element; returns max|got - ref| / max|ref|."""
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    scale = float(ref.abs().max())
    bad = (got - ref).abs() > rtol * ref.abs() + rtol * scale
    assert not bool(bad.any()), (what, int(bad.sum()), _rel(got, ref))
    return _rel(got, ref)


# ------------------------------------------------------------------------------------------------------------------
# 1. the transport on CUDA tensors
# ------------------------------------------------------------------------------------------------------------------
# hand-made graphs: (owner of each atom, edges (centre, neighbour)).  World 2: rank 0 has no ghosts, rank 1 ghosts all
# of rank 0.  World 3: splits [0, 2, 0] / [1, 0, 3] / [4, 0, 0] received, atom 0 is sent to two ranks and atom 5 is
# the source of two edges of rank 0.
TRANSPORT = {
    2: ([0, 0, 0, 1, 1, 1, 1, 1],
        [(0, 1), (1, 2), (2, 0), (3, 0), (4, 1), (5, 2), (6, 2), (7, 4)]),
    3: ([0, 0, 0, 0, 1, 1, 1, 2, 2, 2, 2, 2],
        [(0, 4), (1, 5), (2, 5), (3, 1), (4, 0), (5, 7), (6, 8), (6, 9), (5, 0), (7, 0), (8, 1), (9, 2), (10, 3),
         (11, 10)]),
}
RECV_SPLITS = {2: [[0, 0], [3, 0]], 3: [[0, 2, 0], [1, 0, 3], [4, 0, 0]]}


def _transport_plans(world):
    owner, edges = TRANSPORT[world]
    ei = torch.tensor(edges, dtype=torch.long).t().contiguous()
    return P.make_plans(ei, torch.tensor(owner), world)


def _x_value(gid, c):
    """Small integers: every sum of a few of them is exact in float32, whatever the order."""
    return float((5 * gid + 3 * c) % 17 - 8)


def _g_value(rank, row, c):
    return float((11 * rank + 3 * row + c) % 9 - 4)


def _transport_worker(rank, world, port, ret):
    _init(rank, world, port, ret)
    try:
        plan = _transport_plans(world)[rank]
        dev = torch.device("cuda", 0)
        halo = P.HaloExchange(plan, dev)
        n_loc = plan.n_own + plan.n_ghost
        for dt in (torch.float32, torch.float64):
            x = torch.tensor([[_x_value(int(g), c) for c in range(4)] for g in plan.owned], dtype=dt)
            x = x.reshape(plan.n_own, 4).to(dev).requires_grad_(True)
            g = torch.tensor([[_g_value(rank, r, c) for c in range(4)] for r in range(n_loc)], dtype=dt)
            g = g.reshape(n_loc, 4).to(dev)
            full = halo(x)
            (gx,) = torch.autograd.grad(full, x, g)
            red = P.owner_reduce(g[:, :3].contiguous(), plan, halo)
            torch.cuda.synchronize()
            ret[f"{rank}/{dt}"] = (full.detach().cpu(), gx.cpu(), red.cpu(), full.device.type, gx.device.type)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("world", [2, 3])
def test_halo_exchange_and_owner_reduce_on_cuda_tensors_are_exact(world):
    """``HaloExchange`` forward (owners' rows into the ghosts' rows), its backward (ghost gradients added into the
    owners' rows) and ``owner_reduce`` on cuda:0 tensors moved by gloo, bitwise against the result computed by hand
    from the plans.  If this torch build's gloo refuses CUDA tensors, this fails with its message."""
    plans = _transport_plans(world)
    assert [p.recv_splits for p in plans] == RECV_SPLITS[world]
    assert any(0 in p.send_splits[:r] + p.send_splits[r + 1:] for r, p in enumerate(plans))  # a zero split to a rank
    ret = _spawn(_transport_worker, world, ())
    for r, p in enumerate(plans):
        n_own = p.n_own
        # the owners' share of every ghost gradient, by hand from all the plans
        want_g = [[_g_value(r, i, c) for c in range(4)] for i in range(n_own)]
        for s, q in enumerate(plans):
            for k, gid in enumerate(q.ghosts.tolist()):
                if gid in p.owned.tolist():
                    i = p.owned.tolist().index(gid)
                    for c in range(4):
                        want_g[i][c] += _g_value(s, q.n_own + k, c)
        ids = p.owned.tolist() + p.ghosts.tolist()
        want_full = [[_x_value(gid, c) for c in range(4)] for gid in ids]
        for dt in (torch.float32, torch.float64):
            full, gx, red, dev_full, dev_g = ret[f"{r}/{dt}"]
            assert dev_full == "cuda" and dev_g == "cuda"
            wf = torch.tensor(want_full, dtype=dt).reshape(-1, 4)
            wg = torch.tensor(want_g, dtype=dt).reshape(-1, 4)
            assert torch.equal(full, wf), (r, dt, full, wf)
            assert torch.equal(gx, wg), (r, dt, gx, wg)
            assert torch.equal(red, wg[:, :3]), (r, dt, red, wg)


# ------------------------------------------------------------------------------------------------------------------
# 2. the sharded model against the unsharded model and the oracle
# ------------------------------------------------------------------------------------------------------------------
def _build(spec):
    """Frozen model on cuda:0 from ``spec`` = dict(preset=name or None, kwargs=constructor arguments, fused=bool)."""
    kw = spec["kwargs"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # float64 runs the torch dense blocks, by design
        if spec["preset"]:
            m = NequIPEnergyModel.from_preset(spec["preset"], **kw)
        else:
            m = NequIPEnergyModel(**kw)
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    for layer in m.layers:  # the path is chosen here, never by a per-rank timing ("auto")
        layer.conv.use_fused_radial_tp = bool(spec["fused"])
    return m


def _model_worker(rank, world, port, spec, state, frame, owner, ret):
    _init(rank, world, port, ret)
    try:
        if spec["det"]:
            ops.set_deterministic(True)
        dev = torch.device("cuda", 0)
        model = _build(spec)
        model.load_state_dict(state, strict=True)
        plan = P.make_plans(frame["edge_index"], owner, world)[rank]
        local = D.to_device(P.shard_data(frame, plan), dev)
        halo = P.HaloExchange(plan, dev)
        # what the model's forward really ran: its pair map, the fused kernel, the source-CSR cache
        maps, fused_calls, src_csr_nodes = [], [], []
        edge_pairs, tp_fused_fwd, src_get = model._edge_pairs, ops.tp_fused_fwd, ops.src_csr_cache.get

        def spy_pairs(*a):
            maps.append(edge_pairs(*a))
            return maps[-1]

        def spy_fused(*a, **k):
            fused_calls.append(1)
            return tp_fused_fwd(*a, **k)

        def spy_src(edge_src, num_nodes):
            src_csr_nodes.append(num_nodes)
            return src_get(edge_src, num_nodes)

        model._edge_pairs, ops.tp_fused_fwd, ops.src_csr_cache.get = spy_pairs, spy_fused, spy_src
        energies = []
        for _ in range(2 if spec["det"] else 1):
            pos = local["pos"].detach().requires_grad_(True)  # as sharded_energy_forces builds it
            with torch.enable_grad():
                e_own = model.energy_owned(dict(local, pos=pos), plan.n_own, halo)
            energies.append(e_own.detach().cpu())
        if e_own.shape != (plan.n_own, 1):  # every rank fails here alike: no rank is left waiting in a collective
            raise AssertionError(f"energy_owned returned {tuple(e_own.shape)} for {plan.n_own} owned atoms")
        e, f_own = P.sharded_energy_forces(model, local, plan, halo, reduce_forces="owner")
        e_g, f_g = P.sharded_energy_forces(model, local, plan, halo, reduce_forces="global")
        # both reductions of ONE local gradient: the two calls above run two backward passes, whose float32 atomics
        # add in arrival order, so only these agree to float64 rounding
        _e, f_loc = P.sharded_energy_forces(model, local, plan, halo, reduce_forces=False)
        f_loc_own = P.owner_reduce(f_loc, plan, halo)
        f_loc_g = torch.zeros((plan.num_global, 3), dtype=f_loc.dtype, device=dev)
        f_loc_g.index_add_(0, plan.local_ids.to(dev), f_loc)
        dist.all_reduce(f_loc_g)
        torch.cuda.synchronize()
        unpaired = None
        if maps[0] is not None:
            rows, count = maps[0]
            U = int(count)
            unpaired = int((rows[:U, 1] < 0).sum())
        ei = local["edge_index"]
        ret[rank] = dict(owned=plan.owned.clone(), e_own=energies, e=float(e), e_g=float(e_g), f_own=f_own.cpu(),
                         f_g=f_g.cpu(), f_loc_own=f_loc_own.cpu(), f_loc_g=f_loc_g.cpu(), n_ghost=plan.n_ghost, n_own=plan.n_own, unpaired=unpaired,
                         ghost_src_edges=int((ei[1] >= plan.n_own).sum()),
                         unsorted=bool((ei[0][1:] < ei[0][:-1]).any()) if ei.shape[1] > 1 else False,
                         fused_calls=len(fused_calls), src_csr_nodes=src_csr_nodes)
    finally:
        dist.destroy_process_group()


def _strip(fr):
    fr = dict(fr)
    meta = fr.pop("_meta", None)
    return fr, meta


def _frame(name):
    """(frame, meta) of the named frame, CPU tensors."""
    if name == "li3po4_512":
        return _strip(D.make_system("li3po4", 8, r_max=R_MAX, seed=2))
    if name == "li3po4_216":
        return _strip(D.make_system("li3po4", 6, r_max=R_MAX, seed=7))
    if name == "li3po4_125":
        return _strip(D.make_system("li3po4", 5, r_max=R_MAX, seed=3))
    if name == "li3po4_64":
        return _strip(D.make_system("li3po4", 4, r_max=R_MAX, seed=4))
    if name == "water_125":
        return _strip(D.make_system("water", 5, r_max=R_MAX, seed=3))
    if name == "tilted":
        return _strip(cell_frame("li3po4", 5, "tilted", seed=5))
    if name == "small":  # every perpendicular width below r_max: ghosts under several shifts, self-image edges
        return _strip(cell_frame("li3po4", 2, "small", seed=1))
    if name == "left":
        return _strip(cell_frame("li3po4", 4, "left", seed=2, outside=True))
    if name == "slab":
        return _strip(cell_frame("li3po4", 5, "tilted", seed=1, pbc=(True, True, False)))
    if name == "molecule":
        fr, meta = _strip(cell_frame("li3po4", 5, "cubic", seed=6, pbc=False))
        del fr["cell"], fr["edge_cell_shift"]
        return fr, meta
    if name == "shuffled":
        fr, meta = _strip(D.make_system("li3po4", 6, r_max=R_MAX, seed=5))
        perm = torch.randperm(fr["edge_index"].shape[1], generator=torch.Generator().manual_seed(9))
        fr["edge_index"] = fr["edge_index"][:, perm].contiguous()
        fr["edge_cell_shift"] = fr["edge_cell_shift"][perm].contiguous()
        return fr, meta
    if name == "clusters":  # two molecules 100 A apart
        a, meta = _strip(cell_frame("water", 3, "cubic", seed=8, pbc=False))
        pos = torch.cat([a["pos"], a["pos"] + torch.tensor([100.0, 0.0, 0.0], dtype=torch.float64)])
        ei, _sh = brute_list(pos.numpy(), None, False, R_MAX)
        fr = dict(pos=pos, atom_types=a["atom_types"].repeat(2), edge_index=torch.from_numpy(ei))
        return fr, meta
    raise KeyError(name)


# name: (frame, architecture, dtype, world, decomposition, fused, deterministic, extras)
CASES = {
    "bench_f32_slabs": ("li3po4_512", BENCH, torch.float32, 2, (2, 1, 1), False, False, {}),
    "bench_f32_slabs_fused": ("li3po4_512", BENCH, torch.float32, 2, (2, 1, 1), True, False, {}),
    "bench_f32_bricks": ("li3po4_512", BENCH, torch.float32, 4, (2, 2, 1), False, False, {}),
    "bench_f32_bricks_fused": ("li3po4_512", BENCH, torch.float32, 4, (2, 2, 1), True, False, {}),
    "bench_f64_water": ("water_125", BENCH, torch.float64, 3, "slab", False, False, {}),
    # the float32 variant keeps the 1 x 128 radial MLP that builds the pair map (whose slots the table refuses)
    "zbl_table_f32": ("tilted", dict(TUTORIAL, radial_mlp_depth=1, radial_mlp_width=128), torch.float32, 3, "slab",
                      False, False, dict(pair_potential=ZBL_LI3PO4, per_edge_type_cutoff=LI3PO4_TABLE)),
    "zbl_table_f64": ("tilted", TUTORIAL, torch.float64, 3, "slab", False, False,
                      dict(pair_potential=ZBL_LI3PO4, per_edge_type_cutoff=LI3PO4_TABLE)),
    "preset_M_f32": ("li3po4_125", "M", torch.float32, 2, "slab", False, False, {}),
    "preset_XL_f64": ("li3po4_64", "XL", torch.float64, 2, "slab", False, False, {}),
    "per_type_ann_f32": ("li3po4_216", dict(l_max=2, num_layers=3, num_features=32), torch.float32, 2, "slab", False,
                         False, dict(avg_num_neighbors={"Li": 31.0, "P": 58.5, "O": 47.25})),
    "deterministic_f32": ("li3po4_216", BENCH, torch.float32, 2, "slab", False, True, {}),
    "small_cell": ("small", SMALL, torch.float32, 2, "slab", False, False, {}),
    "left_cell": ("left", SMALL, torch.float32, 2, "slab", False, False, {}),
    "slab_TTF": ("slab", SMALL, torch.float32, 2, "slab", False, False, {}),
    "molecule": ("molecule", SMALL, torch.float32, 2, "slab", False, False, {}),
    "shuffled_edges": ("shuffled", SMALL, torch.float32, 2, "slab", False, False, {}),
    "clusters_no_ghosts": ("clusters", SMALL, torch.float32, 2, "slab", False, False, {}),
}

_ORACLE_CACHE = {}


def _spec(arch, dtype, meta, fused, det, extras):
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
              model_dtype=dtype, strict_fast_path=(dtype == torch.float32))
    if isinstance(arch, str):
        return dict(preset=arch, kwargs=dict(kw, **extras), fused=fused, det=det)
    return dict(preset=None, kwargs=dict(kw, parity=True, **arch, **extras), fused=fused, det=det)


def _oracle(frame_name, frame, model, spec):
    """(total energy, per-atom energies, forces) of the float64 CPU oracle that the feature's own tests use: the
    per-degree-width restatement for presets, the pair oracle with per-edge cutoffs for the ZBL + table models,
    ``oracle.model`` otherwise.  One evaluation per frame and model (the bench variants share it)."""
    dtype = spec["kwargs"]["model_dtype"]
    key = (frame_name, spec["preset"], repr(model.config))
    if key not in _ORACLE_CACHE:
        sd, cfg = model.state_dict(), model.config
        if model.per_edge_type_cutoff is not None:
            recip = eto.edge_recip(frame["atom_types"], frame["edge_index"], model.per_edge_type_cutoff)
            with eto.per_edge_cutoffs(recip):
                _ORACLE_CACHE[key] = opair.energy_and_forces(sd, cfg, frame, dtype, tp_chunk=20000)
        elif spec["preset"]:
            _ORACLE_CACHE[key] = po.energy_and_forces(sd, cfg, frame, dtype, tp_chunk=20000)
        else:
            _ORACLE_CACHE[key] = omodel.energy_and_forces(sd, cfg, frame, dtype, tp_chunk=20000)
    return _ORACLE_CACHE[key]


def _owner(frame, world, decomposition):
    if decomposition == "slab":
        return P.slab_owner(frame["pos"], world)
    return P.brick_owner(frame["pos"], decomposition)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("case", list(CASES))
def test_sharded_model_matches_unsharded_and_oracle(case):
    frame_name, arch, dtype, world, decomposition, fused, det, extras = CASES[case]
    frame, meta = _frame(frame_name)
    spec = _spec(arch, dtype, meta, fused, det, extras)
    model = _build(spec)
    state = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    owner = _owner(frame, world, decomposition)
    plans = P.make_plans(frame["edge_index"], owner, world)
    # the unsharded model on the same GPU: the reference, and the warm-up that builds every kernel library the case
    # needs before W processes would otherwise compile the same ones at once
    prev = ops.deterministic()
    ops.set_deterministic(det)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = model(D.to_device(frame, "cuda"))
        ea_ref, f_ref = ref["atomic_energy"].detach().cpu(), ref["forces"].detach().cpu()
    finally:
        ops.set_deterministic(prev)
    ret = _spawn(_model_worker, world, (spec, state, frame, owner))
    N = frame["pos"].shape[0]
    tol_u = 2e-6 if dtype == torch.float32 else 1e-12
    tol_o = 1e-5 if dtype == torch.float32 else 1e-9

    # every atom is owned by exactly one rank
    seen = torch.zeros(N, dtype=torch.long)
    e_atom = torch.zeros(N, 1, dtype=torch.float64)
    f = torch.zeros(N, 3, dtype=torch.float64)
    for r in range(world):
        o = ret[r]
        assert torch.equal(o["owned"], plans[r].owned)
        seen[o["owned"]] += 1
        e_atom[o["owned"]] = o["e_own"][0]
        f[o["owned"]] = o["f_own"]
        # the two force reductions agree: of one gradient to rounding, of two calls to the backward's atomic-order noise
        fscale = float(o["f_g"].abs().max())
        assert float((o["f_loc_own"] - o["f_loc_g"][o["owned"]]).abs().max()) <= 1e-9 * fscale
        assert float((o["f_own"] - o["f_g"][o["owned"]]).abs().max()) <= tol_u * fscale
        assert o["e"] == o["e_g"] == ret[0]["e"]
        # the case reaches what it claims
        if case == "clusters_no_ghosts":
            assert o["n_ghost"] == 0 and sum(plans[r].send_splits) == 0
        else:
            assert o["n_ghost"] > 0 and o["ghost_src_edges"] > 0
        # every float32 case has the 1 x 128 radial MLP that shares rows over a pair map; float64 builds none
        assert (o["unpaired"] is not None) == (dtype == torch.float32), "pair map built / not built"
        if o["unpaired"] is not None:
            assert o["unpaired"] >= o["ghost_src_edges"]  # an edge from a ghost has no partner on this rank
        if case == "zbl_table_f32":
            assert o["unpaired"] > o["ghost_src_edges"]  # pairs refused by the asymmetric table among the owned
        assert o["fused_calls"] > 0 if fused else o["fused_calls"] == 0
        if det:
            assert torch.equal(o["e_own"][0], o["e_own"][1])  # bitwise repeatable
            assert o["n_own"] + o["n_ghost"] in o["src_csr_nodes"]  # the source CSR over owned + ghost rows
        if case == "shuffled_edges":
            assert o["unsorted"]  # the local lists carry a permutation
    assert bool((seen == 1).all())
    if case == "small_cell":
        for p in plans:
            ei = p.edge_index
            assert bool((ei[0] == ei[1]).any())  # self-image edges
            gh = ei[:, ei[1] >= p.n_own]
            assert gh.shape[1] > torch.unique(gh[0] * (N + 1) + gh[1]).numel()  # a ghost under several shifts

    # per atom against the unsharded model on the same GPU
    err_ea = _per_element(f"{case}: atomic energies vs unsharded", e_atom, ea_ref, tol_u)
    err_f = _per_element(f"{case}: forces vs unsharded", f, f_ref, tol_u)
    # and against the float64 oracle
    e_ref_o, ea_ref_o, f_ref_o = _oracle(frame_name, frame, model, spec)
    escale = float(ea_ref_o.abs().sum())
    err_e_o = abs(ret[0]["e"] - float(e_ref_o)) / escale
    err_f_o = _rel(f, f_ref_o)
    err_ea_o = _rel(e_atom, ea_ref_o)
    print(f"sharded-1gpu {case}: W={world} N={N} ghosts={[ret[r]['n_ghost'] for r in range(world)]} "
          f"unpaired={[ret[r]['unpaired'] for r in range(world)]} | vs unsharded: max|dE_i|/max|E_i|={err_ea:.2e} "
          f"max|dF|/max|F|={err_f:.2e} | vs oracle: |dE|/sum|E_i|={err_e_o:.2e} max|dE_i|/max|E_i|={err_ea_o:.2e} "
          f"max|dF|/max|F|={err_f_o:.2e}")
    assert err_e_o <= tol_o, (case, err_e_o)
    assert err_f_o <= tol_o, (case, err_f_o)


# ------------------------------------------------------------------------------------------------------------------
# 3. the local pair map
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("frame_name,world,grid", [("li3po4_512", 4, (2, 2, 1)), ("shuffled", 2, (2, 1, 1)),
                                                   ("small", 2, (2, 1, 1))])
def test_local_pair_map_matches_host(frame_name, world, grid):
    """The reverse-edge pair map that ``energy_owned`` builds on each rank's local list (owned centres, ghost
    sources without a reverse edge) against the host restatement of its contract, rank by rank."""
    from test_edge_pairs_gpu import host_pairs

    frame, meta = _frame(frame_name)
    model = _build(_spec(BENCH, torch.float32, meta, False, False, {}))
    for plan in P.make_plans(frame["edge_index"], P.brick_owner(frame["pos"], grid), world):
        local = D.to_device(P.shard_data(frame, plan), "cuda")
        ei, sh = local["edge_index"], local["edge_cell_shift"]
        _v, _y, emb = ops.edge_embed(local["pos"], ei, sh, local["cell"], lmax=2, num_bessel=8, r_max=R_MAX,
                                     prefactor=2 * np.pi / R_MAX ** 2)
        rows, count = model._edge_pairs(ei, sh, emb, plan.n_own + plan.n_ghost)
        U = int(count)
        ref = host_pairs(ei.cpu().numpy(), sh.cpu().numpy(), emb.cpu().numpy())
        assert U == ref.shape[0] and np.array_equal(rows[:U].cpu().numpy(), ref), plan.rank
        unpaired = ref[ref[:, 1] < 0, 0]
        assert np.all(np.isin(np.nonzero(ei[1].cpu().numpy() >= plan.n_own)[0], unpaired))
