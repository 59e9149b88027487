"""The device MD driver on the GPU: the nqb_md kernels' write contracts and one step against the float64 oracle
(tests/md_oracle.py), ``GraphedMD`` against a host loop of the eager list, model and oracle update, block sizes, the
one host read per block, rollback after an overflowing block, and conservation."""
import math

import numpy as np
import pytest
import torch

import md_oracle as mo
from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import md, ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel

pytestmark = pytest.mark.gpu

R_MAX = 5.0
WATER_L2 = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)
MASSES = [1.008, 15.999]  # H, O
F_AGREE = 3e-7  # graphed against eager forces, relative to max|F| (DESIGN section 4.9)


def _ptr(t):
    return ops._ptr(t)


# ------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------
def _kernel_cases():
    """(counts, nblk) with nblk in {1, 2, the driver's min(64, ceil(max N_f / 256))}: frames at the CTA size, frames
    above 64 x 256 atoms (every CTA loops even at the driver's nblk) and empty frames.  nblk = 2 keeps the counts'
    name as its id."""
    named = [("one_frame", [37]), ("batch", [5, 600, 1, 0, 80]), ("cta_edges", [255, 256, 257]),
             ("above_64_ctas", [16384, 1, 16385]), ("large_empty_small", [20000, 0, 3])]
    cases = []
    for name, counts in named:
        driver = min(64, -(-max(counts) // 256))
        for nblk in sorted({1, 2, driver}):
            cases.append(pytest.param(counts, nblk, id=name if nblk == 2 else f"{name}-nblk{nblk}"))
    return cases


@pytest.mark.parametrize("counts,nblk", _kernel_cases())
@pytest.mark.parametrize("thermostat", [False, True], ids=["nve", "nh"])
def test_kernels_match_one_oracle_step_and_write_only_their_outputs(counts, nblk, thermostat):
    g = torch.Generator().manual_seed(len(counts) + 10 * thermostat)
    F, N = len(counts), sum(counts)
    ptr = [0] + np.cumsum(counts).tolist()
    pos = 10 * torch.rand(N, 3, generator=g, dtype=torch.float64)
    vel = torch.randn(N, 3, generator=g, dtype=torch.float64)
    frc = torch.randn(N, 3, generator=g, dtype=torch.float64)
    f_new = torch.randn(N, 3, generator=g, dtype=torch.float64)
    mass = 1 + 15 * torch.rand(N, generator=g, dtype=torch.float64)
    zeta = 0.1 * torch.randn(F, generator=g, dtype=torch.float64) if thermostat else torch.zeros(F, dtype=torch.float64)
    eta = torch.randn(F, generator=g, dtype=torch.float64) if thermostat else torch.zeros(F, dtype=torch.float64)
    gkT = torch.tensor([(3 * c + 1) * mo.KB * 150.0 if thermostat else 0.0 for c in counts], dtype=torch.float64)
    Q = 1 + 10 * torch.rand(F, generator=g, dtype=torch.float64) if thermostat else torch.zeros(F, dtype=torch.float64)
    e_pot = torch.randn(F, generator=g, dtype=torch.float64)
    dt = 0.5 * mo.FS
    # oracle
    ref = mo.nh_step(pos, vel, frc, mass, zeta, eta, lambda p: (e_pot, f_new), dt, gkT, Q, ptr, thermostat)
    r_pos, r_vel, _, r_zeta, r_eta, _ = ref
    r_ke = mo.kinetic(r_vel, mass, ptr)
    # device, guarded
    cu = dict(device="cuda")
    d_ptr = torch.tensor(ptr, dtype=torch.int64, device="cuda")
    d_mass, d_frc, d_fnew = mass.cuda(), frc.cuda(), f_new.cuda()
    d_gkT, d_Q, d_epot = gkT.cuda(), Q.cuda(), e_pot.cuda()
    d_pos, c_pos = guarded(N, 3, torch.float64, body=pos, **cu)
    d_vel, c_vel = guarded(N, 3, torch.float64, body=vel, **cu)
    d_part, c_part = guarded(F * nblk, 2, torch.float64, **cu)
    d_zeta, c_zeta = guarded(1, F, torch.float64, body=zeta.view(1, F), **cu)
    d_eta, c_eta = guarded(1, F, torch.float64, body=eta.view(1, F), **cu)
    d_out_f, c_out_f = guarded(N, 3, torch.float64, **cu)
    d_ke, c_ke = guarded(F, nblk, torch.float64, **cu)
    rows = 5
    d_log, c_log = guarded(rows * F, len(md.LOG_FIELDS), torch.float64, **cu)
    d_flags, c_flags = guarded(1, 4, torch.int64, body=torch.tensor([[0, 0, -1, 3]]), **cu)
    d_step, c_step = guarded(1, 1, torch.int64, body=torch.tensor([[12]]), **cu)
    ne = torch.tensor([7], dtype=torch.int64, device="cuda")
    ov = torch.tensor([1], dtype=torch.int32, device="cuda")
    srt = torch.tensor([0], dtype=torch.int32, device="cuda")
    L, st = _capi.lib(), ops._stream()
    _capi.check(L.nqb_md_kick_drift(F, nblk, _ptr(d_ptr), _ptr(d_mass), _ptr(d_frc), _ptr(d_zeta), dt, _ptr(d_pos),
                                    _ptr(d_vel), _ptr(d_part), st))
    if thermostat:
        _capi.check(L.nqb_md_bath(F, nblk, _ptr(d_part), _ptr(d_gkT), _ptr(d_Q), dt, _ptr(d_zeta), _ptr(d_eta), st))
    _capi.check(L.nqb_md_kick(F, nblk, _ptr(d_ptr), _ptr(d_mass), _ptr(d_fnew), _ptr(d_zeta), dt, _ptr(d_vel),
                              _ptr(d_out_f), _ptr(d_ke), st))
    dof = torch.tensor([max(3 * c, 1) * mo.KB for c in counts], dtype=torch.float64, device="cuda")
    _capi.check(L.nqb_md_log(F, nblk, _ptr(d_epot), _ptr(d_ke), _ptr(d_zeta), _ptr(d_eta), _ptr(d_Q), _ptr(d_gkT),
                             _ptr(dof), _ptr(ne), _ptr(ov), _ptr(srt), rows, _ptr(d_step), _ptr(d_log), _ptr(d_flags),
                             st))
    torch.cuda.synchronize()
    for chk, what in ((c_pos, "pos"), (c_vel, "vel"), (c_part, "part"), (c_zeta, "zeta"), (c_eta, "eta"),
                      (c_out_f, "forces"), (c_ke, "ke_part"), (c_log, "log"), (c_flags, "flags"), (c_step, "step")):
        chk(what)
    assert not bool(is_poison(d_part).any()) and not bool(is_poison(d_ke).any()) and not bool(is_poison(d_out_f).any())

    def close(got, want, what, tol=1e-14):
        got, want = got.cpu().reshape(want.shape), want
        scale = want.abs().max().clamp_min(1e-300)
        assert float((got - want).abs().max()) <= tol * float(scale), (what, float((got - want).abs().max() / scale))

    close(d_pos, r_pos, "pos")
    close(d_vel, r_vel, "vel")
    close(d_zeta, r_zeta, "zeta")
    close(d_eta, r_eta, "eta")
    assert torch.equal(d_out_f.cpu(), f_new)
    slot = d_log.view(rows, F, len(md.LOG_FIELDS)).cpu()
    written = slot[12 % rows]
    assert bool(is_poison(torch.cat([slot[:12 % rows], slot[12 % rows + 1:]])).all())  # one row only
    close(written[:, 0], e_pot, "e_pot")
    close(written[:, 1], r_ke, "e_kin")
    close(written[:, 3], r_zeta, "zeta")
    close(written[:, 5], mo.conserved(e_pot, r_vel, mass, r_zeta, r_eta, gkT, Q, ptr), "H")
    assert d_step.cpu().item() == 13
    assert d_flags.cpu().view(-1).tolist() == [1, 1, 12, 7]


# ------------------------------------------------------------------------------------------------------------------
# GraphedMD against a host loop
# ------------------------------------------------------------------------------------------------------------------
def _model(names, ann, dtype=torch.float32):
    m = NequIPEnergyModel(r_max=R_MAX, type_names=names, avg_num_neighbors=ann, model_dtype=dtype, parity=True,
                          strict_fast_path=(dtype == torch.float32), **WATER_L2).cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _cluster(seed, n=21):
    s = D.make_system("water", 4, r_max=R_MAX, seed=seed)
    p = s["pos"].numpy()
    keep = np.sort(np.argsort(np.linalg.norm(p - p.mean(0), axis=1), kind="stable")[:n])
    return torch.from_numpy(p[keep].copy()), s["atom_types"].view(-1)[torch.from_numpy(keep)], s["_meta"]


def _case(kind):
    """(example on cuda, eager-list arguments, meta)."""
    if kind in ("water", "slab"):
        s = D.make_system("water", 4, r_max=R_MAX, seed=1)
        ex = {"pos": s["pos"].double(), "atom_types": s["atom_types"].view(-1), "cell": s["cell"].double().view(3, 3)}
        if kind == "slab":
            ex["pbc"] = torch.tensor([True, True, False])
        meta = s["_meta"]
    elif kind == "molecule":
        pos, types, meta = _cluster(3)
        ex = {"pos": pos, "atom_types": types}
    else:  # a batch: two periodic water boxes of 81 and 192 atoms
        fr = [D.make_system("water", n, r_max=R_MAX, seed=5 + n) for n in (3, 4)]
        meta = fr[1]["_meta"]
        counts = [f["pos"].shape[0] for f in fr]
        ex = {"pos": torch.cat([f["pos"].double() for f in fr]),
              "atom_types": torch.cat([f["atom_types"].view(-1) for f in fr]),
              "cell": torch.stack([f["cell"].double().view(3, 3) for f in fr]),
              "batch": torch.repeat_interleave(torch.arange(2), torch.tensor(counts)),
              "num_atoms": torch.tensor(counts), "pbc": torch.ones(2, 3, dtype=torch.bool)}
    return {k: v.cuda() for k, v in ex.items()}, meta


def _eager(model, ex, pos):
    pbc = ex.get("pbc", ex.get("cell") is not None)
    nl = ops.neighbor_list(pos, ex.get("cell"), pbc, R_MAX, **({"batch": ex["batch"]} if "batch" in ex else {}))
    d = dict(ex, pos=pos, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"])
    d.pop("pbc", None)
    out = model(d)
    return out["total_energy"].detach().double().view(-1), out["forces"].detach().double()


def _host_loop(model, ex, mass, md0, n, dt, gkT, Q, thermostat):
    """The oracle update around the eager list and model, from GraphedMD's initial state ``md0``."""
    ptr = md0["ptr"]
    pos, vel, f = md0["pos"].clone(), md0["vel"].clone(), md0["forces"].clone()
    F = len(ptr) - 1
    zeta = torch.zeros(F, dtype=torch.float64, device="cuda")
    eta = torch.zeros_like(zeta)
    out = []
    for _ in range(n):
        pos, vel, f, zeta, eta, e = mo.nh_step(pos, vel, f, mass, zeta, eta, lambda p: _eager(model, ex, p), dt,
                                               gkT, Q, ptr, thermostat)
        out.append((pos.clone(), e.clone(), mo.conserved(e, vel, mass, zeta, eta, gkT, Q, ptr)))
    return out


def _initial(m):
    counts = [m._atom_ptr[i + 1].item() - m._atom_ptr[i].item() for i in range(m.num_frames)]
    return {k: v.clone() for k, v in m.state.items()} | {"ptr": [0] + np.cumsum(counts).tolist()}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", ["water", "slab", "molecule", "batch"])
@pytest.mark.parametrize("thermostat", [None, "nose_hoover"])
def test_graphed_md_matches_a_host_loop(kind, thermostat):
    """20 steps at 0.5 fs.  Graphed and eager forces agree to F_AGREE max|F| at equal positions, so after n steps the
    positions differ by at most about sum_k k dt^2 F_AGREE max|F| / m_min < n^2 dt^2 F_AGREE max|F| / m_min (a factor
    10 of slack for the growth of the difference through the forces); energies by N max|F| times that."""
    ex, meta = _case(kind)
    model = _model(meta["type_names"], meta["avg_num_neighbors"])
    nh = thermostat is not None
    kw = dict(thermostat=thermostat, temperature=300.0, nvt_q=5.0 if nh else None)
    m = md.GraphedMD(model, ex, MASSES, 0.5, **kw)
    md0 = _initial(m)
    n = 20
    log = m.run(n, block=8)
    mass = m._mass
    ref = _host_loop(model, ex, mass, md0, n, m.dt, m._gkT, m._Q, nh)
    fmax = float(md0["forces"].abs().max())
    dx = 10 * n * n * m.dt ** 2 * F_AGREE * fmax / float(mass.min()) + 1e-12
    N = ex["pos"].shape[0]
    assert float((m.state["pos"] - ref[-1][0]).abs().max()) <= dx
    e_ref = torch.stack([r[1] for r in ref]).cpu()
    h_ref = torch.stack([r[2] for r in ref]).cpu()
    de = N * fmax * dx + 1e-6 * float(e_ref.abs().max())
    assert log["e_pot"].shape == (n, m.num_frames)
    assert float((log["e_pot"] - e_ref).abs().max()) <= de
    assert float((log["conserved"] - h_ref).abs().max()) <= 2 * de
    assert m.recaptures == 0 and m.host_reads == 3 and int(m.state["step"]) == n


# ------------------------------------------------------------------------------------------------------------------
# blocks, host reads, rollback
# ------------------------------------------------------------------------------------------------------------------
def _replays_are_bitwise(model, ex):
    g = GraphedMDStep(model, ex)
    a = g(ex["pos"])["forces"].clone()
    b = g(ex["pos"])["forces"].clone()
    return torch.equal(a, b)


@pytest.mark.timeout(900)
def test_block_size_does_not_change_the_trajectory():
    """Blocks of 1, 7 and 20 steps replay the same captured step; only the host's reads between them differ.  The
    integrator kernels use no floating-point atomics, so the trajectories are bitwise equal whenever two replays of one
    captured step are.  On an H100 they are not, even under ``ops.set_deterministic(True)``: two replays of one
    ``GraphedMDStep`` at the same positions give forces that differ in the last bits.  So the trajectories are
    compared within the force tolerance of ``test_graphed_md_matches_a_host_loop``, and bitwise only if the replays
    are bitwise.  ``host_reads`` is ceil(n_steps / block)."""
    ex, meta = _case("batch")
    model = _model(meta["type_names"], meta["avg_num_neighbors"])
    prev = ops.deterministic()
    ops.set_deterministic(True)
    try:
        bitwise = _replays_are_bitwise(model, ex)
        runs = []
        for block in (1, 7, 20):
            m = md.GraphedMD(model, ex, MASSES, 0.5, thermostat="nose_hoover", temperature=[300.0, 500.0],
                             nvt_q=[5.0, 20.0])
            log = m.run(40, block=block)
            assert m.host_reads == math.ceil(40 / block)
            assert log["e_pot"].shape == (40, 2)
            runs.append((m.state["pos"].clone(), m.state["vel"].clone(), log))
    finally:
        ops.set_deterministic(prev)
    fmax = float(m.state["forces"].abs().max())
    dx = 10 * 40 * 40 * m.dt ** 2 * F_AGREE * fmax / float(m._mass.min()) + 1e-12
    de = ex["pos"].shape[0] * fmax * dx + 1e-6 * float(runs[0][2]["e_pot"].abs().max())
    for pos, vel, log in runs[1:]:
        if bitwise:
            assert torch.equal(pos, runs[0][0]) and torch.equal(vel, runs[0][1])
            for k in md.LOG_FIELDS:
                assert torch.equal(log[k], runs[0][2][k]), k
        else:
            assert float((pos - runs[0][0]).abs().max()) <= dx
            assert float((log["e_pot"] - runs[0][2]["e_pot"]).abs().max()) <= de


@pytest.mark.timeout(900)
def test_overflowing_block_is_rolled_back_and_rerun():
    ex, meta = _case("water")
    model = _model(meta["type_names"], meta["avg_num_neighbors"])
    E0 = ops.neighbor_list(ex["pos"], ex["cell"], True, R_MAX)["edge_index"].shape[1]
    prev = ops.deterministic()
    ops.set_deterministic(True)
    try:
        seen = []
        small = md.GraphedMD(model, ex, MASSES, 0.5, temperature=300.0, capacity=E0 // 2)
        log_s = small.run(30, block=10, on_block=lambda b: seen.append(b["e_pot"].shape[0]))
        ample = md.GraphedMD(model, ex, MASSES, 0.5, temperature=300.0)
        log_a = ample.run(30, block=10)
    finally:
        ops.set_deterministic(prev)
    assert small.recaptures >= 1 and small.capacity >= E0 and ample.recaptures == 0
    assert seen == [10, 10, 10] and log_s["e_pot"].shape == log_a["e_pot"].shape == (30, 1)
    assert small.host_reads == 3 + small.recaptures
    # a different capacity pads the rows with a different number of null edges, which changes nothing but the
    # order of float32 sums: the trajectories agree to the force tolerance
    fmax = float(ample.state["forces"].abs().max())
    dx = 10 * 30 * 30 * ample.dt ** 2 * F_AGREE * fmax / 1.008 + 1e-12
    assert float((small.state["pos"] - ample.state["pos"]).abs().max()) <= dx
    assert int(small.state["step"]) == 30


# ------------------------------------------------------------------------------------------------------------------
# conservation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_nve_conserves_energy_with_a_float64_model():
    """300 steps of 0.5 fs on the periodic water box with a float64 model: E_pot + E_kin stays within 1e-3 of the
    initial kinetic energy (velocity Verlet's error is O(dt^2) and bounded; the float64 forces add no noise)."""
    ex, meta = _case("water")
    model = _model(meta["type_names"], meta["avg_num_neighbors"], torch.float64)
    m = md.GraphedMD(model, ex, MASSES, 0.5, temperature=300.0)
    log = m.run(300, block=100)
    K0 = float(log["e_kin"][0])
    drift = float((log["conserved"] - log["conserved"][0]).abs().max())
    assert drift <= 1e-3 * K0, drift / K0


@pytest.mark.timeout(900)
def test_nose_hoover_conserves_h_and_keeps_a_molecule_from_rotating():
    """300 steps of 0.5 fs on a 21-atom molecule with a float64 model under the bath: H drifts by less than 3 % of the
    initial kinetic energy (the reference's update conserves H to first order in dt, tests/test_md_integrator.py), and
    the angular momentum, removed at the start, stays below 1e-9 of sum m |r| |v|."""
    ex, meta = _case("molecule")
    model = _model(meta["type_names"], meta["avg_num_neighbors"], torch.float64)
    m = md.GraphedMD(model, ex, MASSES, 0.5, thermostat="nose_hoover", temperature=300.0, nvt_q=5.0)
    log = m.run(300, block=50)
    K0 = float(log["e_kin"][0])
    assert float((log["conserved"] - log["conserved"][0]).abs().max()) <= 0.03 * K0
    pos, vel, mass = m.state["pos"].cpu(), m.state["vel"].cpu(), m._mass.cpu().unsqueeze(1)
    r = pos - (mass * pos).sum(0) / mass.sum()
    Lmom = torch.cross(r, mass * vel, dim=1).sum(0)
    assert float(Lmom.abs().max()) <= 1e-9 * float((r.norm(dim=1, keepdim=True) * mass * vel.norm(dim=1, keepdim=True)).sum())
    assert float((mass * vel).sum(0).abs().max()) <= 1e-9 * float((mass * vel.abs()).sum())
